// Training and eval batch norm followed by ReLU over the channel concatenation of a list of channels-last (NHWC) bf16
// segments, read where they lie: DenseNet's `relu(bn(torch.cat(features, 1)))` without the cat.
//
// Channel c of row r of the concatenation is channel c - c0[s] of row r of segment s, where c0[s] <= c < c0[s + 1]:
// seg[s] + r * C_s + (c - c0[s]).  Every segment has C_s % 8 == 0 and sits on the 16-byte grid, so no thread's group
// of 4 or 8 channels straddles two segments, and since a thread's channels are fixed across its row walk in every
// kernel below, it resolves its segment once.  Each kernel is the vector path of its bn:: counterpart
// (norm_kernels.cuh, norm_infer.cuh) with that counterpart's arithmetic, launch shape, row walk and merge order over
// the concatenation's m rows and C channels; only the segment loads differ.  So every result has the bits the
// counterpart writes for the concatenated tensor, which are eager torch's.  y, dy, dx and the mask are whole [m][C]
// tensors, read and written as the counterparts do.
//
// The segment table travels by value as a __grid_constant__ parameter: a run-time index into it reads the constant
// bank, where a by-value struct without that qualifier would be copied to the stack.  The elementwise kernels load
// segment rows with ld.global.nc (__ldg), as the counterparts' __restrict__ const operands compile; the reducing
// kernels copy them with cp.async into their rings, as the counterparts do.
#pragma once
#include "norm_infer.cuh"
#include "norm_kernels.cuh"
#include "norm_launch.h"

namespace b200c {
namespace bn_cat {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;
using bn::kEwVec;
using bn::kMaxBlock;
using bn::kParallelLoads;

using bn::kMaxCatSegs;

struct CatSegs {
  const bf16* ptr[kMaxCatSegs];
  int c0[kMaxCatSegs + 1];   // first channel of each segment; c0[n] = C
  int n;
};

// Where a thread's channels c .. c + V - 1 of row r lie: base + r * cs.
struct SegCol {
  const bf16* base;
  int cs;
  __device__ __forceinline__ const bf16* row(int r) const { return base + (size_t)r * cs; }
};

__device__ __forceinline__ SegCol seg_col(const CatSegs& segs, int c) {
  int lo = 0, hi = segs.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (segs.c0[mid] <= c) lo = mid;
    else hi = mid - 1;
  }
  return SegCol{segs.ptr[lo] + (c - segs.c0[lo]), segs.c0[lo + 1] - segs.c0[lo]};
}

__device__ __forceinline__ BVec<kEwVec> ldg8(const bf16* p) {
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  return *reinterpret_cast<const BVec<kEwVec>*>(&v);
}

// bn::k_bn_stats<kStatsVec> (bn_stats_body's ring path) over the concatenation.
__global__ void __launch_bounds__(kMaxBlock / bn::kStatsVec) k_cat_stats(const __grid_constant__ CatSegs segs, bn::StatsOut o,
                                                                         volatile float* staging_data, int* semaphores,
                                                                         const int reduction_size, const int stride) {
  constexpr int V = bn::kStatsVec;
  constexpr int PARALLEL_LOADS = kParallelLoads;
  if (o.num_batches_tracked && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0)
    *o.num_batches_tracked += 1;
  float x_mean[PARALLEL_LOADS][V];
  float m_2_n[PARALLEL_LOADS][V];
  int count[PARALLEL_LOADS];
#pragma unroll
  for (int i = 0; i < PARALLEL_LOADS; i++) {
#pragma unroll
    for (int k = 0; k < V; k++) {
      x_mean[i][k] = 0.f;
      m_2_n[i][k] = 0.f;
    }
    count[i] = 0;
  }

  int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  int c_offset = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  const bool c_valid = c_offset < stride;
  const SegCol col = c_valid ? seg_col(segs, c_offset) : SegCol{nullptr, 0};

  auto update = [&](int j, const BVec<V>* xv) {
    float x_math[V];
    float x_count_inv;
    float is_valid;
    if (c_valid && m_offset < reduction_size) {
      const BVec<V> x = *xv;
#pragma unroll
      for (int k = 0; k < V; k++) x_math[k] = __bfloat162float(x.v[k]);
      count[j]++;
      x_count_inv = float(1) / count[j];
      is_valid = float(1);
    } else {
#pragma unroll
      for (int k = 0; k < V; k++) x_math[k] = float(0);
      x_count_inv = float(0);
      is_valid = float(0);
    }
    m_offset += inner_loop_stride;
#pragma unroll
    for (int k = 0; k < V; k++) {
      float delta0 = x_math[k] - x_mean[j][k];
      x_mean[j][k] = __fmaf_rn(delta0, x_count_inv, x_mean[j][k]);
      float delta1 = x_math[k] - x_mean[j][k];
      m_2_n[j][k] = __fmaf_rn(__fmul_rn(delta0, delta1), is_valid, m_2_n[j][k]);
    }
  };

  constexpr unsigned D = bn::kStatsStages;
  const int threads = blockDim.x * blockDim.y;
  BVec<V>* ring = reinterpret_cast<BVec<V>*>(bn::ring_smem()) + threadIdx.y * blockDim.x + threadIdx.x;
  const int first_row = m_offset;
  auto issue = [&](unsigned it) {
    BVec<V>* slot = ring + (it % D) * PARALLEL_LOADS * threads;
    int m = first_row + (int)it * PARALLEL_LOADS * inner_loop_stride;
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride)
      if (c_valid && m < reduction_size) bn::cp_async<sizeof(BVec<V>)>(slot + j * threads, col.row(m));
    bn::cp_async_commit();
  };
#pragma unroll
  for (unsigned it = 0; it < D - 1; it++) issue(it);
  for (unsigned i = 0; i < (unsigned)loop_count; i++) {
    issue(i + D - 1);
    bn::cp_async_wait<D - 1>();
    const BVec<V>* slot = ring + (i % D) * PARALLEL_LOADS * threads;
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) update(j, slot + j * threads);
  }

  float mean_th[V], m2_th[V];
  int count_th[V];
#pragma unroll
  for (int k = 0; k < V; k++) {
    count_th[k] = count[0];
    mean_th[k] = x_mean[0][k];
    m2_th[k] = m_2_n[0][k];
#pragma unroll
    for (int j = 1; j < PARALLEL_LOADS; j++)
      bn::welford_merge_element<true>(count_th[k], mean_th[k], m2_th[k], count[j], x_mean[j][k], m_2_n[j][k]);
  }

  __shared__ float shmem_mean[kMaxBlock];
  __shared__ float shmem_m2n[kMaxBlock];
  __shared__ int shmem_count[kMaxBlock];
  bn::welford_merge_block_vertical<V>(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);

  if (gridDim.y > 1) {
    volatile float* staging_mean = staging_data;
    volatile float* staging_m2n = &staging_data[stride * gridDim.y];
    volatile int* staging_count = reinterpret_cast<volatile int*>(&staging_m2n[stride * gridDim.y]);
    int address_base = c_offset + blockIdx.y * stride;
    if (threadIdx.y == 0 && c_valid) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        staging_mean[address_base + k] = mean_th[k];
        staging_m2n[address_base + k] = m2_th[k];
        staging_count[address_base + k] = count_th[k];
      }
    }
    __threadfence();
    __syncthreads();
    __shared__ bool is_last_block_done;
    if (threadIdx.x == 0 && threadIdx.y == 0) {
      int old = atomicAdd(&semaphores[blockIdx.x], 1);
      is_last_block_done = (old == (gridDim.y - 1));
      if (is_last_block_done) semaphores[blockIdx.x] = 0;
    }
    __syncthreads();
    if (is_last_block_done) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        count_th[k] = 0;
        mean_th[k] = float(0.0);
        m2_th[k] = float(0.0);
      }
      for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
        address_base = c_offset + y * stride;
#pragma unroll
        for (int k = 0; k < V; k++) {
          int count_new = c_valid ? staging_count[address_base + k] : 0;
          float mean_new = c_valid ? staging_mean[address_base + k] : float(0.0);
          float m2n_new = c_valid ? staging_m2n[address_base + k] : float(0.0);
          bn::welford_merge_element<false>(count_th[k], mean_th[k], m2_th[k], count_new, mean_new, m2n_new);
        }
      }
      bn::welford_merge_block_vertical<V>(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);
      if (threadIdx.y == 0 && c_valid)
#pragma unroll
        for (int k = 0; k < V; k++) bn::finish_stats(o, c_offset + k, mean_th[k], m2_th[k], count_th[k]);
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_valid)
#pragma unroll
      for (int k = 0; k < V; k++) bn::finish_stats(o, c_offset + k, mean_th[k], m2_th[k], count_th[k]);
  }
}

// bn::k_bn_transform<kEwVec, kTailRelu> with its mask: y = relu(bf16(bn(x))) and one bit !(y <= 0) per element.
__global__ void __launch_bounds__(kEwThreads) k_cat_transform(const __grid_constant__ CatSegs segs, bf16* __restrict__ out,
                                                              uint8_t* __restrict__ mask, const float* __restrict__ mean,
                                                              const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                              const float* __restrict__ shift, const int reduction_size,
                                                              const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  const SegCol col = seg_col(segs, c0);
  float m_c[V], inv_std_c[V], w_c[V], s_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    m_c[j] = mean[c0 + j];
    inv_std_c[j] = inv_std[c0 + j];
    w_c[j] = weight[c0 + j];
    s_c[j] = shift[c0 + j];
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const int a = m * stride + c0;
    const BVec<V> xv = ldg8(col.row(m));
    BVec<V> yv;
    unsigned bits = 0;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
      bits |= (unsigned)!(__bfloat162float(yv.v[j]) <= 0.f) << j;
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
    mask[a >> 3] = (uint8_t)bits;
  }
}

// bn::k_bn_bwd_reduce<kGradBits, false> on its ring path (vec = kBwdVec, operands dy and x): g = mask ? dy : 0, the
// per-channel sums of g and g * (x - mean), and dweight / dbias.
__global__ void __launch_bounds__(kMaxBlock) k_cat_bwd_reduce(const __grid_constant__ CatSegs segs, const bf16* __restrict__ grad_output,
                                                              const uint8_t* __restrict__ mask, const float* __restrict__ mean,
                                                              const float* __restrict__ inv_std, float* __restrict__ sum_dy_o,
                                                              float* __restrict__ sum_dy_xmu_o, float* __restrict__ grad_weight,
                                                              float* __restrict__ grad_bias, volatile float* staging_data,
                                                              int* semaphores, const int reduction_size, const int stride) {
  constexpr int V = bn::kBwdVec;
  constexpr int PARALLEL_LOADS = kParallelLoads;
  constexpr unsigned D = bn::kBwdStages;
  __shared__ float shmem_sum_dy[kMaxBlock];
  __shared__ float shmem_sum_dy_xmu[kMaxBlock];
  __shared__ bool is_last_block_done;

  float sum_dy[PARALLEL_LOADS][V];
  float sum_dy_xmu[PARALLEL_LOADS][V];
#pragma unroll
  for (int i = 0; i < PARALLEL_LOADS; i++) {
#pragma unroll
    for (int k = 0; k < V; k++) {
      sum_dy[i][k] = float(0);
      sum_dy_xmu[i][k] = float(0);
    }
  }
  int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  int c_offset = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c_offset >= stride || m_offset >= reduction_size) return;
  const SegCol col = seg_col(segs, c_offset);

  int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  int address_base = m_offset * stride + c_offset;
  int address_increment = inner_loop_stride * stride;
  float r_mean[V], factor[V];
#pragma unroll
  for (int k = 0; k < V; k++) {
    r_mean[k] = mean[c_offset + k];
    factor[k] = inv_std[c_offset + k];
  }

  auto consume = [&](int j, const BVec<V>* dy_p, uint8_t mask_byte, const BVec<V>* x_p) {
    float x_input[V], x_grad_output[V];
    if (m_offset < reduction_size) {
      const unsigned bits = mask_byte >> (address_base & 7);
#pragma unroll
      for (int k = 0; k < V; k++) {
        x_input[k] = __bfloat162float(x_p->v[k]);
        x_grad_output[k] = __bfloat162float(bn::relu_grad_bit(dy_p->v[k], (bits >> k) & 1u));
      }
    } else {
#pragma unroll
      for (int k = 0; k < V; k++) {
        x_input[k] = float(0);
        x_grad_output[k] = float(0);
      }
    }
    m_offset += inner_loop_stride;
    address_base += address_increment;
#pragma unroll
    for (int k = 0; k < V; k++) {
      sum_dy[j][k] += x_grad_output[k];
      sum_dy_xmu[j][k] = __fmaf_rn(x_grad_output[k], x_input[k] - r_mean[k], sum_dy_xmu[j][k]);
    }
  };

  // the ring of dy (operand 0) and x (operand 1); the mask is a plain load one iteration ahead
  const int threads = blockDim.x * blockDim.y;
  BVec<V>* ring = reinterpret_cast<BVec<V>*>(bn::ring_smem()) + threadIdx.y * blockDim.x + threadIdx.x;
  auto stage = [&](unsigned it) { return ring + (it % D) * 2 * PARALLEL_LOADS * threads; };
  const int first_row = m_offset;
  const int iteration_rows = PARALLEL_LOADS * inner_loop_stride;
  auto issue = [&](unsigned it) {
    BVec<V>* slot = stage(it);
    int m = first_row + (int)it * iteration_rows;
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride, slot += threads) {
      if (m < reduction_size) {
        bn::cp_async<sizeof(BVec<V>)>(slot, grad_output + ((size_t)m * stride + c_offset));
        bn::cp_async<sizeof(BVec<V>)>(slot + PARALLEL_LOADS * threads, col.row(m));
      }
    }
    bn::cp_async_commit();
  };
  uint8_t mask_next[PARALLEL_LOADS];
  auto load_mask = [&](unsigned it) {
    int m = first_row + (int)it * iteration_rows;
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride)
      if (m < reduction_size) mask_next[j] = mask[((size_t)m * stride + c_offset) >> 3];
  };
  load_mask(0);
#pragma unroll
  for (unsigned it = 0; it < D - 1; it++) issue(it);
  for (unsigned i = 0; i < (unsigned)loop_count; i++) {
    issue(i + D - 1);
    uint8_t mask_v[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) mask_v[j] = mask_next[j];
    load_mask(i + 1);
    bn::cp_async_wait<D - 1>();
    const BVec<V>* slot = stage(i);
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++, slot += threads) consume(j, slot, mask_v[j], slot + PARALLEL_LOADS * threads);
  }

  float sum_dy_th[V], sum_dy_xmu_th[V];
#pragma unroll
  for (int k = 0; k < V; k++) {
#pragma unroll
    for (int j = 1; j < PARALLEL_LOADS; j++) {
      sum_dy[0][k] += sum_dy[j][k];
      sum_dy_xmu[0][k] += sum_dy_xmu[j][k];
    }
    sum_dy_th[k] = sum_dy[0][k];
    sum_dy_xmu_th[k] = sum_dy_xmu[0][k];
  }
  bn::merge_block_vertical_backward<V>(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);

  auto write_sums = [&]() {
#pragma unroll
    for (int k = 0; k < V; k++) {
      const int c = c_offset + k;
      grad_bias[c] = sum_dy_th[k];
      grad_weight[c] = sum_dy_xmu_th[k] * factor[k];
      sum_dy_o[c] = sum_dy_th[k];
      sum_dy_xmu_o[c] = sum_dy_xmu_th[k];
    }
  };
  if (gridDim.y > 1) {
    volatile float* staging_sum_dy = staging_data;
    volatile float* staging_sum_dy_xmu = &staging_data[stride * gridDim.y];
    address_base = c_offset + blockIdx.y * stride;
    if (threadIdx.y == 0 && c_offset < stride) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        staging_sum_dy[address_base + k] = sum_dy_th[k];
        staging_sum_dy_xmu[address_base + k] = sum_dy_xmu_th[k];
      }
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
      int old = atomicAdd(&semaphores[blockIdx.x], 1);
      is_last_block_done = (old == (gridDim.y - 1));
      if (is_last_block_done) semaphores[blockIdx.x] = 0;
    }
    __syncthreads();
    if (is_last_block_done) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        sum_dy_th[k] = float(0.0);
        sum_dy_xmu_th[k] = float(0.0);
      }
      for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
        address_base = c_offset + y * stride;
#pragma unroll
        for (int k = 0; k < V; k++) {
          sum_dy_th[k] += (c_offset < stride ? staging_sum_dy[address_base + k] : float(0.0));
          sum_dy_xmu_th[k] += (c_offset < stride ? staging_sum_dy_xmu[address_base + k] : float(0.0));
        }
      }
      bn::merge_block_vertical_backward<V>(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);
      if (threadIdx.y == 0 && c_offset < stride) write_sums();
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_offset < stride) write_sums();
  }
}

// bn::k_bn_bwd_elemt<kEwVec, kGradBits, false, false>: dx with g = mask ? dy : 0 and this call's norm_fct = 1 / m.
__global__ void __launch_bounds__(kEwThreads) k_cat_bwd_elemt(const __grid_constant__ CatSegs segs, const bf16* __restrict__ grad_output,
                                                              const uint8_t* __restrict__ mask, bf16* __restrict__ grad_input,
                                                              const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                              const float* __restrict__ weight, const float* __restrict__ sum_dy,
                                                              const float* __restrict__ sum_dy_xmu, const float norm_fct,
                                                              const int reduction_size, const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  const SegCol col = seg_col(segs, c0);
  float m_c[V], m_dy_c[V], factor_1_c[V], factor_2_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    m_c[j] = mean[c0 + j];
    m_dy_c[j] = sum_dy[c0 + j] * norm_fct;
    factor_1_c[j] = inv_std[c0 + j];
    factor_2_c[j] = weight[c0 + j] * factor_1_c[j];
    factor_1_c[j] = factor_1_c[j] * factor_1_c[j] * sum_dy_xmu[c0 + j] * norm_fct;
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const int a = m * stride + c0;
    const BVec<V> gv = *reinterpret_cast<const BVec<V>*>(grad_output + a);
    const unsigned bits = mask[a >> 3] >> (a & 7);
    const BVec<V> xv = ldg8(col.row(m));
    BVec<V> dxv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const float g = __bfloat162float(bn::relu_grad_bit(gv.v[j], (bits >> j) & 1u));
      dxv.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(xv.v[j]) - m_c[j]) * factor_1_c[j]) * factor_2_c[j]);
    }
    *reinterpret_cast<BVec<V>*>(grad_input + a) = dxv;
  }
}

// bn_infer::k_infer_transform<kEwVec, kTailRelu, P>: the eval site, y = relu(bf16(bn(x))) from the running statistics.
template <typename P>
__global__ void __launch_bounds__(kEwThreads) k_cat_infer(const __grid_constant__ CatSegs segs, bf16* __restrict__ out,
                                                          const P* __restrict__ running_mean, const P* __restrict__ running_var,
                                                          const P* __restrict__ weight, const P* __restrict__ bias, const float eps,
                                                          const int reduction_size, const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  const SegCol col = seg_col(segs, c0);
  float m_c[V], inv_std_c[V], w_c[V], s_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const bn_infer::Channel<P> k(running_mean, running_var, weight, bias, eps, c0 + j);
    m_c[j] = k.mean, inv_std_c[j] = k.inv_std, w_c[j] = k.w, s_c[j] = k.s;
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const BVec<V> xv = ldg8(col.row(m));
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
    }
    *reinterpret_cast<BVec<V>*>(out + m * stride + c0) = yv;
  }
}

}  // namespace bn_cat
}  // namespace b200c
