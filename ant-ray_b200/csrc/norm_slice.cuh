// Training and eval batch norm followed by ReLU whose output is a channel slice of a wider channels-last (NHWC) bf16
// tensor: Inception's and GoogLeNet's `torch.cat([relu(bn(conv(x))) for each branch], 1)` with each branch written
// into its channels of the concatenation, which is never assembled by a copy.
//
// x is the branch's own [m][C] tensor.  y is the slice out[:, c0:c0+C] of the module's [m][ldy] output: row r,
// channel c of the branch lands at y + r * ldy + c, where y already points at out + c0.  The backward reads dy, the
// gradient of y, the same way with its own row stride lddy; the mask is the branch's own m * C / 8 bytes.  C, ldy and
// lddy are multiples of 8 and x, y and dy sit on the 16-byte grid, so every thread's 8 channels are one 16-byte
// access as in the counterparts.  Each kernel is the vector path of its bn:: counterpart (norm_kernels.cuh,
// norm_infer.cuh) with that counterpart's arithmetic, launch shape, row walk and merge order over the branch's m rows
// and C channels; only the row stride of y or dy differs.  So every result has the bits the counterpart writes for
// the branch, which are eager torch's.  The statistics are bn::k_bn_stats itself: x is an ordinary tensor.
#pragma once
#include "norm_infer.cuh"
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_slice {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;
using bn::kEwVec;
using bn::kMaxBlock;
using bn::kParallelLoads;

// bn::k_bn_transform<kEwVec, kTailRelu> with its mask: y = relu(bf16(bn(x))) stored with row stride ldy, and one bit
// !(y <= 0) per element of the branch's own mask.
__global__ void __launch_bounds__(kEwThreads) k_slice_transform(const bf16* __restrict__ input, bf16* __restrict__ out, const int ldy,
                                                                uint8_t* __restrict__ mask, const float* __restrict__ mean,
                                                                const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                                const float* __restrict__ shift, const int reduction_size,
                                                                const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
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
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> yv;
    unsigned bits = 0;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
      bits |= (unsigned)!(__bfloat162float(yv.v[j]) <= 0.f) << j;
    }
    *reinterpret_cast<BVec<V>*>(out + m * ldy + c0) = yv;
    mask[a >> 3] = (uint8_t)bits;
  }
}

// bn::k_bn_bwd_reduce<kGradBits, false> on its ring path (vec = kBwdVec, operands dy and x): g = mask ? dy : 0 with dy
// read at row stride lddy, the per-channel sums of g and g * (x - mean), and dweight / dbias.
__global__ void __launch_bounds__(kMaxBlock) k_slice_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output,
                                                                const int lddy, const uint8_t* __restrict__ mask,
                                                                const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                                float* __restrict__ sum_dy_o, float* __restrict__ sum_dy_xmu_o,
                                                                float* __restrict__ grad_weight, float* __restrict__ grad_bias,
                                                                volatile float* staging_data, int* semaphores, const int reduction_size,
                                                                const int stride) {
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
        bn::cp_async<sizeof(BVec<V>)>(slot, grad_output + ((size_t)m * lddy + c_offset));
        bn::cp_async<sizeof(BVec<V>)>(slot + PARALLEL_LOADS * threads, input + ((size_t)m * stride + c_offset));
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

// bn::k_bn_bwd_elemt<kEwVec, kGradBits, false, false>: dx with g = mask ? dy : 0, dy read at row stride lddy, and this
// call's norm_fct = 1 / m.
__global__ void __launch_bounds__(kEwThreads) k_slice_bwd_elemt(const bf16* __restrict__ grad_output, const int lddy,
                                                                const uint8_t* __restrict__ mask, const bf16* __restrict__ input,
                                                                bf16* __restrict__ grad_input, const float* __restrict__ mean,
                                                                const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                                const float* __restrict__ sum_dy, const float* __restrict__ sum_dy_xmu,
                                                                const float norm_fct, const int reduction_size, const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
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
    const BVec<V> gv = *reinterpret_cast<const BVec<V>*>(grad_output + m * lddy + c0);
    const unsigned bits = mask[a >> 3] >> (a & 7);
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> dxv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const float g = __bfloat162float(bn::relu_grad_bit(gv.v[j], (bits >> j) & 1u));
      dxv.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(xv.v[j]) - m_c[j]) * factor_1_c[j]) * factor_2_c[j]);
    }
    *reinterpret_cast<BVec<V>*>(grad_input + a) = dxv;
  }
}

// bn_infer::k_infer_transform<kEwVec, kTailRelu, P>: the eval site, y = relu(bf16(bn(x))) from the running statistics,
// stored with row stride ldy.
template <typename P>
__global__ void __launch_bounds__(kEwThreads) k_slice_infer(const bf16* __restrict__ input, bf16* __restrict__ out, const int ldy,
                                                            const P* __restrict__ running_mean, const P* __restrict__ running_var,
                                                            const P* __restrict__ weight, const P* __restrict__ bias, const float eps,
                                                            const int reduction_size, const int stride) {
  constexpr int V = kEwVec;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], inv_std_c[V], w_c[V], s_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const bn_infer::Channel<P> k(running_mean, running_var, weight, bias, eps, c0 + j);
    m_c[j] = k.mean, inv_std_c[j] = k.inv_std, w_c[j] = k.w, s_c[j] = k.s;
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + m * stride + c0);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
    }
    *reinterpret_cast<BVec<V>*>(out + m * ldy + c0) = yv;
  }
}

}  // namespace bn_slice
}  // namespace b200c
