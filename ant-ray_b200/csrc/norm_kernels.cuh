// Training-mode batch norm over channels-last (NHWC) bf16 activations with fp32 weight, bias and statistics,
// fused with what follows it in a ResNet block: ReLU, or `+= identity` then ReLU.
//
// The statistics and backward-reduce kernels are ports of the channels-last kernels of PyTorch's
// aten/src/ATen/native/cuda/Normalization.cuh (PyTorch, BSD-3-Clause licence, Copyright (c) 2016- Facebook, Inc.
// and its contributors; the kernels originate in NVIDIA Apex).  They keep torch's launch shape, per-thread
// sequence of rows, block tree and grid merge, and torch's expressions, so that every per-channel sum is rounded
// exactly as torch rounds it.  That is what makes the outputs bit-identical to eager torch (torch 2.x runs bf16
// batch norm on these native kernels, not on cuDNN).  The elementwise kernels (transform, backward elementwise)
// have no cross-element rounding, so they are restructured freely: 16-byte loads of 8 channels per thread.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200c {
namespace bn {

// torch's constants (MAX_BLOCK_SIZE, ELEMENTS_PER_ITER, ELEMENTS_PER_THREAD, OPTIMAL_TILE_W, MAX_H_BLOCK): the
// reduction order depends on them.
constexpr int kMaxBlock = 512;
constexpr int kParallelLoads = 4;
constexpr int kElemsPerThread = 16;
constexpr int kTileW = 32;
constexpr int kMaxHBlock = 128;
// elementwise kernels
constexpr int kEwThreads = 256;
constexpr int kEwVec = 8;

typedef __nv_bfloat16 bf16;

template <int V>
struct alignas(2 * V) BVec {
  bf16 v[V];
};

// ---- reduction helpers (verbatim from torch) ----
__device__ __forceinline__ void welford_merge_element(int& count, float& mean, float& m2n, const int& count_new,
                                                      const float& mean_new, const float& m2n_new) {
  float factor = float(1.0) / ::max(1, (count + count_new));
  float delta0 = mean - mean_new;
  mean = (mean_new * count_new + mean * count) * factor;
  m2n += m2n_new + delta0 * delta0 * count_new * count * factor;
  count += count_new;
}

__device__ __forceinline__ void welford_merge_block_vertical(int& count, float& mean, float& m2n, int* shmem_count,
                                                             float* shmem_mean, float* shmem_m2n) {
  auto address_base = threadIdx.x + threadIdx.y * blockDim.x;
#pragma unroll
  for (int offset = blockDim.y / 2; offset > 0; offset >>= 1) {
    if (threadIdx.y < offset * 2) {
      shmem_mean[address_base] = mean;
      shmem_m2n[address_base] = m2n;
      shmem_count[address_base] = count;
    }
    __syncthreads();
    if (threadIdx.y < offset && threadIdx.y + offset < blockDim.y) {
      auto address = address_base + offset * blockDim.x;
      auto count_new = shmem_count[address];
      auto mean_new = shmem_mean[address];
      auto m2n_new = shmem_m2n[address];
      welford_merge_element(count, mean, m2n, count_new, mean_new, m2n_new);
    }
  }
}

__device__ __forceinline__ void merge_block_vertical_backward(float& sum_dy, float& sum_dy_xmu, float* shmem_sum_dy,
                                                              float* shmem_sum_dy_xmu) {
  auto address_base = threadIdx.x + threadIdx.y * blockDim.x;
#pragma unroll
  for (int offset = blockDim.y / 2; offset > 0; offset >>= 1) {
    if (threadIdx.y < offset * 2) {
      shmem_sum_dy[address_base] = sum_dy;
      shmem_sum_dy_xmu[address_base] = sum_dy_xmu;
    }
    __syncthreads();
    if (threadIdx.y < offset && threadIdx.y + offset < blockDim.y) {
      auto address = address_base + offset * blockDim.x;
      sum_dy += shmem_sum_dy[address];
      sum_dy_xmu += shmem_sum_dy_xmu[address];
    }
  }
}

struct StatsOut {
  float* save_mean;
  float* save_invstd;
  float* running_mean;
  float* running_var;
  long long* num_batches_tracked;  // may be null
  float momentum, bessel, eps;     // torch: static_cast<float> of momentum, N / (N - 1) in double, eps
};

// Channel c's final (mean, biased variance): what torch's statistics kernel writes, followed by the body of
// batch_norm_update_stats_and_invert, with the same expressions.
__device__ __forceinline__ void finish_stats(const StatsOut& o, int c, float mean_th, float m2_th, int count_th) {
  const float mean = mean_th;
  const float var = m2_th / count_th;
  const float momentum = o.momentum;
  const float unbiased_var = var * o.bessel;
  o.save_mean[c] = mean;
  o.running_mean[c] = mean * momentum + (1 - momentum) * o.running_mean[c];
  o.running_var[c] = unbiased_var * momentum + (1 - momentum) * o.running_var[c];
  o.save_invstd[c] = rsqrtf(var + o.eps);
}

// Welford statistics per channel (torch: batch_norm_collect_statistics_channels_last_kernel<Var, ..., 4>), then
// the running-statistics update and inversion by the thread that owns the channel's final value.  The last block
// of each column leaves its semaphore at zero for the next call.
__global__ void k_bn_stats(const bf16* __restrict__ input, StatsOut o, volatile float* staging_data, int* semaphores,
                           const int reduction_size, const int stride) {
  constexpr int PARALLEL_LOADS = kParallelLoads;
  float x_mean[PARALLEL_LOADS];
  float m_2_n[PARALLEL_LOADS];
  int count[PARALLEL_LOADS];
#pragma unroll
  for (int i = 0; i < PARALLEL_LOADS; i++) {
    x_mean[i] = 0.f;
    m_2_n[i] = 0.f;
    count[i] = 0;
  }
  if (o.num_batches_tracked && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0)
    *o.num_batches_tracked += 1;

  int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  int c_offset = blockIdx.x * blockDim.x + threadIdx.x;
  int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  int address_base = m_offset * stride + c_offset;
  int address_increment = inner_loop_stride * stride;

  for (int i = 0; i < loop_count; i++) {
    float x_math[PARALLEL_LOADS];
    float x_count_inv[PARALLEL_LOADS];
    float is_valid[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      if (c_offset < stride && m_offset < reduction_size) {
        x_math[j] = __bfloat162float(input[address_base]);
        count[j]++;
        x_count_inv[j] = float(1) / count[j];
        is_valid[j] = float(1);
      } else {
        x_math[j] = float(0);
        x_count_inv[j] = float(0);
        is_valid[j] = float(0);
      }
      m_offset += inner_loop_stride;
      address_base += address_increment;
    }
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      float delta0 = x_math[j] - x_mean[j];
      x_mean[j] += delta0 * x_count_inv[j];
      float delta1 = x_math[j] - x_mean[j];
      m_2_n[j] += delta0 * delta1 * is_valid[j];
    }
  }
#pragma unroll
  for (int j = 1; j < PARALLEL_LOADS; j++) welford_merge_element(count[0], x_mean[0], m_2_n[0], count[j], x_mean[j], m_2_n[j]);

  auto mean_th = x_mean[0];
  auto m2_th = m_2_n[0];
  auto count_th = count[0];

  __shared__ float shmem_mean[kMaxBlock];
  __shared__ float shmem_m2n[kMaxBlock];
  __shared__ int shmem_count[kMaxBlock];
  welford_merge_block_vertical(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);

  if (gridDim.y > 1) {
    volatile float* staging_mean = staging_data;
    volatile float* staging_m2n = &staging_data[stride * gridDim.y];
    volatile int* staging_count = reinterpret_cast<volatile int*>(&staging_m2n[stride * gridDim.y]);
    address_base = c_offset + blockIdx.y * stride;
    if (threadIdx.y == 0 && c_offset < stride) {
      staging_mean[address_base] = mean_th;
      staging_m2n[address_base] = m2_th;
      staging_count[address_base] = count_th;
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
      count_th = 0;
      mean_th = float(0.0);
      m2_th = float(0.0);
      for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
        address_base = c_offset + y * stride;
        int count_new = c_offset < stride ? staging_count[address_base] : 0;
        float mean_new = c_offset < stride ? staging_mean[address_base] : float(0.0);
        float m2n_new = c_offset < stride ? staging_m2n[address_base] : float(0.0);
        welford_merge_element(count_th, mean_th, m2_th, count_new, mean_new, m2n_new);
      }
      welford_merge_block_vertical(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);
      if (threadIdx.y == 0 && c_offset < stride) finish_stats(o, c_offset, mean_th, m2_th, count_th);
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_offset < stride) finish_stats(o, c_offset, mean_th, m2_th, count_th);
  }
}

// y = relu(bn(x)) (RESID false) or y = relu(bf16(bn(x)) + identity) (RESID true), rounded where eager torch
// rounds: the batch-norm output to bf16, the bf16 sum of the residual add to bf16.  `t <= 0 ? 0 : bf16(t)` is
// relu(bf16(t)) because rounding keeps the sign; NaN passes through as in torch's relu.
template <int V, bool RESID>
__global__ void __launch_bounds__(kEwThreads) k_bn_transform(const bf16* __restrict__ input, const bf16* __restrict__ identity,
                                                             bf16* __restrict__ out, const float* __restrict__ mean,
                                                             const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                             const float* __restrict__ shift, const int reduction_size,
                                                             const int stride) {
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
    BVec<V> zv;
    if (RESID) zv = *reinterpret_cast<const BVec<V>*>(identity + a);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      if (RESID) {
        const bf16 r = __float2bfloat16(__bfloat162float(__float2bfloat16(tmp)) + __bfloat162float(zv.v[j]));
        yv.v[j] = __bfloat162float(r) <= 0.f ? __float2bfloat16(0.f) : r;
      } else {
        yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
      }
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

// The ReLU's backward (threshold_backward: y <= 0 ? 0 : dy), read from dy and the saved output y.
__device__ __forceinline__ bf16 relu_grad(bf16 dy, bf16 y) { return __bfloat162float(y) <= 0.f ? __float2bfloat16(0.f) : dy; }

// Per-channel sums of g and g * (x - mean) with g = relu_grad(dy, y) (torch:
// batch_norm_backward_reduce_channels_last_kernel<4>), and dweight / dbias.  With `masked` set (the block tail,
// where g is also the identity branch's gradient) g is written there as well.
__global__ void k_bn_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output, const bf16* __restrict__ output,
                                bf16* __restrict__ masked, const float* __restrict__ mean, const float* __restrict__ inv_std,
                                float* __restrict__ sum_dy_o, float* __restrict__ sum_dy_xmu_o, float* __restrict__ grad_weight,
                                float* __restrict__ grad_bias, volatile float* staging_data, int* semaphores,
                                const int reduction_size, const int stride) {
  constexpr int PARALLEL_LOADS = kParallelLoads;
  float sum_dy[PARALLEL_LOADS];
  float sum_dy_xmu[PARALLEL_LOADS];
#pragma unroll
  for (int i = 0; i < PARALLEL_LOADS; i++) {
    sum_dy[i] = float(0);
    sum_dy_xmu[i] = float(0);
  }
  int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  int c_offset = blockIdx.x * blockDim.x + threadIdx.x;
  if (c_offset >= stride || m_offset >= reduction_size) return;

  int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  int address_base = m_offset * stride + c_offset;
  int address_increment = inner_loop_stride * stride;
  auto r_mean = mean[c_offset];
  auto factor = inv_std[c_offset];

  for (int i = 0; i < loop_count; i++) {
    float x_input[PARALLEL_LOADS];
    float x_grad_output[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      if (c_offset < stride && m_offset < reduction_size) {
        const bf16 g = relu_grad(grad_output[address_base], output[address_base]);
        if (masked) masked[address_base] = g;
        x_input[j] = __bfloat162float(input[address_base]);
        x_grad_output[j] = __bfloat162float(g);
      } else {
        x_input[j] = float(0);
        x_grad_output[j] = float(0);
      }
      m_offset += inner_loop_stride;
      address_base += address_increment;
    }
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      sum_dy[j] += x_grad_output[j];
      sum_dy_xmu[j] += x_grad_output[j] * (x_input[j] - r_mean);
    }
  }
#pragma unroll
  for (int j = 1; j < PARALLEL_LOADS; j++) {
    sum_dy[0] += sum_dy[j];
    sum_dy_xmu[0] += sum_dy_xmu[j];
  }
  auto sum_dy_th = sum_dy[0];
  auto sum_dy_xmu_th = sum_dy_xmu[0];

  __shared__ float shmem_sum_dy[kMaxBlock];
  __shared__ float shmem_sum_dy_xmu[kMaxBlock];
  merge_block_vertical_backward(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);

  if (gridDim.y > 1) {
    volatile float* staging_sum_dy = staging_data;
    volatile float* staging_sum_dy_xmu = &staging_data[stride * gridDim.y];
    address_base = c_offset + blockIdx.y * stride;
    if (threadIdx.y == 0 && c_offset < stride) {
      staging_sum_dy[address_base] = sum_dy_th;
      staging_sum_dy_xmu[address_base] = sum_dy_xmu_th;
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
      sum_dy_th = float(0.0);
      sum_dy_xmu_th = float(0.0);
      for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
        address_base = c_offset + y * stride;
        sum_dy_th += (c_offset < stride ? staging_sum_dy[address_base] : float(0.0));
        sum_dy_xmu_th += (c_offset < stride ? staging_sum_dy_xmu[address_base] : float(0.0));
      }
      merge_block_vertical_backward(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);
      if (threadIdx.y == 0 && c_offset < stride) {
        grad_bias[c_offset] = sum_dy_th;
        grad_weight[c_offset] = sum_dy_xmu_th * factor;
        sum_dy_o[c_offset] = sum_dy_th;
        sum_dy_xmu_o[c_offset] = sum_dy_xmu_th;
      }
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_offset < stride) {
      grad_bias[c_offset] = sum_dy_th;
      grad_weight[c_offset] = sum_dy_xmu_th * factor;
      sum_dy_o[c_offset] = sum_dy_th;
      sum_dy_xmu_o[c_offset] = sum_dy_xmu_th;
    }
  }
}

// dx (torch: batch_norm_backward_elemt_channels_last_kernel_impl) with g = relu_grad(dy, y) (MASKED false) or g
// read from the tensor the reduce kernel wrote (MASKED true).
template <int V, bool MASKED>
__global__ void __launch_bounds__(kEwThreads) k_bn_bwd_elemt(const bf16* __restrict__ grad_output, const bf16* __restrict__ output,
                                                             const bf16* __restrict__ input, bf16* __restrict__ grad_input,
                                                             const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                             const float* __restrict__ weight, const float* __restrict__ sum_dy,
                                                             const float* __restrict__ sum_dy_xmu, const float norm_fct,
                                                             const int reduction_size, const int stride) {
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
    const BVec<V> gv = *reinterpret_cast<const BVec<V>*>(grad_output + a);
    BVec<V> yv;
    if (!MASKED) yv = *reinterpret_cast<const BVec<V>*>(output + a);
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> dxv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const float g = __bfloat162float(MASKED ? gv.v[j] : relu_grad(gv.v[j], yv.v[j]));
      dxv.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(xv.v[j]) - m_c[j]) * factor_1_c[j]) * factor_2_c[j]);
    }
    *reinterpret_cast<BVec<V>*>(grad_input + a) = dxv;
  }
}

}  // namespace bn
}  // namespace b200c
