// Batch norm followed by ReLU6, SiLU or Hardswish over channels-last (NHWC) bf16 activations: torchvision's
// Conv2dNormActivation blocks (MobileNetV2 / V3, EfficientNet).  Training and eval sites, bit-identical to eager
// torch's batch norm followed by its activation module.
//
// Eager torch rounds the batch-norm output t to bf16, applies the activation in fp32 and rounds its output to bf16;
// the activation's backward reads the saved t and writes its input gradient g in bf16, which the batch-norm backward
// reads.  Here t is never stored: the forward computes t and writes act(t), and the backward reduce recomputes t from
// x and the saved statistics (the batch-norm backward reads x anyway), derives g from dy and t, and writes g for the
// batch-norm backward's elementwise kernel, bn::k_bn_bwd_elemt.  act_fwd and
// act_grad are torch 2.11's CUDA expressions as its sm_90 build compiles them (DESIGN.md section 10), so every kernel
// below, training and eval, rounds them alike.  The statistics are bn::k_bn_stats; the reduce keeps
// bn::k_bn_bwd_reduce's launch shape, row walk, block tree and grid merge, so its sums round as torch's do.
#pragma once
#include "norm_infer.cuh"
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_act {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;

// include/b200coll.h's b200c_act_t
enum Act { kActRelu6 = 1, kActSilu = 2, kActHardswish = 3 };

// torch's forward kernels: hardtanh(t, 0, 6) runs as clamp_scalar (a NaN t is returned as it is, bits included;
// anything else goes through fmaxf, fminf and a rounding that is exact); silu is
// t / (1 + expf(-t)) with the full-range expf and an IEEE division; hardswish is t * min(max(t + 3, 0), 6) * (1/6)
// with std::min / std::max (compare and select).
template <Act A>
__device__ __forceinline__ bf16 act_fwd(bf16 t) {
  const float v = __bfloat162float(t);
  if (A == kActRelu6) return isnan(v) ? t : __float2bfloat16(fminf(fmaxf(v, 0.f), 6.f));
  if (A == kActSilu) return __float2bfloat16(v / (1.f + expf(-v)));
  const float lo = v + 3.f < 0.f ? 0.f : v + 3.f;
  const float clamped = 6.f < lo ? 6.f : lo;
  return __float2bfloat16(v * clamped * (1.f / 6.f));
}

// torch's backward kernels, g of dy and the batch norm's bf16 output t: hardtanh_backward (t <= 0 || t >= 6 ? 0 : dy),
// silu_backward (dy * s * (1 + t * (1 - s)), s = 1 / (1 + expf(-t)), nvcc fusing t * (1 - s) + 1) and
// hardswish_backward (t <= -3 ? 0 : t < 3 ? dy * (t / 3 + 0.5) : dy, an IEEE division by 3).  A NaN t passes dy
// through ReLU6 and Hardswish.  Like torch, every result is rounded from fp32, dy included (F2FP, which also decides
// what a NaN dy becomes).
template <Act A>
__device__ __forceinline__ bf16 act_grad(bf16 dy, bf16 t) {
  const float v = __bfloat162float(t);
  const float d = __bfloat162float(dy);
  if (A == kActRelu6) return __float2bfloat16((v <= 0.f || v >= 6.f) ? 0.f : d);
  if (A == kActSilu) {
    const float s = 1.f / (1.f + expf(-v));
    return __float2bfloat16(d * s * (1.f + v * (1.f - s)));
  }
  return __float2bfloat16(v <= -3.f ? 0.f : v < 3.f ? d * (v / 3.f + 0.5f) : d);
}

// t = bf16(bn(x)), with k_bn_transform's expression
__device__ __forceinline__ bf16 bn_out(bf16 x, float mean, float inv_std, float w, float s) {
  return __float2bfloat16(w * (__bfloat162float(x) - mean) * inv_std + s);
}

// y = act(bf16(bn(x))) of a training site, from the statistics k_bn_stats saved.
template <int V, Act A>
__global__ void __launch_bounds__(kEwThreads) k_act_transform(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                              const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                              const float* __restrict__ weight, const float* __restrict__ shift,
                                                              const int reduction_size, const int stride) {
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
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = act_fwd<A>(bn_out(xv.v[j], m_c[j], inv_std_c[j], w_c[j], s_c[j]));
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

// Per-channel sums of g and g * (x - mean), and dweight / dbias, with g = act_grad(dy, t) and t recomputed from x:
// bn::k_bn_bwd_reduce<kGradDy, false>'s walk and merges, with g in place of dy.  Writes g to g_out, which
// bn::k_bn_bwd_elemt<V, kGradMasked, false, false> reads for dx.
template <Act A>
__global__ void k_act_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output, const float* __restrict__ mean,
                                 const float* __restrict__ inv_std, const float* __restrict__ weight, const float* __restrict__ shift,
                                 float* __restrict__ sum_dy_o, float* __restrict__ sum_dy_xmu_o, float* __restrict__ grad_weight,
                                 float* __restrict__ grad_bias, volatile float* staging_data, int* semaphores, bf16* __restrict__ g_out,
                                 const int reduction_size, const int stride) {
  constexpr int PARALLEL_LOADS = bn::kParallelLoads;
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
  const float w = weight[c_offset], s = shift[c_offset];

  for (int i = 0; i < loop_count; i++) {
    bf16 dy_v[PARALLEL_LOADS], x_v[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      if (m_offset + j * inner_loop_stride < reduction_size) {
        const int a = address_base + j * address_increment;
        dy_v[j] = grad_output[a];
        x_v[j] = input[a];
      }
    }
    float x_input[PARALLEL_LOADS];
    float x_grad_output[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      if (c_offset < stride && m_offset < reduction_size) {
        x_input[j] = __bfloat162float(x_v[j]);
        const bf16 g = act_grad<A>(dy_v[j], bn_out(x_v[j], r_mean, factor, w, s));
        g_out[address_base] = g;
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
      sum_dy_xmu[j] = __fmaf_rn(x_grad_output[j], x_input[j] - r_mean, sum_dy_xmu[j]);   // += g * (x - mean)
    }
  }
#pragma unroll
  for (int j = 1; j < PARALLEL_LOADS; j++) {
    sum_dy[0] += sum_dy[j];
    sum_dy_xmu[0] += sum_dy_xmu[j];
  }
  auto sum_dy_th = sum_dy[0];
  auto sum_dy_xmu_th = sum_dy_xmu[0];

  __shared__ float shmem_sum_dy[bn::kMaxBlock];
  __shared__ float shmem_sum_dy_xmu[bn::kMaxBlock];
  bn::merge_block_vertical_backward(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);

  auto write_sums = [&]() {
    grad_bias[c_offset] = sum_dy_th;
    grad_weight[c_offset] = sum_dy_xmu_th * factor;
    sum_dy_o[c_offset] = sum_dy_th;
    sum_dy_xmu_o[c_offset] = sum_dy_xmu_th;
  };
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
      bn::merge_block_vertical_backward(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);
      if (threadIdx.y == 0 && c_offset < stride) write_sums();
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_offset < stride) write_sums();
  }
}

// y = act(bf16(bn(x))) of an eval site: bn_infer::Channel's constants (running statistics, fp32 or bf16 parameters P),
// then the training transform's expression.
template <int V, Act A, typename P>
__global__ void __launch_bounds__(kEwThreads) k_act_infer(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                          const P* __restrict__ running_mean, const P* __restrict__ running_var,
                                                          const P* __restrict__ weight, const P* __restrict__ bias, const float eps,
                                                          const int reduction_size, const int stride) {
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
    const int a = m * stride + c0;
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = act_fwd<A>(bn_out(xv.v[j], m_c[j], inv_std_c[j], w_c[j], s_c[j]));
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

}  // namespace bn_act
}  // namespace b200c
