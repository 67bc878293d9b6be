// Batch norm whose output goes to a residual add, optionally through stochastic depth, over channels-last (NHWC) bf16
// activations: the projection batch norm that ends MobileNetV2 / V3 and EfficientNet inverted-residual blocks.
// Training and eval sites, bit-identical to eager torch's batch norm followed by `x + f` or `f += x`, and in
// EfficientNet by torchvision's stochastic_depth(f, p, "row") before the add.
//
// Eager torch rounds the batch-norm output t to bf16.  Stochastic depth multiplies it by a bf16 noise value per sample
// (0 or the survival rate's reciprocal, built by torch's own bernoulli_ and div_) and rounds to bf16; the add sums in
// fp32 and rounds to bf16.  Backward: the add hands dy to both operands, stochastic depth's mul writes
// g = bf16(dy * noise[n]), and the batch-norm backward reads g.  Here the forward writes only the sum, and the backward
// reduce derives g from dy and the noise and writes it for bn::k_bn_bwd_elemt.  A site without stochastic depth has
// g = dy and runs bn::k_bn_bwd_reduce<kGradDy, false> on dy itself, so it needs no kernel here.  The statistics are
// bn::k_bn_stats; the reduce keeps bn::k_bn_bwd_reduce's launch shape, row walk, block tree and grid merge, so its sums
// round as torch's do.
#pragma once
#include "norm_act.cuh"
#include "norm_infer.cuh"
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_res {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;

// What follows the batch norm: nothing (kResPlain, eval only: the training forward is k_bn_transform<V, kTailNone>),
// `+ identity` (kResAdd) or stochastic depth and then `+ identity` (kResDropAdd, training only).
enum Res { kResPlain, kResAdd, kResDropAdd };

// y = bf16(t + identity) or, with the noise, bf16(bf16(t * noise) + identity), each operand widened from bf16
__device__ __forceinline__ bf16 res_add(bf16 t, bf16 z) { return __float2bfloat16(__bfloat162float(t) + __bfloat162float(z)); }
__device__ __forceinline__ bf16 drop(bf16 t, float noise) { return __float2bfloat16(__bfloat162float(t) * noise); }

// y of a training site, from the statistics k_bn_stats saved: t = bf16(bn(x)) as k_bn_transform computes it, then the
// epilogue.  kResDropAdd reads noise[m / rows_per_sample], row m being in sample m / (H * W).
template <int V, Res R>
__global__ void __launch_bounds__(kEwThreads) k_res_transform(const bf16* __restrict__ input, const bf16* __restrict__ identity,
                                                              const bf16* __restrict__ noise, bf16* __restrict__ out,
                                                              const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                              const float* __restrict__ weight, const float* __restrict__ shift,
                                                              const int rows_per_sample, const int reduction_size, const int stride) {
  static_assert(R == kResAdd || R == kResDropAdd, "a plain training site runs k_bn_transform<V, kTailNone>");
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
    const BVec<V> zv = *reinterpret_cast<const BVec<V>*>(identity + a);
    const float nz = R == kResDropAdd ? __bfloat162float(noise[m / rows_per_sample]) : 0.f;
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const bf16 t = bn_act::bn_out(xv.v[j], m_c[j], inv_std_c[j], w_c[j], s_c[j]);
      yv.v[j] = res_add(R == kResDropAdd ? drop(t, nz) : t, zv.v[j]);
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

// Per-channel sums of g and g * (x - mean), and dweight / dbias, with g = bf16(dy * noise[m / rows_per_sample]):
// bn::k_bn_bwd_reduce<kGradDy, false>'s walk and merges, with g in place of dy.  Writes g to g_out, which
// bn::k_bn_bwd_elemt<V, kGradMasked, false, false> reads for dx.  A dropped sample's g is dy * 0: +-0, or NaN where dy
// is +-Inf or NaN, as torch's mul gives.
__global__ void k_res_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output, const bf16* __restrict__ noise,
                                 const float* __restrict__ mean, const float* __restrict__ inv_std, float* __restrict__ sum_dy_o,
                                 float* __restrict__ sum_dy_xmu_o, float* __restrict__ grad_weight, float* __restrict__ grad_bias,
                                 volatile float* staging_data, int* semaphores, bf16* __restrict__ g_out, const int rows_per_sample,
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

  for (int i = 0; i < loop_count; i++) {
    bf16 dy_v[PARALLEL_LOADS], x_v[PARALLEL_LOADS], n_v[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      const int row = m_offset + j * inner_loop_stride;
      if (row < reduction_size) {
        const int a = address_base + j * address_increment;
        dy_v[j] = grad_output[a];
        x_v[j] = input[a];
        n_v[j] = noise[row / rows_per_sample];
      }
    }
    float x_input[PARALLEL_LOADS];
    float x_grad_output[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      if (c_offset < stride && m_offset < reduction_size) {
        x_input[j] = __bfloat162float(x_v[j]);
        const bf16 g = drop(dy_v[j], __bfloat162float(n_v[j]));
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

// y of an eval site: bn_infer::Channel's constants (running statistics, fp32 or bf16 parameters P), t as the training
// transform computes it, then nothing (kResPlain) or `+ identity` (kResAdd).  Stochastic depth is the identity in eval.
template <int V, Res R, typename P>
__global__ void __launch_bounds__(kEwThreads) k_res_infer(const bf16* __restrict__ input, const bf16* __restrict__ identity,
                                                          bf16* __restrict__ out, const P* __restrict__ running_mean,
                                                          const P* __restrict__ running_var, const P* __restrict__ weight,
                                                          const P* __restrict__ bias, const float eps, const int reduction_size,
                                                          const int stride) {
  static_assert(R == kResPlain || R == kResAdd, "stochastic depth is the identity in eval");
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
    BVec<V> zv;
    if (R == kResAdd) zv = *reinterpret_cast<const BVec<V>*>(identity + a);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const bf16 t = bn_act::bn_out(xv.v[j], m_c[j], inv_std_c[j], w_c[j], s_c[j]);
      yv.v[j] = R == kResAdd ? res_add(t, zv.v[j]) : t;
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

}  // namespace bn_res
}  // namespace b200c
