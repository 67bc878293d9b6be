// Eval-mode batch norm over channels-last (NHWC) bf16 activations, fused with what follows it in a ResNet: ReLU,
// `+= identity` then ReLU, `+=` a downsample branch's batch norm then ReLU, or (the stem) ReLU then max_pool2d(3, 2, 1).
//
// Eager torch runs an eval batch norm (batch_norm_cuda_out with train = false) as save_mean.copy_(running_mean),
// batch_norm_calc_invstd (invstd = rsqrt(float(running_var) + eps)) and batch_norm_elementwise (the channels-last
// transform w * (x - mean) * invstd + bias), and the ReLU, the residual add and the max-pool each as a pass of its own.
// Here each thread computes its channels' invstd with torch's expression and then applies the transform and the
// epilogue of the training kernels (norm_kernels.cuh), so one launch writes the site's output with eager torch's bits.
// Weight, bias and running statistics are fp32 or bf16 (P); bf16 ones are widened to fp32 as torch widens them.
// Nothing else is written: no mask, no running statistic, no num_batches_tracked.
#pragma once
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_infer {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;
using bn::PoolDims;
using bn::Tail;

__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(bf16 v) { return __bfloat162float(v); }

// One batch norm's per-channel constants: torch's save_mean (the running mean, widened), batch_norm_calc_invstd's
// rsqrt(var + eps) in fp32 (MUFU.RSQ, as torch's sm_90 build computes it), weight and bias.
template <typename P>
struct Channel {
  float mean, inv_std, w, s;
  __device__ __forceinline__ Channel(const P* __restrict__ running_mean, const P* __restrict__ running_var, const P* __restrict__ weight,
                                     const P* __restrict__ bias, const float eps, const int c)
      : mean(widen(running_mean[c])), inv_std(rsqrtf(widen(running_var[c]) + eps)), w(widen(weight[c])), s(widen(bias[c])) {}
};

// y = relu(bn(x)) (kTailRelu), relu(bf16(bn(x)) + identity) (kTailAddRelu) or relu(bf16(bn(x)) + bf16(bn2(identity)))
// (kTailBnAddRelu), rounded where eager torch rounds, as k_bn_transform computes them.  No kernel without a ReLU: every
// eval batch norm of a ResNet is one of these three sites or the stem.
template <int V, Tail TAIL, typename P>
__global__ void __launch_bounds__(kEwThreads) k_infer_transform(const bf16* __restrict__ input, const bf16* __restrict__ identity,
                                                                bf16* __restrict__ out, const P* __restrict__ running_mean,
                                                                const P* __restrict__ running_var, const P* __restrict__ weight,
                                                                const P* __restrict__ bias, const float eps,
                                                                const P* __restrict__ running_mean2, const P* __restrict__ running_var2,
                                                                const P* __restrict__ weight2, const P* __restrict__ bias2, const float eps2,
                                                                const int reduction_size, const int stride) {
  static_assert(TAIL == bn::kTailRelu || TAIL == bn::kTailAddRelu || TAIL == bn::kTailBnAddRelu, "an eval site ends in a ReLU");
  constexpr bool ADD = TAIL != bn::kTailRelu;
  constexpr bool BN2 = TAIL == bn::kTailBnAddRelu;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], inv_std_c[V], w_c[V], s_c[V], m2_c[V], inv_std2_c[V], w2_c[V], s2_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const Channel<P> k(running_mean, running_var, weight, bias, eps, c0 + j);
    m_c[j] = k.mean, inv_std_c[j] = k.inv_std, w_c[j] = k.w, s_c[j] = k.s;
    if (BN2) {
      const Channel<P> k2(running_mean2, running_var2, weight2, bias2, eps2, c0 + j);
      m2_c[j] = k2.mean, inv_std2_c[j] = k2.inv_std, w2_c[j] = k2.w, s2_c[j] = k2.s;
    }
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const int a = m * stride + c0;
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> zv;
    if (ADD) zv = *reinterpret_cast<const BVec<V>*>(identity + a);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      if (ADD) {
        if (BN2) zv.v[j] = __float2bfloat16(w2_c[j] * (__bfloat162float(zv.v[j]) - m2_c[j]) * inv_std2_c[j] + s2_c[j]);
        const bf16 r = __float2bfloat16(__bfloat162float(__float2bfloat16(tmp)) + __bfloat162float(zv.v[j]));
        yv.v[j] = __bfloat162float(r) <= 0.f ? __float2bfloat16(0.f) : r;
      } else {
        yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
      }
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
  }
}

// The stem: pooled = max over the 3 x 3 / stride 2 / padding 1 window of relu(bf16(bn(x))), selected as k_bn_pool_fwd
// selects it (rows first; a value greater than the maximum so far or NaN replaces it, so the first maximum wins a tie
// and the last NaN wins).  Only the pooled output is written: no argmax, and no int64 indices as torch's
// max_pool2d_with_indices writes.
template <int V, typename P>
__global__ void __launch_bounds__(kEwThreads) k_infer_pool(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                           const P* __restrict__ running_mean, const P* __restrict__ running_var,
                                                           const P* __restrict__ weight, const P* __restrict__ bias, const float eps,
                                                           const PoolDims d, const int pooled_rows, const int stride) {
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], inv_std_c[V], w_c[V], s_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const Channel<P> k(running_mean, running_var, weight, bias, eps, c0 + j);
    m_c[j] = k.mean, inv_std_c[j] = k.inv_std, w_c[j] = k.w, s_c[j] = k.s;
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int p = blockIdx.y * blockDim.y + threadIdx.y; p < pooled_rows; p += row_step) {
    const int pw = p % d.ow, ph = (p / d.ow) % d.oh, n = p / (d.ow * d.oh);
    float best[V];
#pragma unroll
    for (int j = 0; j < V; j++) best[j] = -INFINITY;
    for (int ih = max(2 * ph - 1, 0); ih < min(2 * ph + 2, d.h); ih++) {
      for (int iw = max(2 * pw - 1, 0); iw < min(2 * pw + 2, d.w); iw++) {
        const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + ((size_t)(n * d.h + ih) * d.w + iw) * stride + c0);
#pragma unroll
        for (int j = 0; j < V; j++) {
          const auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
          const float y = __bfloat162float(tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp));
          if (y > best[j] || isnan(y)) best[j] = y;
        }
      }
    }
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = __float2bfloat16(best[j]);
    *reinterpret_cast<BVec<V>*>(out + (size_t)p * stride + c0) = yv;
  }
}

}  // namespace bn_infer
}  // namespace b200c
