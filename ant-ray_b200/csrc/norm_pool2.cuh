// VGG-BN's stage end, max_pool2d(relu(bn(x)), kernel_size=2, stride=2), in training and eval, with only the pooled
// output written: relu(bn(x)) never exists.
//
// Shapes.  x is channels-last (NHWC) bf16, n images of h x w rows of C channels (m = n * h * w rows).  The pooled
// output y is n * oh * ow channels-last rows with oh = h / 2 and ow = w / 2 (floor mode: with odd h or w the last row or
// column of the input belongs to no window).  Window (ph, pw) covers input rows 2 * ph, 2 * ph + 1 and columns 2 * pw,
// 2 * pw + 1; an element's position in it is (ih & 1) * 2 + (iw & 1).
//
// Argmax.  One byte per pooled element: the position 0..3 of the element the window selected, or bn::kPoolNoGrad where
// the maximum is <= 0.  As at the stem, that byte stands in for the ReLU mask: a selected element holds its window's
// maximum, so its ReLU passes the gradient exactly when the maximum is not <= 0.
//
// Bits.  The statistics are bn::k_bn_stats.  Each element of relu(bn(x)) is computed as bn::k_bn_transform<V,
// kTailRelu> (training) and bn_infer::k_infer_transform<V, kTailRelu, P> (eval) compute it, and the window's maximum is
// selected as torch's channels-last max_pool2d selects it (rows first, then columns; a value greater than the maximum so
// far or NaN replaces it, so the first maximum wins a tie and the last NaN wins), as bn::k_bn_pool_fwd does.  A window
// of 2 with stride 2 never overlaps another, so the gradient g of an input element is the pooled gradient of its one
// window, taken as it is (a -0.0 stays -0.0), where that window selected it, and +0 otherwise.  The backward reduce is
// bn::k_bn_bwd_reduce's walk for [m][C] with torch's launch shape, per-thread row sequence, block tree and grid merge,
// with V = kBwdVec torch threads per hardware thread where the rows allow it, so every sum is torch's.  The backward
// elementwise kernel is bn::k_bn_bwd_elemt<V, kGradMasked, false, false>'s expression per element; both backward
// kernels rebuild g from the pooled gradient and the argmax bytes, so no full-size g is written.
#pragma once
#include "norm_infer.cuh"
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_pool2 {

using bn::bf16;
using bn::BVec;
using bn::kEwThreads;
using bn::kMaxBlock;
using bn::kParallelLoads;
using bn::kPoolNoGrad;

// n images of h x w input rows and their oh = h / 2 by ow = w / 2 pooled rows
struct Dims {
  int h, w, oh, ow;
};

// V bytes stored or loaded at once (the launcher picks V > 1 only with argmax on the 16-byte grid and C % 8 == 0)
template <int V>
struct alignas(V) Bytes {
  uint8_t v[V];
};

// The window maximum of relu(bf16(w * (x - mean) * inv_std + s)) for V channels of pooled row p, and each channel's
// position (or kPoolNoGrad) in `pos`.
template <int V>
__device__ __forceinline__ void window_max(const bf16* __restrict__ input, const Dims& d, const int p, const int c0, const int stride,
                                           const float (&m_c)[V], const float (&inv_std_c)[V], const float (&w_c)[V],
                                           const float (&s_c)[V], float (&best)[V], uint8_t (&pos)[V]) {
  const int pw = p % d.ow, ph = (p / d.ow) % d.oh, n = p / (d.ow * d.oh);
  const size_t row0 = ((size_t)(n * d.h + 2 * ph) * d.w + 2 * pw) * stride + c0;
  // the four rows are loaded together, none waiting for another's compare
  const size_t offs[4] = {0, (size_t)stride, (size_t)d.w * stride, (size_t)(d.w + 1) * stride};
  BVec<V> xv[4];
#pragma unroll
  for (int k = 0; k < 4; k++) xv[k] = *reinterpret_cast<const BVec<V>*>(input + row0 + offs[k]);
#pragma unroll
  for (int j = 0; j < V; j++) {
    best[j] = -INFINITY;
    pos[j] = 0;
  }
#pragma unroll
  for (int k = 0; k < 4; k++) {
#pragma unroll
    for (int j = 0; j < V; j++) {
      const auto tmp = w_c[j] * (__bfloat162float(xv[k].v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      const float y = __bfloat162float(tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp));
      if (y > best[j] || isnan(y)) {
        best[j] = y;
        pos[j] = k;
      }
    }
  }
#pragma unroll
  for (int j = 0; j < V; j++)
    if (best[j] <= 0.f) pos[j] = kPoolNoGrad;
}

// Training: the pooled rows and their argmax bytes from x and the saved statistics.  One thread per pooled row and V
// channels, launched as the elementwise kernels are over the pooled rows.
template <int V>
__global__ void __launch_bounds__(kEwThreads) k_pool2_fwd(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                          uint8_t* __restrict__ argmax, const float* __restrict__ mean,
                                                          const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                          const float* __restrict__ shift, const Dims d, const int pooled_rows,
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
  for (int p = blockIdx.y * blockDim.y + threadIdx.y; p < pooled_rows; p += row_step) {
    float best[V];
    Bytes<V> av;
    window_max<V>(input, d, p, c0, stride, m_c, inv_std_c, w_c, s_c, best, av.v);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = __float2bfloat16(best[j]);
    const size_t a = (size_t)p * stride + c0;
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
    *reinterpret_cast<Bytes<V>*>(argmax + a) = av;
  }
}

// Eval: the pooled rows alone, from the running statistics.  Launched as k_pool2_fwd.
template <int V, typename P>
__global__ void __launch_bounds__(kEwThreads) k_pool2_infer(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                            const P* __restrict__ running_mean, const P* __restrict__ running_var,
                                                            const P* __restrict__ weight, const P* __restrict__ bias, const float eps,
                                                            const Dims d, const int pooled_rows, const int stride) {
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], inv_std_c[V], w_c[V], s_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    const bn_infer::Channel<P> k(running_mean, running_var, weight, bias, eps, c0 + j);
    m_c[j] = k.mean, inv_std_c[j] = k.inv_std, w_c[j] = k.w, s_c[j] = k.s;
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int p = blockIdx.y * blockDim.y + threadIdx.y; p < pooled_rows; p += row_step) {
    float best[V];
    uint8_t pos[V];
    window_max<V>(input, d, p, c0, stride, m_c, inv_std_c, w_c, s_c, best, pos);
    BVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = __float2bfloat16(best[j]);
    *reinterpret_cast<BVec<V>*>(out + (size_t)p * stride + c0) = yv;
  }
}

// Where input row m's gradient comes from: the offset of its window's pooled element (channel 0) and its position in
// that window, or a negative offset for a row in no window (the last row or column of an odd h or w).
struct Source {
  int offset;   // (pooled row) * stride, or -1
  int at;
};
__device__ __forceinline__ Source source(const Dims& d, const int m, const int stride) {
  const int iw = m % d.w, ih = (m / d.w) % d.h, n = m / (d.w * d.h);
  const int ph = ih >> 1, pw = iw >> 1;
  if (ph >= d.oh || pw >= d.ow) return Source{-1, 0};
  return Source{((n * d.oh + ph) * d.ow + pw) * stride, (ih & 1) * 2 + (iw & 1)};
}

// g of V channels from the pooled gradient and argmax bytes of the row's window: the gradient as it is where the window
// selected this position, else +0
template <int V>
__device__ __forceinline__ void pool2_grad(const BVec<V>& dyv, const Bytes<V>& av, const int at, BVec<V>& g) {
#pragma unroll
  for (int k = 0; k < V; k++) g.v[k] = av.v[k] == at ? dyv.v[k] : __float2bfloat16(0.f);
}

// Per-channel sums of g and g * (x - mean) over [m][C] (torch: batch_norm_backward_reduce_channels_last_kernel<4>), and
// dweight / dbias, as bn::k_bn_bwd_reduce computes them: V adjacent torch threads per hardware thread (block.x is
// reduce_config's divided by V), each iteration's kParallelLoads rows loaded before the first sum uses one.
template <int V>
__global__ void __launch_bounds__(kMaxBlock) k_pool2_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output,
                                                                const uint8_t* __restrict__ argmax, const float* __restrict__ mean,
                                                                const float* __restrict__ inv_std, float* __restrict__ sum_dy_o,
                                                                float* __restrict__ sum_dy_xmu_o, float* __restrict__ grad_weight,
                                                                float* __restrict__ grad_bias, volatile float* staging_data,
                                                                int* semaphores, const Dims d, const int reduction_size,
                                                                const int stride) {
  constexpr int PARALLEL_LOADS = kParallelLoads;
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
  const int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  const int c_offset = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c_offset >= stride || m_offset >= reduction_size) return;

  const int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  float r_mean[V];
#pragma unroll
  for (int k = 0; k < V; k++) r_mean[k] = mean[c_offset + k];

  for (int i = 0; i < loop_count; i++) {
    // all rows of the iteration are loaded before any sum uses one
    BVec<V> g_v[PARALLEL_LOADS], x_v[PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      const int m = m_offset + j * inner_loop_stride;
      if (m < reduction_size) {
        x_v[j] = *reinterpret_cast<const BVec<V>*>(input + ((size_t)m * stride + c_offset));
        const Source src = source(d, m, stride);
        if (src.offset >= 0) {
          const Bytes<V> av = *reinterpret_cast<const Bytes<V>*>(argmax + src.offset + c_offset);
          const BVec<V> dyv = *reinterpret_cast<const BVec<V>*>(grad_output + src.offset + c_offset);
          pool2_grad<V>(dyv, av, src.at, g_v[j]);
        } else {
#pragma unroll
          for (int k = 0; k < V; k++) g_v[j].v[k] = __float2bfloat16(0.f);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      float x_input[V], x_grad_output[V];
#pragma unroll
      for (int k = 0; k < V; k++) {
        x_input[k] = m_offset < reduction_size ? __bfloat162float(x_v[j].v[k]) : float(0);
        x_grad_output[k] = m_offset < reduction_size ? __bfloat162float(g_v[j].v[k]) : float(0);
      }
      m_offset += inner_loop_stride;
#pragma unroll
      for (int k = 0; k < V; k++) {
        sum_dy[j][k] += x_grad_output[k];
        sum_dy_xmu[j][k] = __fmaf_rn(x_grad_output[k], x_input[k] - r_mean[k], sum_dy_xmu[j][k]);   // += g * (x - mean)
      }
    }
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
      grad_weight[c] = sum_dy_xmu_th[k] * inv_std[c];
      sum_dy_o[c] = sum_dy_th[k];
      sum_dy_xmu_o[c] = sum_dy_xmu_th[k];
    }
  };
  if (gridDim.y > 1) {
    volatile float* staging_sum_dy = staging_data;
    volatile float* staging_sum_dy_xmu = &staging_data[stride * gridDim.y];
    if (threadIdx.y == 0) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        staging_sum_dy[c_offset + k + blockIdx.y * stride] = sum_dy_th[k];
        staging_sum_dy_xmu[c_offset + k + blockIdx.y * stride] = sum_dy_xmu_th[k];
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
#pragma unroll
        for (int k = 0; k < V; k++) {
          sum_dy_th[k] += staging_sum_dy[c_offset + k + y * stride];
          sum_dy_xmu_th[k] += staging_sum_dy_xmu[c_offset + k + y * stride];
        }
      }
      bn::merge_block_vertical_backward<V>(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);
      if (threadIdx.y == 0) write_sums();
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0) write_sums();
  }
}

// dx (torch: batch_norm_backward_elemt_channels_last_kernel_impl) with g rebuilt from the pooled gradient and the argmax
// bytes, and this call's norm_fct = 1 / m passed by value, as a local site's bn::k_bn_bwd_elemt takes it.  ew_config's
// launch for [m][C].
template <int V>
__global__ void __launch_bounds__(kEwThreads) k_pool2_bwd_elemt(const bf16* __restrict__ grad_output, const uint8_t* __restrict__ argmax,
                                                                const bf16* __restrict__ input, bf16* __restrict__ grad_input,
                                                                const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                                const float* __restrict__ weight, const float* __restrict__ sum_dy,
                                                                const float* __restrict__ sum_dy_xmu, const float norm_fct, const Dims d,
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
    const size_t a = (size_t)m * stride + c0;
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    const Source src = source(d, m, stride);
    BVec<V> gv;
    if (src.offset >= 0) {
      const Bytes<V> av = *reinterpret_cast<const Bytes<V>*>(argmax + src.offset + c0);
      const BVec<V> dyv = *reinterpret_cast<const BVec<V>*>(grad_output + src.offset + c0);
      pool2_grad<V>(dyv, av, src.at, gv);
    } else {
#pragma unroll
      for (int j = 0; j < V; j++) gv.v[j] = __float2bfloat16(0.f);
    }
    BVec<V> dxv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const float g = __bfloat162float(gv.v[j]);
      dxv.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(xv.v[j]) - m_c[j]) * factor_1_c[j]) * factor_2_c[j]);
    }
    *reinterpret_cast<BVec<V>*>(grad_input + a) = dxv;
  }
}

}  // namespace bn_pool2
}  // namespace b200c
