// Squeeze-and-excitation over channels-last (NHWC) bf16 activations: torchvision's SqueezeExcitation without its
// squeeze path (fc1, activation, fc2, scale activation run on torch), bit-identical to eager torch.
//
// For x of [N, C, H, W] (HW = H * W rows of C channels per sample) eager torch runs:
//   pooled = x.mean((-1, -2))            pooled[n, c] = bf16(sum_hw float(x) * factor), factor = float(N*C) / (N*C*HW)
//   y      = s * x                       y = bf16(float(s[n, c]) * float(x))
//   ds     = sum_to(dy * x, s.shape)     ds[n, c] = bf16(sum_hw float(bf16(float(dy) * float(x)))); with HW = 1 the
//                                        product itself (sum_to reduces nothing, so a -0.0 stays -0.0)
//   dx     = dy * s  +  gp / HW          dx = bf16(float(bf16(float(dy) * float(s))) + float(bf16(float(gp) * (1 / HW))))
// The two sums run in Reduce.cuh's gpu_reduce_kernel, "vectorize along output" (C is the fastest output dimension,
// HW one reduced dimension of stride C).  k_se_pool and k_se_bwd_reduce keep that kernel's launch shape and per-output
// order: output_vec_size V adjacent channels per thread, vt0 = 4 accumulators per channel walking the rows with stride
// step_input and combined 0 + 1 + 2 + 3, then block_y_reduce's tree over threadIdx.y when the rows are split across
// warps, then, with ctas_per_output > 1, global_reduce: staging, a semaphore per blockIdx.x, and the last block's walk
// over the staged rows followed by the same tree.  The host (inst_se.cu) restates setReduceConfig for the launch.
// The elementwise kernels are free in layout.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200c {
namespace se {

typedef __nv_bfloat16 bf16;

template <int V>
struct alignas(2 * V) SVec {
  bf16 v[V];
};

constexpr int kVt0 = 4;              // Reduce.cuh's vt0: accumulators per output
constexpr int kMaxThreads = 512;     // mnt_wrapper<float>::MAX_NUM_THREADS
constexpr int kEwThreads = 256;
constexpr int kEwVec = 8;            // 16 bytes of channels per thread in the elementwise kernels' vector form
// Semaphores sit at the start of the scratch buffer, one per blockIdx.x of a split reduction, and are left at zero;
// a split reduction has at most num_mp * maxThreadsPerMultiProcessor / 128 blocks in x (its block has at least 128
// threads), which this bounds for up to 256 SMs of 2048 threads.
constexpr int kSemaphores = 4096;

__device__ __forceinline__ float f(bf16 v) { return __bfloat162float(v); }

// The launch of a reducing kernel, as setReduceConfig leaves it for V = output_vec_size.
struct ReduceShape {
  int num_outputs;   // N * C
  int c;             // channels: the input stride of one row
  int hw;            // rows per sample (inputs_per_output)
  int split;         // input_mult[BLOCK_Y] != 0: the rows are split across threadIdx.y (block_y_reduce)
  int ctas;          // ctas_per_output (gridDim.y); > 1 only when split
};

// Loads V channels of row `row` of output `o`'s sample: x itself (pool) or bf16(dy * x) (backward reduce).  kAligned:
// one vector load per operand; otherwise V scalar loads (an operand off the 2V-byte grid).
template <int V, bool kProduct, bool kAligned>
__device__ __forceinline__ void load_rows(const bf16* __restrict__ a, const bf16* __restrict__ b, long long off, float* out) {
  bf16 va[V], vb[V];
  if (kAligned) {
    const SVec<V> ta = *reinterpret_cast<const SVec<V>*>(a + off);
#pragma unroll
    for (int j = 0; j < V; j++) va[j] = ta.v[j];
    if (kProduct) {
      const SVec<V> tb = *reinterpret_cast<const SVec<V>*>(b + off);
#pragma unroll
      for (int j = 0; j < V; j++) vb[j] = tb.v[j];
    }
  } else {
#pragma unroll
    for (int j = 0; j < V; j++) {
      va[j] = a[off + j];
      if (kProduct) vb[j] = b[off + j];
    }
  }
#pragma unroll
  for (int j = 0; j < V; j++) out[j] = kProduct ? f(__float2bfloat16(f(va[j]) * f(vb[j]))) : f(va[j]);
}

// block_y_reduce: shared[tx + ty * bw] holds each thread's V values; halving offsets over threadIdx.y.
template <int V>
__device__ __forceinline__ void block_y_reduce(float (&value)[V], float* shared) {
  const int base = (threadIdx.x + threadIdx.y * blockDim.x) * V;
#pragma unroll
  for (int j = 0; j < V; j++) shared[base + j] = value[j];
  for (int offset = blockDim.y / 2; offset > 0; offset >>= 1) {
    __syncthreads();
    if (threadIdx.y < offset && threadIdx.y + offset < blockDim.y) {
      const int other = base + offset * blockDim.x * V;
#pragma unroll
      for (int j = 0; j < V; j++) value[j] += shared[other + j];
#pragma unroll
      for (int j = 0; j < V; j++) shared[base + j] = value[j];
    }
  }
}

// gpu_reduce_kernel's run<V>() for this geometry, writing bf16(sum * scale) (MeanOps' project, scale = factor) or
// bf16(sum) (the sum functor, kProduct).  Outputs are [N][C], output index n * C + c.
template <int V, bool kProduct, bool kAligned>
__device__ __forceinline__ void reduce_run(const bf16* __restrict__ a, const bf16* __restrict__ b, bf16* __restrict__ out, float scale,
                                           const ReduceShape& r, volatile float* staging, int* semaphores) {
  __shared__ float shared[kMaxThreads];   // num_threads * V <= 512 floats
  const int bw = blockDim.x, bh = blockDim.y;
  // output_mult = {1, split ? 0 : bw}, step_output = split ? bw : bw * bh; input_mult = {0, split, split ? bh : 0}
  const int step_output = r.split ? bw : bw * bh;
  const int output_idx = (threadIdx.x + (r.split ? 0 : threadIdx.y * bw) + blockIdx.x * step_output) * V;
  const int input_idx = r.split ? threadIdx.y + blockIdx.y * bh : 0;
  const int step_input = r.split ? bh * r.ctas : 1;

  float value[V];
#pragma unroll
  for (int j = 0; j < V; j++) value[j] = 0.f;
  if (output_idx < r.num_outputs && input_idx < r.hw) {
    const int n = output_idx / r.c;
    const long long base = (long long)n * r.hw * r.c + (output_idx - n * r.c);
    // thread_reduce_impl<V>: vt0 accumulators, full groups of vt0 rows, then the tail, then the combine
    float acc[kVt0][V];
#pragma unroll
    for (int i = 0; i < kVt0; i++)
#pragma unroll
      for (int j = 0; j < V; j++) acc[i][j] = 0.f;
    int idx = input_idx;
    const int end = r.hw;
    while (idx + (kVt0 - 1) * step_input < end) {
      float vals[kVt0][V];
#pragma unroll
      for (int i = 0; i < kVt0; i++) load_rows<V, kProduct, kAligned>(a, b, base + (long long)(idx + i * step_input) * r.c, vals[i]);
#pragma unroll
      for (int i = 0; i < kVt0; i++)
#pragma unroll
        for (int j = 0; j < V; j++) acc[i][j] += vals[i][j];
      idx += step_input * kVt0;
    }
#pragma unroll
    for (int i = 0; i < kVt0; i++) {
      if (idx >= end) break;
      float vals[V];
      load_rows<V, kProduct, kAligned>(a, b, base + (long long)idx * r.c, vals);
#pragma unroll
      for (int j = 0; j < V; j++) acc[i][j] += vals[j];
      idx += step_input;
    }
#pragma unroll
    for (int i = 1; i < kVt0; i++)
#pragma unroll
      for (int j = 0; j < V; j++) acc[0][j] += acc[i][j];
#pragma unroll
    for (int j = 0; j < V; j++) value[j] = acc[0][j];
  }
  if (r.split) block_y_reduce<V>(value, shared);

  const bool should_store = output_idx < r.num_outputs && (!r.split || threadIdx.y == 0);
  if (r.ctas > 1) {
    // global_reduce: staging_memory_offset(cta2) = tx + (cta2 + bx * gridDim.y) * bw, V floats per slot
    if (should_store) {
      const int slot = (threadIdx.x + (blockIdx.y + blockIdx.x * gridDim.y) * bw) * V;
#pragma unroll
      for (int j = 0; j < V; j++) staging[slot + j] = value[j];
    }
    __threadfence();
    __syncthreads();
    __shared__ bool is_last_block_done;
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
      const int prev = atomicAdd(&semaphores[blockIdx.x], 1);
      is_last_block_done = prev == gridDim.y - 1;
      if (is_last_block_done) semaphores[blockIdx.x] = 0;   // leave the scratch as it was found
    }
    __syncthreads();
    if (!is_last_block_done) return;
    __threadfence();
#pragma unroll
    for (int j = 0; j < V; j++) value[j] = 0.f;
    if (output_idx < r.num_outputs) {
      for (int cta = threadIdx.y; cta < r.ctas; cta += bh) {
        const int slot = (threadIdx.x + (cta + blockIdx.x * gridDim.y) * bw) * V;
#pragma unroll
        for (int j = 0; j < V; j++) value[j] += staging[slot + j];
      }
    }
    block_y_reduce<V>(value, shared);
  }
  // One bf16 store per output, as set_results_to_output stores them: V follows the inputs, so `out` may sit anywhere on
  // the 2-byte grid.
  if (should_store) {
#pragma unroll
    for (int j = 0; j < V; j++) out[output_idx + j] = __float2bfloat16(kProduct ? value[j] : value[j] * scale);
  }
}

// pooled = x.mean((-1, -2)): V is torch's output_vec_size, which x's address allows, so x is always read in vectors.
template <int V>
__global__ void __launch_bounds__(kMaxThreads) k_se_pool(const bf16* __restrict__ x, bf16* __restrict__ pooled, float factor, ReduceShape r,
                                                         float* staging, int* semaphores) {
  reduce_run<V, false, true>(x, nullptr, pooled, factor, r, staging, semaphores);
}

// ds = sum_hw(bf16(dy * x)): V is the output_vec_size of the aligned product tensor torch reduces, so dy and x are read
// in vectors only where both sit on the 2V-byte grid (kAligned).
template <int V, bool kAligned>
__global__ void __launch_bounds__(kMaxThreads) k_se_bwd_reduce(const bf16* __restrict__ dy, const bf16* __restrict__ x, bf16* __restrict__ ds,
                                                               ReduceShape r, float* staging, int* semaphores) {
  if (r.hw == 1) {
    // s and x have one shape, so sum_to hands back the product itself: store it (0 + p would turn a -0.0 into +0.0).
    // One row: no split, one block per output column, so no thread of the block waits at a barrier.
    const int o = (threadIdx.x + threadIdx.y * blockDim.x + blockIdx.x * blockDim.x * blockDim.y) * V;
    if (o < r.num_outputs) {
      float p[V];
      load_rows<V, true, kAligned>(dy, x, o, p);
#pragma unroll
      for (int j = 0; j < V; j++) ds[o + j] = __float2bfloat16(p[j]);
    }
    return;
  }
  reduce_run<V, true, kAligned>(dy, x, ds, 1.f, r, staging, semaphores);
}

// Rows m = n * HW + hw of C channels; thread (x, y) of block (bx, by) owns V channels and strides over the rows.
#define SE_EW_LOOP                                                                  \
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;                       \
  if (c0 >= c) return;                                                              \
  const int row_step = blockDim.y * gridDim.y;                                      \
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < rows; m += row_step)

// y = bf16(float(s[n, c]) * float(x))
template <int V>
__global__ void __launch_bounds__(kEwThreads) k_se_scale(const bf16* __restrict__ x, const bf16* __restrict__ s, bf16* __restrict__ y,
                                                         const int rows, const int c, const int hw) {
  SE_EW_LOOP {
    const long long a = (long long)m * c + c0;
    const int sc = (m / hw) * c + c0;
    const SVec<V> xv = *reinterpret_cast<const SVec<V>*>(x + a);
    const SVec<V> sv = *reinterpret_cast<const SVec<V>*>(s + sc);
    SVec<V> yv;
#pragma unroll
    for (int j = 0; j < V; j++) yv.v[j] = __float2bfloat16(f(sv.v[j]) * f(xv.v[j]));
    *reinterpret_cast<SVec<V>*>(y + a) = yv;
  }
}

// dx = bf16(float(bf16(float(dy) * float(s))) + float(bf16(float(gp) * inv_hw))): the scale's gradient of x plus the
// mean's, added as autograd adds them.
template <int V>
__global__ void __launch_bounds__(kEwThreads) k_se_bwd_elemt(const bf16* __restrict__ dy, const bf16* __restrict__ s, const bf16* __restrict__ gp,
                                                             bf16* __restrict__ dx, const float inv_hw, const int rows, const int c,
                                                             const int hw) {
  SE_EW_LOOP {
    const long long a = (long long)m * c + c0;
    const int sc = (m / hw) * c + c0;
    const SVec<V> dv = *reinterpret_cast<const SVec<V>*>(dy + a);
    const SVec<V> sv = *reinterpret_cast<const SVec<V>*>(s + sc);
    const SVec<V> gv = *reinterpret_cast<const SVec<V>*>(gp + sc);
    SVec<V> xv;
#pragma unroll
    for (int j = 0; j < V; j++) {
      const bf16 t = __float2bfloat16(f(dv.v[j]) * f(sv.v[j]));
      const bf16 g = __float2bfloat16(f(gv.v[j]) * inv_hw);
      xv.v[j] = __float2bfloat16(f(t) + f(g));
    }
    *reinterpret_cast<SVec<V>*>(dx + a) = xv;
  }
}
#undef SE_EW_LOOP

}  // namespace se
}  // namespace b200c
