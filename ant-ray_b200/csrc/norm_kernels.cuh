// Training-mode batch norm over channels-last (NHWC) bf16 activations with fp32 weight, bias and statistics,
// fused with what follows it in a ResNet block: ReLU, or `+= identity` then ReLU.
//
// The statistics and backward-reduce kernels are ports of the channels-last kernels of PyTorch's
// aten/src/ATen/native/cuda/Normalization.cuh (PyTorch, BSD-3-Clause licence, Copyright (c) 2016- Facebook, Inc.
// and its contributors; the kernels originate in NVIDIA Apex).  They keep torch's launch shape, per-thread
// sequence of rows, block tree and grid merge, and torch's expressions, so that every per-channel sum is rounded
// exactly as torch rounds it.  That is what makes the outputs bit-identical to eager torch (torch 2.x runs bf16
// batch norm on these native kernels, not on cuDNN).  Within those constraints the reducing kernels carry 4 channels
// per thread where C % 8 == 0 and keep several iterations of rows in flight through per-thread cp.async rings.  The elementwise
// kernels (transform, backward elementwise) have no cross-element rounding, so they are restructured freely: 16-byte
// loads of 8 channels per thread.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

namespace b200c {
namespace bn {

// torch's constants (MAX_BLOCK_SIZE, ELEMENTS_PER_ITER, ELEMENTS_PER_THREAD, OPTIMAL_TILE_W, MAX_H_BLOCK): the
// reduction order depends on them.
constexpr int kMaxBlock = 512;
constexpr int kParallelLoads = 4;
constexpr int kElemsPerThread = 16;
constexpr int kTileW = 32;
constexpr int kMaxHBlock = 128;
// statistics kernel: channels per hardware thread on its vector path (8-byte loads).  Measured on H100 against 1, 2
// and 8 (DESIGN.md section 7).
constexpr int kStatsVec = 4;
// backward reduce: channels per hardware thread on its vector path (8-byte copies)
constexpr int kBwdVec = 4;
// The vector paths' ring depth, in iterations of kParallelLoads rows, measured on H100 against 6 and 8 for the
// statistics and 4 for the backward (DESIGN.md section 7).  A backward ring of 3 or more operands keeps 2 stages: at
// 3 stages a tail's ring (dy, dy2, x) took 36 KB per block and ran slower than torch's register walk.  Every ring
// and its kernel's static shared memory stay within the 48 KB a block gets without an opt-in, so every launch is
// valid whether or not the context has set any function attribute.
constexpr int kStatsStages = 4;
constexpr unsigned kBwdStages = 3;       // a backward ring of dy and x
constexpr unsigned kBwdStagesWide = 2;   // one of 3 or more operands (a tail's dy2, y, a downsample branch's x2)
__host__ __device__ constexpr unsigned bwd_ring_stages(int ops) { return ops >= 3 ? kBwdStagesWide : kBwdStages; }
// operands of the backward reduce's ring: dy, x, and dy2, y, x2 where the site has them
__host__ __device__ constexpr int bwd_ring_operands(bool y, bool dy2, bool dual) { return 2 + dy2 + y + dual; }
// elementwise kernels
constexpr int kEwThreads = 256;
constexpr int kEwVec = 8;

typedef __nv_bfloat16 bf16;

template <int V>
struct alignas(2 * V) BVec {
  bf16 v[V];
};

// ---- the vector paths' row rings ----
// A thread copies its own rows with cp.async into its own slots of a ring in dynamic shared memory, one commit
// group per iteration of kParallelLoads rows, and reads back only what it copied itself: cp.async.wait_group alone
// makes a slot visible to its thread, so the row walk has no barrier.  Slots are laid out [stage][operand][row j]
// [thread] in words of one thread's V channels, so that consecutive threads touch consecutive words.
__device__ __forceinline__ unsigned char* ring_smem() {
  extern __shared__ __align__(16) unsigned char bn_ring[];
  return bn_ring;
}
template <int BYTES>
__device__ __forceinline__ void cp_async(void* smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem), "n"(BYTES)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// ---- reduction helpers (torch's, per channel) ----
// The statistics kernel runs V adjacent torch threads in one hardware thread: hardware thread (tx, ty) of a block
// blockDim.x wide holds torch's threads (tx * V + k, ty), k < V, of a block blockDim.x * V wide, i.e. channels
// c .. c + V - 1.  Every per-channel value is computed by torch's expression in torch's order; V only changes how
// many channels one instruction stream carries.

// torch's welford_merge_element, with its roundings spelled out.  nvcc contracts `mean_new * count_new + mean *
// count` into one FMA on either product, and which one depends on the call site: in torch's statistics kernel the
// merge of a thread's accumulators fuses mean_new * count_new (FUSE_NEW), every other merge fuses mean * count.
template <bool FUSE_NEW>
__device__ __forceinline__ void welford_merge_element(int& count, float& mean, float& m2n, const int& count_new,
                                                      const float& mean_new, const float& m2n_new) {
  float factor = float(1.0) / ::max(1, (count + count_new));
  float delta0 = mean - mean_new;
  const float c = count, c_new = count_new;
  mean = __fmul_rn(FUSE_NEW ? __fmaf_rn(mean_new, c_new, __fmul_rn(mean, c)) : __fmaf_rn(mean, c, __fmul_rn(mean_new, c_new)),
                   factor);
  // m2n += m2n_new + delta0 * delta0 * count_new * count * factor
  m2n = __fadd_rn(m2n, __fmaf_rn(__fmul_rn(__fmul_rn(__fmul_rn(delta0, delta0), c_new), c), factor, m2n_new));
  count += count_new;
}

// torch's vertical tree over threadIdx.y; shared memory is indexed by torch's thread (tx * V + k, ty)
template <int V>
__device__ __forceinline__ void welford_merge_block_vertical(int (&count)[V], float (&mean)[V], float (&m2n)[V],
                                                             int* shmem_count, float* shmem_mean, float* shmem_m2n) {
  const int block_x = blockDim.x * V;
  auto address_base = threadIdx.x * V + threadIdx.y * block_x;
#pragma unroll
  for (int offset = blockDim.y / 2; offset > 0; offset >>= 1) {
    if (threadIdx.y < offset * 2) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        shmem_mean[address_base + k] = mean[k];
        shmem_m2n[address_base + k] = m2n[k];
        shmem_count[address_base + k] = count[k];
      }
    }
    __syncthreads();
    if (threadIdx.y < offset && threadIdx.y + offset < blockDim.y) {
      auto address = address_base + offset * block_x;
#pragma unroll
      for (int k = 0; k < V; k++) {
        auto count_new = shmem_count[address + k];
        auto mean_new = shmem_mean[address + k];
        auto m2n_new = shmem_m2n[address + k];
        welford_merge_element<false>(count[k], mean[k], m2n[k], count_new, mean_new, m2n_new);
      }
    }
  }
}

// torch's backward tree over threadIdx.y, with shared memory indexed by torch's thread as above
template <int V>
__device__ __forceinline__ void merge_block_vertical_backward(float (&sum_dy)[V], float (&sum_dy_xmu)[V], float* shmem_sum_dy,
                                                              float* shmem_sum_dy_xmu) {
  const int block_x = blockDim.x * V;
  auto address_base = threadIdx.x * V + threadIdx.y * block_x;
#pragma unroll
  for (int offset = blockDim.y / 2; offset > 0; offset >>= 1) {
    if (threadIdx.y < offset * 2) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        shmem_sum_dy[address_base + k] = sum_dy[k];
        shmem_sum_dy_xmu[address_base + k] = sum_dy_xmu[k];
      }
    }
    __syncthreads();
    if (threadIdx.y < offset && threadIdx.y + offset < blockDim.y) {
      auto address = address_base + offset * block_x;
#pragma unroll
      for (int k = 0; k < V; k++) {
        sum_dy[k] += shmem_sum_dy[address + k];
        sum_dy_xmu[k] += shmem_sum_dy_xmu[address + k];
      }
    }
  }
}

__device__ __forceinline__ void merge_block_vertical_backward(float& sum_dy, float& sum_dy_xmu, float* shmem_sum_dy,
                                                              float* shmem_sum_dy_xmu) {
  float a[1] = {sum_dy}, b[1] = {sum_dy_xmu};
  merge_block_vertical_backward<1>(a, b, shmem_sum_dy, shmem_sum_dy_xmu);
  sum_dy = a[0];
  sum_dy_xmu = b[0];
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
  o.running_mean[c] = __fmaf_rn(mean, momentum, __fmul_rn(1 - momentum, o.running_mean[c]));     // mean * momentum + (1 - momentum) * rm
  o.running_var[c] = __fmaf_rn(unbiased_var, momentum, __fmul_rn(1 - momentum, o.running_var[c]));
  o.save_invstd[c] = rsqrtf(var + o.eps);
}

// Welford statistics per channel (torch: batch_norm_collect_statistics_channels_last_kernel<..., 4>), ending in
// finish(c, mean, m2n, count) by the thread that owns channel c's final value.  The last block of each column
// leaves its semaphore at zero for the next call.
//
// Each of torch's threads walks rows m_offset + r * inner_loop_stride into PARALLEL_LOADS accumulators, one
// iteration of PARALLEL_LOADS rows at a time.  With V = 1 all rows of an iteration are loaded before the first
// update, so that they are in flight together; torch's kernel waits for each row's value before it loads the next.
// With V = kStatsVec the rows come through the ring (V channels in one 8-byte copy), kStatsStages - 1 iterations
// ahead of the updates.  The V channels of a thread share each row's validity, hence count[j] and its reciprocal.
template <int V, typename Finish>
__device__ __forceinline__ void bn_stats_body(const bf16* __restrict__ input, volatile float* staging_data, int* semaphores,
                                              const int reduction_size, const int stride, Finish finish) {
  constexpr int PARALLEL_LOADS = kParallelLoads;
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

  // torch's update of accumulator j with the next row of the walk, read from *xv when the row exists
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
      x_mean[j][k] = __fmaf_rn(delta0, x_count_inv, x_mean[j][k]);   // x_mean += delta0 * x_count_inv
      float delta1 = x_math[k] - x_mean[j][k];
      m_2_n[j][k] = __fmaf_rn(__fmul_rn(delta0, delta1), is_valid, m_2_n[j][k]);   // m_2_n += delta0 * delta1 * is_valid
    }
  };

  if constexpr (V == 1) {
    for (int i = 0; i < loop_count; i++) {
      // all rows of the iteration are loaded before any update uses one
      BVec<V> xv[PARALLEL_LOADS];
#pragma unroll
      for (int j = 0; j < PARALLEL_LOADS; j++) {
        const int m = m_offset + j * inner_loop_stride;
        if (c_valid && m < reduction_size) xv[j] = *reinterpret_cast<const BVec<V>*>(input + ((size_t)m * stride + c_offset));
      }
#pragma unroll
      for (int j = 0; j < PARALLEL_LOADS; j++) update(j, &xv[j]);
    }
  } else {
    // the ring: iterations i + 1 .. i + kStatsStages - 1 are in flight while iteration i is consumed
    constexpr unsigned D = kStatsStages;
    const int threads = blockDim.x * blockDim.y;
    BVec<V>* ring = reinterpret_cast<BVec<V>*>(ring_smem()) + threadIdx.y * blockDim.x + threadIdx.x;
    const int first_row = m_offset;
    auto issue = [&](unsigned it) {
      BVec<V>* slot = ring + (it % D) * PARALLEL_LOADS * threads;
      int m = first_row + (int)it * PARALLEL_LOADS * inner_loop_stride;
#pragma unroll
      for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride)
        if (c_valid && m < reduction_size) cp_async<sizeof(BVec<V>)>(slot + j * threads, input + ((size_t)m * stride + c_offset));
      cp_async_commit();
    };
#pragma unroll
    for (unsigned it = 0; it < D - 1; it++) issue(it);
    for (unsigned i = 0; i < (unsigned)loop_count; i++) {
      issue(i + D - 1);
      cp_async_wait<D - 1>();
      const BVec<V>* slot = ring + (i % D) * PARALLEL_LOADS * threads;
#pragma unroll
      for (int j = 0; j < PARALLEL_LOADS; j++) update(j, slot + j * threads);
    }
  }
  float mean_th[V], m2_th[V];
  int count_th[V];
#pragma unroll
  for (int k = 0; k < V; k++) {
    count_th[k] = count[0];
    mean_th[k] = x_mean[0][k];
    m2_th[k] = m_2_n[0][k];
#pragma unroll
    for (int j = 1; j < PARALLEL_LOADS; j++) welford_merge_element<true>(count_th[k], mean_th[k], m2_th[k], count[j], x_mean[j][k], m_2_n[j][k]);
  }

  __shared__ float shmem_mean[kMaxBlock];
  __shared__ float shmem_m2n[kMaxBlock];
  __shared__ int shmem_count[kMaxBlock];
  welford_merge_block_vertical<V>(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);

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
          welford_merge_element<false>(count_th[k], mean_th[k], m2_th[k], count_new, mean_new, m2n_new);
        }
      }
      welford_merge_block_vertical<V>(count_th, mean_th, m2_th, shmem_count, shmem_mean, shmem_m2n);
      if (threadIdx.y == 0 && c_valid)
#pragma unroll
        for (int k = 0; k < V; k++) finish(c_offset + k, mean_th[k], m2_th[k], count_th[k]);
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0 && c_valid)
#pragma unroll
      for (int k = 0; k < V; k++) finish(c_offset + k, mean_th[k], m2_th[k], count_th[k]);
  }
}

// Local batch norm: the statistics, then the running-statistics update and inversion (finish_stats).
template <int V>
__global__ void __launch_bounds__(kMaxBlock / V) k_bn_stats(const bf16* __restrict__ input, StatsOut o, volatile float* staging_data,
                                                            int* semaphores, const int reduction_size, const int stride) {
  if (o.num_batches_tracked && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0)
    *o.num_batches_tracked += 1;
  bn_stats_body<V>(input, staging_data, semaphores, reduction_size, stride,
                   [&](int c, float mean, float m2n, int count) { finish_stats(o, c, mean, m2n, count); });
}

// Two batch norms of one shape (a block tail's and its downsample branch's): grid.z = 2, z selecting the input and
// the outputs.  Each z plane is k_bn_stats over its input with the launch shape torch uses for it, so the bits are
// those of two k_bn_stats launches; plane 1 stages in its own region and counts on semaphores[gridDim.x + x].
template <int V>
__global__ void __launch_bounds__(kMaxBlock / V) k_bn_stats_dual(const bf16* __restrict__ input0, const bf16* __restrict__ input1,
                                                                 StatsOut o0, StatsOut o1, volatile float* staging0,
                                                                 volatile float* staging1, int* semaphores, const int reduction_size,
                                                                 const int stride) {
  const bool z = blockIdx.z != 0;
  // field by field: a reference to either parameter would put both on the stack
  const StatsOut o{z ? o1.save_mean : o0.save_mean, z ? o1.save_invstd : o0.save_invstd, z ? o1.running_mean : o0.running_mean,
                   z ? o1.running_var : o0.running_var, z ? o1.num_batches_tracked : o0.num_batches_tracked,
                   z ? o1.momentum : o0.momentum, z ? o1.bessel : o0.bessel, z ? o1.eps : o0.eps};
  if (o.num_batches_tracked && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0)
    *o.num_batches_tracked += 1;
  bn_stats_body<V>(z ? input1 : input0, z ? staging1 : staging0, semaphores + (z ? gridDim.x : 0), reduction_size, stride,
                   [&](int c, float mean, float m2n, int count) { finish_stats(o, c, mean, m2n, count); });
}

// ---- sync batch norm (torch.nn.SyncBatchNorm's autograd function) ----
// A rank's statistics travel as one row [mean (C) | invstd (C) | count] of fp32, as in torch's all_gather.

// torch.batch_norm_stats: the same statistics, ending in torch's InvStd transform instead of Var.  InvStd computes
// in double: invstd = (var != 0 || eps != 0) ? 1 / sqrt(var + (double)eps) : 0, where eps is the kernel's fp32
// copy.  Writes this rank's row `local`, with count = (float)m; no running statistics.
template <int V>
__global__ void __launch_bounds__(kMaxBlock / V) k_bn_sync_stats(const bf16* __restrict__ input, float* __restrict__ local,
                                                                 const float eps, volatile float* staging_data, int* semaphores,
                                                                 const int reduction_size, const int stride) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0 && threadIdx.y == 0) local[2 * stride] = (float)reduction_size;
  bn_stats_body<V>(input, staging_data, semaphores, reduction_size, stride, [&](int c, float mean, float m2n, int count) {
    const float var = m2n / count;
    local[c] = mean;
    local[stride + c] = (var != 0.f || eps != 0.f) ? (float)(1.0 / sqrt((double)var + (double)eps)) : 0.f;
  });
}

// torch.batch_norm_gather_stats_with_counts (batch_norm_reduce_statistics_kernel<float, float, int>) over the W
// gathered rows, ranks folded 0..W-1; ranks with count < 1 are skipped, as torch's SyncBatchNorm drops them before
// the call.  The expressions are torch's with the contractions nvcc made in its sm_90 build (read from the SASS of
// libtorch_cuda.so): v * v - eps and (v * v - eps) * count + t are FMAs, as is the mean's n * factor * avg term;
// factor = 1.0 / (n + count) is a correctly rounded fp32 reciprocal, and n stays an int, n = int(float(n) + count).
// Also writes norm_fct = 1 / float(sum of int(count)), torch.batch_norm_backward_elemt's factor for the backward,
// and adds 1 to num_batches_tracked (the module's increment).
__global__ void __launch_bounds__(kEwThreads) k_bn_sync_merge(const float* __restrict__ rows, const int row_stride, const int world,
                                                              float* __restrict__ save_mean, float* __restrict__ save_invstd,
                                                              float* __restrict__ norm_fct, float* __restrict__ running_mean,
                                                              float* __restrict__ running_var, long long* num_batches_tracked,
                                                              const float momentum, const float eps, const int stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    long long total = 0;
    for (int j = 0; j < world; j++) {
      const float count = rows[(size_t)j * row_stride + 2 * stride];
      if (count >= 1.f) total += (int)count;
    }
    *norm_fct = 1.f / (float)total;
    if (num_batches_tracked) *num_batches_tracked += 1;
  }
  if (i >= stride) return;
  float avg = 0.f, var_n = 0.f;
  int n = 0;
  for (int j = 0; j < world; j++) {
    const float* row = rows + (size_t)j * row_stride;
    const float count = row[2 * stride];
    if (!(count >= 1.f)) continue;
    const float m = row[i];
    float v = __fdiv_rn(1.f, row[stride + i]);
    v = __fmaf_rn(v, v, -eps);
    const float nf = (float)n;
    const float factor = __fdiv_rn(1.f, __fadd_rn(nf, count));
    const float d = __fsub_rn(avg, m);
    const float t = __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), nf), count), factor);   // (avg - m)^2 * n * count * factor
    var_n = __fadd_rn(var_n, __fmaf_rn(v, count, t));
    avg = __fmaf_rn(__fmul_rn(nf, factor), avg, __fmul_rn(__fmul_rn(count, factor), m));  // n * factor * avg + count * factor * m
    n = (int)__fadd_rn(nf, count);
  }
  save_mean[i] = avg;
  save_invstd[i] = __fdiv_rn(1.f, __fsqrt_rn(__fadd_rn(__fdiv_rn(var_n, (float)n), eps)));
  running_mean[i] = __fmaf_rn(avg, momentum, __fmul_rn(1 - momentum, running_mean[i]));
  const float unbiased_var = __fdiv_rn(var_n, (float)(n - 1));
  running_var[i] = __fmaf_rn(unbiased_var, momentum, __fmul_rn(1 - momentum, running_var[i]));
}

// What is fused after the batch norm: nothing, a ReLU, `+= identity` and a ReLU (a block's tail), or `+=` a second
// batch norm's output and a ReLU (a tail whose identity is a downsample branch's batch norm).
enum Tail { kTailNone, kTailRelu, kTailAddRelu, kTailBnAddRelu };
constexpr int kTails = 4;

// y = bf16(bn(x)) (kTailNone: torch.batch_norm_elemt), y = relu(bn(x)) (kTailRelu) or y = relu(bf16(bn(x)) +
// identity) (kTailAddRelu), rounded where eager torch rounds: the batch-norm output to bf16, the bf16 sum of the
// residual add to bf16.  `t <= 0 ? 0 : bf16(t)` is relu(bf16(t)) because rounding keeps the sign; NaN passes
// through as in torch's relu.  kTailBnAddRelu reads the downsample branch's input from `identity` and applies its
// batch norm (mean2 .. shift2) first: y = relu(bf16(bn(x)) + bf16(bn2(identity))), each rounded as eager torch
// rounds the two batch norms' outputs; that output is never written.
//
// With `mask` set (C % 8 == 0) a kernel with a ReLU also writes the ReLU's backward predicate !(y <= 0), computed
// from the stored bf16 y, as one bit per element: element a = m * C + c is bit a % 8 of byte a / 8.  V = 8 threads
// write one byte each per row.  V = 1 threads pack a byte with a ballot over the 8 lanes of one 8-channel group:
// block.x = min(C, 256) is then a multiple of 8, so those lanes share a row and are all in or all out of range, and
// they reach the ballot together or return together.
template <int V, Tail TAIL>
__global__ void __launch_bounds__(kEwThreads) k_bn_transform(const bf16* __restrict__ input, const bf16* __restrict__ identity,
                                                             bf16* __restrict__ out, uint8_t* __restrict__ mask,
                                                             const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                             const float* __restrict__ weight, const float* __restrict__ shift,
                                                             const float* __restrict__ mean2, const float* __restrict__ inv_std2,
                                                             const float* __restrict__ weight2, const float* __restrict__ shift2,
                                                             const int reduction_size, const int stride) {
  static_assert(V == 1 || V == 8, "a thread writes a whole mask byte (V = 8) or one bit of a ballot (V = 1)");
  constexpr bool BN2 = TAIL == kTailBnAddRelu;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], inv_std_c[V], w_c[V], s_c[V], m2_c[V], inv_std2_c[V], w2_c[V], s2_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    m_c[j] = mean[c0 + j];
    inv_std_c[j] = inv_std[c0 + j];
    w_c[j] = weight[c0 + j];
    s_c[j] = shift[c0 + j];
    if (BN2) {
      m2_c[j] = mean2[c0 + j];
      inv_std2_c[j] = inv_std2[c0 + j];
      w2_c[j] = weight2[c0 + j];
      s2_c[j] = shift2[c0 + j];
    }
  }
  const unsigned lane = (threadIdx.x + threadIdx.y * blockDim.x) % 32;
  const unsigned group = 0xffu << (lane & ~7u);
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const int a = m * stride + c0;
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> zv;
    if (TAIL == kTailAddRelu || BN2) zv = *reinterpret_cast<const BVec<V>*>(identity + a);
    BVec<V> yv;
    unsigned bits = 0;
#pragma unroll
    for (int j = 0; j < V; j++) {
      auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
      if (TAIL == kTailAddRelu || BN2) {
        if (BN2) zv.v[j] = __float2bfloat16(w2_c[j] * (__bfloat162float(zv.v[j]) - m2_c[j]) * inv_std2_c[j] + s2_c[j]);
        const bf16 r = __float2bfloat16(__bfloat162float(__float2bfloat16(tmp)) + __bfloat162float(zv.v[j]));
        yv.v[j] = __bfloat162float(r) <= 0.f ? __float2bfloat16(0.f) : r;
      } else if (TAIL == kTailRelu) {
        yv.v[j] = tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
      } else {
        yv.v[j] = __float2bfloat16(tmp);
      }
      bits |= (unsigned)!(__bfloat162float(yv.v[j]) <= 0.f) << j;
    }
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
    if (TAIL != kTailNone && mask) {
      if (V == 1) bits = (__ballot_sync(group, bits) >> (lane & ~7u)) & 0xffu;
      if (V == 8 || lane % 8 == 0) mask[a >> 3] = (uint8_t)bits;
    }
  }
}

// ---- the ResNet stem: batch norm -> ReLU -> max_pool2d(kernel 3, stride 2, padding 1) ----
// Pooled rows are N * OH * OW with OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1.  Window (ph, pw) covers input rows
// 2 * ph - 1 .. 2 * ph + 1 and columns 2 * pw - 1 .. 2 * pw + 1, clipped to the input; an element's position in it
// is (ih - 2 * ph + 1) * 3 + (iw - 2 * pw + 1).
struct PoolDims {
  int h, w, oh, ow;
};
// The argmax byte of a window whose maximum is 0: the ReLU passes no gradient to any of its elements.
constexpr uint8_t kPoolNoGrad = 0xff;

// pooled = max over the window of y = relu(bf16(bn(x))) (y as k_bn_transform<V, kTailRelu> computes it), selected
// as torch's channels-last max_pool2d selects it: rows first, then columns, and a y greater than the maximum so far
// or NaN replaces it, so the first maximum wins a tie and the last NaN wins.  `argmax` receives the winner's
// position, or kPoolNoGrad where the maximum is 0.  That one byte stands in for the ReLU mask: every element a
// window selects holds that window's maximum, so the element's ReLU passes its gradient exactly when the maximum
// is not <= 0.  The 112 x 112 y is never written.
template <int V>
__global__ void __launch_bounds__(kEwThreads) k_bn_pool_fwd(const bf16* __restrict__ input, bf16* __restrict__ out,
                                                            uint8_t* __restrict__ argmax, const float* __restrict__ mean,
                                                            const float* __restrict__ inv_std, const float* __restrict__ weight,
                                                            const float* __restrict__ shift, const PoolDims d, const int pooled_rows,
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
    const int pw = p % d.ow, ph = (p / d.ow) % d.oh, n = p / (d.ow * d.oh);
    float best[V];
    uint8_t pos[V];
#pragma unroll
    for (int j = 0; j < V; j++) {
      best[j] = -INFINITY;
      pos[j] = 0;
    }
    for (int ih = max(2 * ph - 1, 0); ih < min(2 * ph + 2, d.h); ih++) {
      for (int iw = max(2 * pw - 1, 0); iw < min(2 * pw + 2, d.w); iw++) {
        const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + ((size_t)(n * d.h + ih) * d.w + iw) * stride + c0);
        const uint8_t at = (ih - 2 * ph + 1) * 3 + (iw - 2 * pw + 1);
#pragma unroll
        for (int j = 0; j < V; j++) {
          const auto tmp = w_c[j] * (__bfloat162float(xv.v[j]) - m_c[j]) * inv_std_c[j] + s_c[j];
          const float y = __bfloat162float(tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp));
          if (y > best[j] || isnan(y)) {
            best[j] = y;
            pos[j] = at;
          }
        }
      }
    }
    BVec<V> yv;
    struct alignas(V) {
      uint8_t v[V];
    } av;   // one V-byte store (the launcher picks V = 8 only with argmax on the 16-byte grid and C % 8 == 0)
#pragma unroll
    for (int j = 0; j < V; j++) {
      yv.v[j] = __float2bfloat16(best[j]);
      av.v[j] = best[j] <= 0.f ? kPoolNoGrad : pos[j];
    }
    const size_t a = (size_t)p * stride + c0;
    *reinterpret_cast<BVec<V>*>(out + a) = yv;
    *reinterpret_cast<decltype(av)*>(argmax + a) = av;
  }
}

// g of input row m, channel c: torch's channels-last max_pool2d backward followed by threshold_backward.  An element
// inside one window only takes that window's gradient as it is (-0.0 stays -0.0); one inside several sums the
// gradients of the windows that selected it in fp32 from 0, in (ph, pw) order, and rounds once.  An element no
// window selected, or whose ReLU stops the gradient (kPoolNoGrad), gets +0.
__device__ __forceinline__ bf16 pool_grad(const bf16* __restrict__ dpool, const uint8_t* __restrict__ argmax, const PoolDims& d,
                                          const int m, const int c, const int stride) {
  const int iw = m % d.w, ih = (m / d.w) % d.h, n = m / (d.w * d.h);
  const int ph0 = ih >> 1, ph1 = min((ih + 1) >> 1, d.oh - 1);
  const int pw0 = iw >> 1, pw1 = min((iw + 1) >> 1, d.ow - 1);
  // the (up to) four windows' bytes and gradients are loaded together, none waiting for another's compare; a
  // missing second row or column repeats the first, whose slot is then never selected
  const int o = ((n * d.oh + ph0) * d.ow + pw0) * stride + c;
  const int dr = (ph1 - ph0) * d.ow * stride, dc = (pw1 - pw0) * stride;
  const uint8_t a[4] = {argmax[o], argmax[o + dc], argmax[o + dr], argmax[o + dr + dc]};
  const bf16 v[4] = {dpool[o], dpool[o + dc], dpool[o + dr], dpool[o + dr + dc]};
  const int at = (ih - 2 * ph0 + 1) * 3 + (iw - 2 * pw0 + 1);   // position in window (ph0, pw0); -2 per later row / column
  if (ph0 == ph1 && pw0 == pw1) return a[0] == at ? v[0] : __float2bfloat16(0.f);
  float sum = 0.f;
  if (a[0] == at) sum += __bfloat162float(v[0]);
  if (pw1 != pw0 && a[1] == at - 2) sum += __bfloat162float(v[1]);
  if (ph1 != ph0 && a[2] == at - 6) sum += __bfloat162float(v[2]);
  if (ph1 != ph0 && pw1 != pw0 && a[3] == at - 8) sum += __bfloat162float(v[3]);
  return __float2bfloat16(sum);
}

// The ReLU's backward (threshold_backward: y <= 0 ? 0 : dy), read from dy and the saved output y, or from dy and
// the predicate !(y <= 0) that k_bn_transform wrote as a bit.
__device__ __forceinline__ bf16 relu_grad(bf16 dy, bf16 y) { return __bfloat162float(y) <= 0.f ? __float2bfloat16(0.f) : dy; }
__device__ __forceinline__ bf16 relu_grad_bit(bf16 dy, unsigned bit) { return bit ? dy : __float2bfloat16(0.f); }
// autograd's sum of two gradients of one bf16 tensor
__device__ __forceinline__ bf16 add_grads(bf16 a, bf16 b) { return __float2bfloat16(__bfloat162float(a) + __bfloat162float(b)); }

// Where the backward kernels take g, the batch norm's output gradient, from: the tensor the reduce kernel wrote
// (kGradMasked), relu_grad of dy and y (kGradY) or of dy and k_bn_transform's bits (kGradBits), dy itself, for
// a batch norm without a ReLU after it (kGradDy), or pool_grad of the pooled gradient dy and k_bn_pool_fwd's
// argmax bytes (kGradPool, the stem; the reduce kernel only).
enum GradSrc { kGradMasked, kGradY, kGradBits, kGradDy, kGradPool };
constexpr int kGradSrcs = 5;

// Per-channel sums of g and g * (x - mean) with g from G (torch: batch_norm_backward_reduce_channels_last_kernel<4>),
// and dweight / dbias.  kGradBits reads the ReLU's predicate from `mask` (k_bn_transform's bits) instead of y from
// `output`.  With `grad_output2` set, dy is the bf16 sum of the two gradients, as autograd rounds it when a tensor
// has two consumers; without it dy is taken as it is, so a -0.0 gradient stays -0.0.  With `masked` set (the block
// tail, where g is also the identity branch's gradient, and the stem) g is written there as well.  kGradPool reads
// the pooled gradient from `grad_output` and the argmax bytes from `mask`, over the input geometry `pool`.
//
// With `vec` = kBwdVec (the launcher divides block.x by it) a hardware thread carries kBwdVec adjacent torch
// threads, as in k_bn_stats, and reads dy, x, dy2, y and x2 through the ring, bwd_ring_stages(operands) - 1 iterations
// ahead of the sums; g is written kBwdVec channels at a time.  With `vec` = 1 (C % 8 != 0, an operand off the
// 16-byte grid, the stem's kGradPool) each thread loads all rows of an iteration before the first sum uses one.
//
// DUAL (a tail whose identity is a downsample branch's batch norm, fed the same g): `input2` is that batch norm's
// input, and the same walk also sums g * (x2 - mean2).  Each of the three sums is accumulated, merged over the block
// and over the grid exactly as a k_bn_bwd_reduce launch for its own batch norm would, so Σg is both dbias values.
template <GradSrc G, bool DUAL>
__global__ void __launch_bounds__(kMaxBlock) k_bn_bwd_reduce(const bf16* __restrict__ input, const bf16* __restrict__ grad_output,
                                const bf16* __restrict__ grad_output2, const bf16* __restrict__ output,
                                const uint8_t* __restrict__ mask, bf16* __restrict__ masked, const float* __restrict__ mean,
                                const float* __restrict__ inv_std, float* __restrict__ sum_dy_o, float* __restrict__ sum_dy_xmu_o,
                                float* __restrict__ grad_weight, float* __restrict__ grad_bias, volatile float* staging_data,
                                int* semaphores, const PoolDims pool, const bf16* __restrict__ input2,
                                const float* __restrict__ mean2, const float* __restrict__ inv_std2, float* __restrict__ sum_dy_xmu2_o,
                                float* __restrict__ grad_weight2, float* __restrict__ grad_bias2, const int reduction_size,
                                const int stride, const int vec) {
  static_assert(G != kGradMasked, "the reduce kernel computes g");
  constexpr bool BITS = G == kGradBits;
  constexpr bool POOL = G == kGradPool;
  constexpr int PARALLEL_LOADS = kParallelLoads;
  __shared__ float shmem_sum_dy[kMaxBlock];
  __shared__ float shmem_sum_dy_xmu[kMaxBlock];
  __shared__ bool is_last_block_done;

  // V channels (torch threads) per hardware thread: 1, the register walk, or kBwdVec, the ring
  auto body = [&](auto vec_c) {
    constexpr int V = decltype(vec_c)::value;
    float sum_dy[PARALLEL_LOADS][V];
    float sum_dy_xmu[PARALLEL_LOADS][V];
    float sum_dy_xmu2[PARALLEL_LOADS][V];
#pragma unroll
    for (int i = 0; i < PARALLEL_LOADS; i++) {
#pragma unroll
      for (int k = 0; k < V; k++) {
        sum_dy[i][k] = float(0);
        sum_dy_xmu[i][k] = float(0);
        sum_dy_xmu2[i][k] = float(0);
      }
    }
    int inner_loop_stride = blockDim.y * gridDim.y;
    int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
    int c_offset = (blockIdx.x * blockDim.x + threadIdx.x) * V;
    if (c_offset >= stride || m_offset >= reduction_size) return;

    int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
    int address_base = m_offset * stride + c_offset;
    int address_increment = inner_loop_stride * stride;
    float r_mean[V], factor[V], r_mean2[V];
#pragma unroll
    for (int k = 0; k < V; k++) {
      r_mean[k] = mean[c_offset + k];
      factor[k] = inv_std[c_offset + k];
      r_mean2[k] = DUAL ? mean2[c_offset + k] : 0.f;
    }

    // the next row of the walk into accumulators j: g from dy (, dy2) and y or the mask byte, written to `masked`
    // where that is set, then torch's sums; the operands are read only when the row exists
    auto consume = [&](int j, const BVec<V>* dy_p, const BVec<V>* dy2_p, const BVec<V>* y_p, uint8_t mask_byte, const BVec<V>* x_p,
                       const BVec<V>* x2_p) {
      float x_input[V], x_input2[V], x_grad_output[V];
      if (m_offset < reduction_size) {
        const unsigned bits = BITS ? mask_byte >> (address_base & 7) : 0u;
        BVec<V> gv;
#pragma unroll
        for (int k = 0; k < V; k++) {
          const bf16 dy = !POOL && grad_output2 ? add_grads(dy_p->v[k], dy2_p->v[k]) : dy_p->v[k];
          gv.v[k] = BITS ? relu_grad_bit(dy, (bits >> k) & 1u) : G == kGradY ? relu_grad(dy, y_p->v[k]) : dy;
          x_input[k] = __bfloat162float(x_p->v[k]);
          x_input2[k] = DUAL ? __bfloat162float(x2_p->v[k]) : 0.f;
          x_grad_output[k] = __bfloat162float(gv.v[k]);
        }
        if (masked) *reinterpret_cast<BVec<V>*>(masked + address_base) = gv;
      } else {
#pragma unroll
        for (int k = 0; k < V; k++) {
          x_input[k] = float(0);
          x_input2[k] = float(0);
          x_grad_output[k] = float(0);
        }
      }
      m_offset += inner_loop_stride;
      address_base += address_increment;
#pragma unroll
      for (int k = 0; k < V; k++) {
        sum_dy[j][k] += x_grad_output[k];
        sum_dy_xmu[j][k] = __fmaf_rn(x_grad_output[k], x_input[k] - r_mean[k], sum_dy_xmu[j][k]);   // += g * (x - mean)
        if (DUAL) sum_dy_xmu2[j][k] = __fmaf_rn(x_grad_output[k], x_input2[k] - r_mean2[k], sum_dy_xmu2[j][k]);
      }
    };

    if constexpr (V == 1) {
      for (int i = 0; i < loop_count; i++) {
        // all rows of the iteration are loaded before any sum uses one
        BVec<V> dy_v[PARALLEL_LOADS], dy2_v[PARALLEL_LOADS], y_v[PARALLEL_LOADS], x_v[PARALLEL_LOADS], x2_v[PARALLEL_LOADS];
        uint8_t mask_v[PARALLEL_LOADS];
#pragma unroll
        for (int j = 0; j < PARALLEL_LOADS; j++) {
          if (m_offset + j * inner_loop_stride < reduction_size) {
            const int a = address_base + j * address_increment;
            if (POOL) dy_v[j].v[0] = pool_grad(grad_output, mask, pool, m_offset + j * inner_loop_stride, c_offset, stride);
            else dy_v[j].v[0] = grad_output[a];
            if (grad_output2) dy2_v[j].v[0] = grad_output2[a];
            if (BITS) mask_v[j] = mask[a >> 3];
            else if (G == kGradY) y_v[j].v[0] = output[a];
            x_v[j].v[0] = input[a];
            if (DUAL) x2_v[j].v[0] = input2[a];
          }
        }
#pragma unroll
        for (int j = 0; j < PARALLEL_LOADS; j++) consume(j, &dy_v[j], &dy2_v[j], &y_v[j], mask_v[j], &x_v[j], &x2_v[j]);
      }
    } else {
      const int ops = bwd_ring_operands(G == kGradY, grad_output2 != nullptr, DUAL);
      // the ring: iterations i + 1 .. i + D - 1 are in flight while iteration i is consumed
      auto ring_walk = [&](auto stages_c) {
        constexpr unsigned D = decltype(stages_c)::value;
        const int threads = blockDim.x * blockDim.y;
        const int op_dy2 = 2, op_y = op_dy2 + (grad_output2 != nullptr), op_x2 = op_y + (G == kGradY);   // dy is 0, x is 1
        BVec<V>* ring = reinterpret_cast<BVec<V>*>(ring_smem()) + threadIdx.y * blockDim.x + threadIdx.x;
        auto stage = [&](unsigned it) { return ring + (it % D) * ops * PARALLEL_LOADS * threads; };
        const int first_row = m_offset;
        const int iteration_rows = PARALLEL_LOADS * inner_loop_stride;
        auto issue = [&](unsigned it) {
          BVec<V>* slot = stage(it);
          int m = first_row + (int)it * iteration_rows;
#pragma unroll
          for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride, slot += threads) {
            if (m < reduction_size) {
              const size_t a = (size_t)m * stride + c_offset;
              cp_async<sizeof(BVec<V>)>(slot, grad_output + a);
              cp_async<sizeof(BVec<V>)>(slot + PARALLEL_LOADS * threads, input + a);
              if (grad_output2) cp_async<sizeof(BVec<V>)>(slot + op_dy2 * PARALLEL_LOADS * threads, grad_output2 + a);
              if (G == kGradY) cp_async<sizeof(BVec<V>)>(slot + op_y * PARALLEL_LOADS * threads, output + a);
              if (DUAL) cp_async<sizeof(BVec<V>)>(slot + op_x2 * PARALLEL_LOADS * threads, input2 + a);
            }
          }
          cp_async_commit();
        };
        // the mask (1/16 of the traffic; one byte holds a thread's V bits) is a plain load, one iteration ahead
        uint8_t mask_next[PARALLEL_LOADS];
        auto load_mask = [&](unsigned it) {
          int m = first_row + (int)it * iteration_rows;
#pragma unroll
          for (int j = 0; j < PARALLEL_LOADS; j++, m += inner_loop_stride)
            if (m < reduction_size) mask_next[j] = mask[((size_t)m * stride + c_offset) >> 3];
        };
        if (BITS) load_mask(0);
#pragma unroll
        for (unsigned it = 0; it < D - 1; it++) issue(it);
        for (unsigned i = 0; i < (unsigned)loop_count; i++) {
          issue(i + D - 1);
          uint8_t mask_v[PARALLEL_LOADS];
#pragma unroll
          for (int j = 0; j < PARALLEL_LOADS; j++) mask_v[j] = mask_next[j];
          if (BITS) load_mask(i + 1);
          cp_async_wait<D - 1>();
          const BVec<V>* slot = stage(i);
#pragma unroll
          for (int j = 0; j < PARALLEL_LOADS; j++, slot += threads)
            consume(j, slot, slot + op_dy2 * PARALLEL_LOADS * threads, slot + op_y * PARALLEL_LOADS * threads, mask_v[j],
                    slot + PARALLEL_LOADS * threads, slot + op_x2 * PARALLEL_LOADS * threads);
        }
      };
      if (DUAL || bwd_ring_stages(ops) == kBwdStagesWide) ring_walk(std::integral_constant<unsigned, kBwdStagesWide>{});
      else ring_walk(std::integral_constant<unsigned, kBwdStages>{});
    }

    float sum_dy_th[V], sum_dy_xmu_th[V], sum_dy_xmu2_th[V];
#pragma unroll
    for (int k = 0; k < V; k++) {
#pragma unroll
      for (int j = 1; j < PARALLEL_LOADS; j++) {
        sum_dy[0][k] += sum_dy[j][k];
        sum_dy_xmu[0][k] += sum_dy_xmu[j][k];
        if (DUAL) sum_dy_xmu2[0][k] += sum_dy_xmu2[j][k];
      }
      sum_dy_th[k] = sum_dy[0][k];
      sum_dy_xmu_th[k] = sum_dy_xmu[0][k];
      sum_dy_xmu2_th[k] = sum_dy_xmu2[0][k];
    }

    // the third sum takes the same tree after the first two (each value's tree is independent of the others)
    auto merge = [&]() {
      merge_block_vertical_backward<V>(sum_dy_th, sum_dy_xmu_th, shmem_sum_dy, shmem_sum_dy_xmu);
      if (DUAL) {
        __syncthreads();
        float unused[V] = {};
        merge_block_vertical_backward<V>(sum_dy_xmu2_th, unused, shmem_sum_dy, shmem_sum_dy_xmu);
      }
    };
    merge();

    auto write_sums = [&]() {
#pragma unroll
      for (int k = 0; k < V; k++) {
        const int c = c_offset + k;
        grad_bias[c] = sum_dy_th[k];
        grad_weight[c] = sum_dy_xmu_th[k] * factor[k];
        sum_dy_o[c] = sum_dy_th[k];
        sum_dy_xmu_o[c] = sum_dy_xmu_th[k];
        if (DUAL) {
          grad_bias2[c] = sum_dy_th[k];
          grad_weight2[c] = sum_dy_xmu2_th[k] * inv_std2[c];
          sum_dy_xmu2_o[c] = sum_dy_xmu2_th[k];
        }
      }
    };
    if (gridDim.y > 1) {
      volatile float* staging_sum_dy = staging_data;
      volatile float* staging_sum_dy_xmu = &staging_data[stride * gridDim.y];
      volatile float* staging_sum_dy_xmu2 = &staging_data[2 * stride * gridDim.y];
      address_base = c_offset + blockIdx.y * stride;
      if (threadIdx.y == 0 && c_offset < stride) {
#pragma unroll
        for (int k = 0; k < V; k++) {
          staging_sum_dy[address_base + k] = sum_dy_th[k];
          staging_sum_dy_xmu[address_base + k] = sum_dy_xmu_th[k];
          if (DUAL) staging_sum_dy_xmu2[address_base + k] = sum_dy_xmu2_th[k];
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
          sum_dy_xmu2_th[k] = float(0.0);
        }
        for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
          address_base = c_offset + y * stride;
#pragma unroll
          for (int k = 0; k < V; k++) {
            sum_dy_th[k] += (c_offset < stride ? staging_sum_dy[address_base + k] : float(0.0));
            sum_dy_xmu_th[k] += (c_offset < stride ? staging_sum_dy_xmu[address_base + k] : float(0.0));
            if (DUAL) sum_dy_xmu2_th[k] += (c_offset < stride ? staging_sum_dy_xmu2[address_base + k] : float(0.0));
          }
        }
        merge();
        if (threadIdx.y == 0 && c_offset < stride) write_sums();
      }
    } else {
      if (blockIdx.y == 0 && threadIdx.y == 0 && c_offset < stride) write_sums();
    }
  };
  if constexpr (POOL) body(std::integral_constant<int, 1>{});
  else if (vec == kBwdVec) body(std::integral_constant<int, kBwdVec>{});
  else body(std::integral_constant<int, 1>{});
}

// dx (torch: batch_norm_backward_elemt_channels_last_kernel_impl) with g from G (kGradMasked: `grad_output` is the
// tensor the reduce kernel wrote); dy is summed with `grad_output2` when that is set, as in k_bn_bwd_reduce.
//
// norm_fct is torch's 1 / rows.  A local site passes the value, (float)(1.0 / m) computed by the launcher from this
// call's rows (FCT_PTR false); a sync site passes a pointer to what k_bn_sync_merge wrote, 1 / float(rows of all
// ranks) (FCT_PTR true).  The choice is a template parameter because the two round differently, as torch's two
// kernels do: with norm_fct a kernel parameter nvcc contracts `g - sum_dy * norm_fct` into one FMA per element,
// with norm_fct loaded from memory it multiplies once per channel and subtracts.  One kernel that selects between
// value and pointer at run time rounds a local site's dx like a sync site's, which is not eager torch's.
//
// DUAL: also dx2 of the downsample branch's batch norm (input2, mean2 .. sum_dy_xmu2), fed the same g, which the
// kernel derives from dy (and dy2) and the mask or y; Σg is the same for both.
template <int V, GradSrc G, bool FCT_PTR, bool DUAL>
__global__ void __launch_bounds__(kEwThreads) k_bn_bwd_elemt(const bf16* __restrict__ grad_output, const bf16* __restrict__ grad_output2,
                                                             const bf16* __restrict__ output, const uint8_t* __restrict__ mask,
                                                             const bf16* __restrict__ input, bf16* __restrict__ grad_input,
                                                             const float* __restrict__ mean, const float* __restrict__ inv_std,
                                                             const float* __restrict__ weight, const float* __restrict__ sum_dy,
                                                             const float* __restrict__ sum_dy_xmu,
                                                             const float* __restrict__ norm_fct_ptr, const float norm_fct_value,
                                                             const bf16* __restrict__ input2, bf16* __restrict__ grad_input2,
                                                             const float* __restrict__ mean2, const float* __restrict__ inv_std2,
                                                             const float* __restrict__ weight2, const float* __restrict__ sum_dy_xmu2,
                                                             const int reduction_size, const int stride) {
  static_assert(!DUAL || (G == kGradY || G == kGradBits), "a dual tail derives g from dy and the ReLU");
  const float norm_fct = FCT_PTR ? *norm_fct_ptr : norm_fct_value;
  const int c0 = (blockIdx.x * blockDim.x + threadIdx.x) * V;
  if (c0 >= stride) return;
  float m_c[V], m_dy_c[V], factor_1_c[V], factor_2_c[V];
  float m2_c[V], factor2_1_c[V], factor2_2_c[V];
#pragma unroll
  for (int j = 0; j < V; j++) {
    m_c[j] = mean[c0 + j];
    m_dy_c[j] = sum_dy[c0 + j] * norm_fct;
    factor_1_c[j] = inv_std[c0 + j];
    factor_2_c[j] = weight[c0 + j] * factor_1_c[j];
    factor_1_c[j] = factor_1_c[j] * factor_1_c[j] * sum_dy_xmu[c0 + j] * norm_fct;
    if (DUAL) {
      m2_c[j] = mean2[c0 + j];
      factor2_1_c[j] = inv_std2[c0 + j];
      factor2_2_c[j] = weight2[c0 + j] * factor2_1_c[j];
      factor2_1_c[j] = factor2_1_c[j] * factor2_1_c[j] * sum_dy_xmu2[c0 + j] * norm_fct;
    }
  }
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const int a = m * stride + c0;
    const BVec<V> gv = *reinterpret_cast<const BVec<V>*>(grad_output + a);
    BVec<V> gv2, yv;
    if (G != kGradMasked && grad_output2) gv2 = *reinterpret_cast<const BVec<V>*>(grad_output2 + a);
    unsigned bits = 0;
    if (G == kGradY) yv = *reinterpret_cast<const BVec<V>*>(output + a);
    if (G == kGradBits) bits = mask[a >> 3] >> (a & 7);
    const BVec<V> xv = *reinterpret_cast<const BVec<V>*>(input + a);
    BVec<V> x2v, dxv, dx2v;
    if (DUAL) x2v = *reinterpret_cast<const BVec<V>*>(input2 + a);
#pragma unroll
    for (int j = 0; j < V; j++) {
      const bf16 dy = G != kGradMasked && grad_output2 ? add_grads(gv.v[j], gv2.v[j]) : gv.v[j];
      const float g = __bfloat162float(G == kGradMasked || G == kGradDy ? dy
                                       : G == kGradY ? relu_grad(dy, yv.v[j]) : relu_grad_bit(dy, (bits >> j) & 1u));
      dxv.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(xv.v[j]) - m_c[j]) * factor_1_c[j]) * factor_2_c[j]);
      if (DUAL)
        dx2v.v[j] = __float2bfloat16((g - m_dy_c[j] - (__bfloat162float(x2v.v[j]) - m2_c[j]) * factor2_1_c[j]) * factor2_2_c[j]);
    }
    *reinterpret_cast<BVec<V>*>(grad_input + a) = dxv;
    if (DUAL) *reinterpret_cast<BVec<V>*>(grad_input2 + a) = dx2v;
  }
}

}  // namespace bn
}  // namespace b200c
