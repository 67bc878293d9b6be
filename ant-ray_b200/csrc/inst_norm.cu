// Launchers of the fused batch-norm kernels (norm_kernels.cuh, norm_infer.cuh, norm_act.cuh, norm_res.cuh, norm_cat.cuh,
// norm_slice.cuh, norm_shuffle.cuh, norm_pool2.cuh); argument checking lives in b200coll.cu.
#include <algorithm>
#include <initializer_list>
#include <type_traits>

#include "norm_act.cuh"
#include "norm_cat.cuh"
#include "norm_infer.cuh"
#include "norm_kernels.cuh"
#include "norm_launch.h"
#include "norm_pool2.cuh"
#include "norm_res.cuh"
#include "norm_shuffle.cuh"
#include "norm_slice.cuh"

namespace b200c {
namespace bn {

static int ceil_div(int a, int b) { return (a + b - 1) / b; }

// torch's lastPow2 (ATen/native/cuda/LaunchUtils.h)
static int last_pow2(unsigned n) {
  n |= (n >> 1);
  n |= (n >> 2);
  n |= (n >> 4);
  n |= (n >> 8);
  n |= (n >> 16);
  return std::max<int>(1, n - (n >> 1));
}

// torch's flexible_launch_configs with coop_flag = true: the statistics and backward-reduce kernels must run
// with exactly this block and grid, because the per-channel reduction order follows from them.
static void reduce_config(int reduction, int stride, dim3* block, dim3* grid) {
  int block_x = std::min(last_pow2(stride), kTileW);
  int block_y = std::min(last_pow2(ceil_div(reduction, kElemsPerThread)), kMaxBlock / block_x);
  if (block_x * block_y != kMaxBlock) block_x = std::min(last_pow2(stride), kMaxBlock / block_y);
  int grid_y = std::min(ceil_div(reduction, block_y * kElemsPerThread), kMaxHBlock);
  *block = dim3(block_x, block_y, 1);
  *grid = dim3(ceil_div(stride, block_x), grid_y < 8 ? 1 : grid_y, 1);
}

// 8 channels (16 bytes) per thread when the rows allow it: C % 8 == 0 and every operand on the 16-byte grid.  The
// statistics kernel's vector path takes the same condition: C % 8 == 0 also makes its block.x (a power of two, at
// least 8 when C >= 8) a multiple of kStatsVec, so no group of kStatsVec channels straddles C or a block.
static_assert(kEwVec % kStatsVec == 0, "vec_ok covers the statistics kernel's vector width");
static bool vec_ok(int stride, const void* const* ptrs, int n) {
  if (stride % kEwVec) return false;
  for (int i = 0; i < n; i++)
    if (reinterpret_cast<uintptr_t>(ptrs[i]) % 16) return false;
  return true;
}

// The vector paths' rings (norm_kernels.cuh) live in dynamic shared memory and, with each kernel's static shared
// memory, stay within the 48 KB a block may use without an opt-in attribute, so no launch depends on one being set.
constexpr size_t kBlockSmem = 48 * 1024;
constexpr size_t kStatsStaticSmem = 3 * kMaxBlock * 4 + 16;   // bn_stats_body's tree and last-block flag
constexpr size_t kBwdStaticSmem = 2 * kMaxBlock * 4 + 16;     // k_bn_bwd_reduce's tree and last-block flag

// The statistics ring: kStatsStages iterations of kParallelLoads rows of kStatsVec channels per hardware thread.
static size_t stats_ring_bytes(dim3 block) {
  return (size_t)kStatsStages * kParallelLoads * block.x * block.y * sizeof(BVec<kStatsVec>);
}
static_assert(kStatsStaticSmem + (size_t)kStatsStages * kParallelLoads * (kMaxBlock / kStatsVec) * sizeof(BVec<kStatsVec>) <= kBlockSmem,
              "the statistics ring fits every block");

// The backward reduce runs kBwdVec channels per hardware thread with a ring when the rows allow it (C % 8 == 0 and
// every operand it copies or writes on the 16-byte grid, as vec_ok decides for the elementwise kernels); otherwise
// one channel per thread with the register walk.  The logical block is reduce_config's.
static_assert(kBwdStaticSmem + (size_t)kBwdStagesWide * 5 * kParallelLoads * (kMaxBlock / kBwdVec) * sizeof(BVec<kBwdVec>) <= kBlockSmem &&
                  kBwdStaticSmem + (size_t)kBwdStages * 2 * kParallelLoads * (kMaxBlock / kBwdVec) * sizeof(BVec<kBwdVec>) <= kBlockSmem,
              "the backward ring fits every block: 2 stages of up to 5 operands, 3 of 2");
struct BwdReduceLaunch {
  dim3 block, grid;
  int vec;
  size_t smem;
};
static BwdReduceLaunch bwd_reduce_launch(int m, int c, GradSrc src, bool dy2, bool dual, const void* const* ptrs, int n) {
  BwdReduceLaunch l;
  reduce_config(m, c, &l.block, &l.grid);
  l.vec = 1;
  l.smem = 0;
  if (src == kGradPool || !vec_ok(c, ptrs, n)) return l;
  const int ops = bwd_ring_operands(src == kGradY, dy2, dual);
  const size_t ring = (size_t)bwd_ring_stages(ops) * ops * kParallelLoads * (l.block.x / kBwdVec) * l.block.y * sizeof(BVec<kBwdVec>);
  l.block.x /= kBwdVec;
  l.vec = kBwdVec;
  l.smem = ring;
  return l;
}

// Elementwise kernels: `rows` rows per block, and enough blocks for a few waves on the GPU (each thread then
// strides over the rows).
static void ew_config(int reduction, int stride, int vec, dim3* block, dim3* grid) {
  const int groups = stride / vec;
  const int bx = std::min(groups, kEwThreads);
  const int by = kEwThreads / bx;
  const int gx = ceil_div(groups, bx);
  const int gy = std::max(1, std::min(ceil_div(reduction, by), 4096 / gx));
  *block = dim3(bx, by, 1);
  *grid = dim3(gx, gy, 1);
}

// One scratch buffer serves sites of every channel count, so the semaphores sit in a fixed region at its start
// that no call's staging overlaps: each call finds zeros there and leaves zeros.  For c >= kTileW the reducing
// kernels' grid.x is at most c / kTileW (block.x >= kTileW), below that it is at most 2.
constexpr int kSemaphores = kMaxChannels / kTileW;
constexpr size_t kSemaphoreBytes = (size_t)kSemaphores * 4;

size_t scratch_bytes(int stride) {
  // semaphores [kSemaphores] ints | staging 3 * stride * kMaxHBlock floats | sum_dy, sum_dy_xmu [stride] floats each
  return kSemaphoreBytes + (size_t)3 * stride * kMaxHBlock * 4 + (size_t)2 * stride * 4;
}

struct Scratch {
  int* semaphores;
  float* staging;
  float* sums;
};
static Scratch carve(void* scratch, int stride) {
  char* p = static_cast<char*>(scratch);
  Scratch s;
  s.semaphores = reinterpret_cast<int*>(p);
  s.staging = reinterpret_cast<float*>(p + kSemaphoreBytes);
  s.sums = s.staging + (size_t)3 * stride * kMaxHBlock;
  return s;
}

// ---- the kernels, by their runtime keys ----
// The launchers and load_kernels() both get their kernels from the *_kernel functions below, so what is preloaded is
// what can launch; keys without a kernel give null, which a launcher reports and load_kernels() skips.
//
// with_const calls f(std::integral_constant<int, C>) for the candidate C that equals `key` (as with_world_t does in
// launch_typed.cuh) and returns the kernel f returns, or null without such a candidate.
template <int... Cs, typename F>
static auto with_const(int key, F&& f) {
  std::common_type_t<decltype(f(std::integral_constant<int, Cs>{}))...> kernel = nullptr;
  ((key == Cs ? void(kernel = f(std::integral_constant<int, Cs>{})) : void()), ...);
  return kernel;
}

using StatsKernel = void (*)(const bf16*, StatsOut, volatile float*, int*, int, int);
using SyncStatsKernel = void (*)(const bf16*, float*, float, volatile float*, int*, int, int);
using StatsDualKernel = void (*)(const bf16*, const bf16*, StatsOut, StatsOut, volatile float*, volatile float*, int*, int, int);
using TransformKernel = void (*)(const bf16*, const bf16*, bf16*, uint8_t*, const float*, const float*, const float*, const float*,
                                 const float*, const float*, const float*, const float*, int, int);
using PoolFwdKernel = void (*)(const bf16*, bf16*, uint8_t*, const float*, const float*, const float*, const float*, PoolDims, int, int);
using BwdReduceKernel = void (*)(const bf16*, const bf16*, const bf16*, const bf16*, const uint8_t*, bf16*, const float*, const float*,
                                 float*, float*, float*, float*, volatile float*, int*, PoolDims, const bf16*, const float*, const float*,
                                 float*, float*, float*, int, int, int);
using BwdElemtKernel = void (*)(const bf16*, const bf16*, const bf16*, const uint8_t*, const bf16*, bf16*, const float*, const float*,
                                const float*, const float*, const float*, const float*, float, const bf16*, bf16*, const float*,
                                const float*, const float*, const float*, int, int);

static StatsKernel stats_kernel(int vec) {
  return with_const<1, kStatsVec>(vec, [](auto v) -> StatsKernel { return k_bn_stats<decltype(v)::value>; });
}
static StatsDualKernel stats_dual_kernel(int vec) {
  return with_const<1, kStatsVec>(vec, [](auto v) -> StatsDualKernel { return k_bn_stats_dual<decltype(v)::value>; });
}
static SyncStatsKernel sync_stats_kernel(int vec) {
  return with_const<1, kStatsVec>(vec, [](auto v) -> SyncStatsKernel { return k_bn_sync_stats<decltype(v)::value>; });
}
static TransformKernel transform_kernel(int vec, int tail) {
  return with_const<1, kEwVec>(vec, [&](auto v) {
    return with_const<kTailNone, kTailRelu, kTailAddRelu, kTailBnAddRelu>(
        tail, [](auto t) -> TransformKernel { return k_bn_transform<decltype(v)::value, (Tail) decltype(t)::value>; });
  });
}
static PoolFwdKernel pool_fwd_kernel(int vec) {
  return with_const<1, kEwVec>(vec, [](auto v) -> PoolFwdKernel { return k_bn_pool_fwd<decltype(v)::value>; });
}
// the reduce kernel computes g, so it has no kGradMasked; a dual tail (a local site) reads y or its mask bits
static BwdReduceKernel bwd_reduce_kernel(int src, bool dual) {
  if (dual)
    return with_const<kGradY, kGradBits>(src, [](auto g) -> BwdReduceKernel { return k_bn_bwd_reduce<(GradSrc) decltype(g)::value, true>; });
  return with_const<kGradY, kGradBits, kGradDy, kGradPool>(
      src, [](auto g) -> BwdReduceKernel { return k_bn_bwd_reduce<(GradSrc) decltype(g)::value, false>; });
}
static BwdElemtKernel bwd_elemt_kernel(int vec, int src, bool fct_ptr, bool dual) {
  return with_const<1, kEwVec>(vec, [&](auto v) {
    if (dual)
      return with_const<kGradY, kGradBits>(src, [](auto g) -> BwdElemtKernel {
        return k_bn_bwd_elemt<decltype(v)::value, (GradSrc) decltype(g)::value, false, true>;
      });
    return with_const<kGradMasked, kGradY, kGradBits, kGradDy>(src, [&](auto g) {
      auto kernel = [](auto p) -> BwdElemtKernel {
        return k_bn_bwd_elemt<decltype(v)::value, (GradSrc) decltype(g)::value, decltype(p)::value != 0, false>;
      };
      // a batch norm without a ReLU after it runs only as a sync site, which brings its norm_fct pointer
      if constexpr (decltype(g)::value == kGradDy) return with_const<true>(fct_ptr, kernel);
      else return with_const<false, true>(fct_ptr, kernel);
    });
  });
}

// the eval-mode kernels, one pointer type per parameter type P (float or bf16)
template <typename P>
using InferTransformKernel = void (*)(const bf16*, const bf16*, bf16*, const P*, const P*, const P*, const P*, float, const P*, const P*,
                                      const P*, const P*, float, int, int);
template <typename P>
using InferPoolKernel = void (*)(const bf16*, bf16*, const P*, const P*, const P*, const P*, float, PoolDims, int, int);

template <typename P>
static InferTransformKernel<P> infer_transform_kernel(int vec, int tail) {
  return with_const<1, kEwVec>(vec, [&](auto v) {
    return with_const<kTailRelu, kTailAddRelu, kTailBnAddRelu>(tail, [](auto t) -> InferTransformKernel<P> {
      return bn_infer::k_infer_transform<decltype(v)::value, (Tail) decltype(t)::value, P>;
    });
  });
}
template <typename P>
static InferPoolKernel<P> infer_pool_kernel(int vec) {
  return with_const<1, kEwVec>(vec, [](auto v) -> InferPoolKernel<P> { return bn_infer::k_infer_pool<decltype(v)::value, P>; });
}

// the kernels of a batch norm followed by ReLU6, SiLU or Hardswish (norm_act.cuh), by b200c_act_t
using bn_act::Act;
using ActTransformKernel = void (*)(const bf16*, bf16*, const float*, const float*, const float*, const float*, int, int);
using ActBwdReduceKernel = void (*)(const bf16*, const bf16*, const float*, const float*, const float*, const float*, float*, float*,
                                    float*, float*, volatile float*, int*, bf16*, int, int);
template <typename P>
using ActInferKernel = void (*)(const bf16*, bf16*, const P*, const P*, const P*, const P*, float, int, int);

template <typename F>
static auto with_act(int act, F&& f) {
  return with_const<bn_act::kActRelu6, bn_act::kActSilu, bn_act::kActHardswish>(act, f);
}
bool act_ok(int act) { return act == bn_act::kActRelu6 || act == bn_act::kActSilu || act == bn_act::kActHardswish; }

static ActTransformKernel act_transform_kernel(int vec, int act) {
  return with_const<1, kEwVec>(vec, [&](auto v) {
    return with_act(act, [](auto a) -> ActTransformKernel { return bn_act::k_act_transform<decltype(v)::value, (Act) decltype(a)::value>; });
  });
}
static ActBwdReduceKernel act_bwd_reduce_kernel(int act) {
  return with_act(act, [](auto a) -> ActBwdReduceKernel { return bn_act::k_act_bwd_reduce<(Act) decltype(a)::value>; });
}
template <typename P>
static ActInferKernel<P> act_infer_kernel(int vec, int act) {
  return with_const<1, kEwVec>(vec, [&](auto v) {
    return with_act(act, [](auto a) -> ActInferKernel<P> { return bn_act::k_act_infer<decltype(v)::value, (Act) decltype(a)::value, P>; });
  });
}

// the kernels of a batch norm followed by a residual add, with or without stochastic depth (norm_res.cuh)
using bn_res::Res;
using ResTransformKernel = void (*)(const bf16*, const bf16*, const bf16*, bf16*, const float*, const float*, const float*, const float*,
                                    int, int, int);
using ResBwdReduceKernel = void (*)(const bf16*, const bf16*, const bf16*, const float*, const float*, float*, float*, float*, float*,
                                    volatile float*, int*, bf16*, int, int, int);
template <typename P>
using ResInferKernel = void (*)(const bf16*, const bf16*, bf16*, const P*, const P*, const P*, const P*, float, int, int);

static ResTransformKernel res_transform_kernel(int vec, bool drop) {
  return with_const<1, kEwVec>(vec, [&](auto v) -> ResTransformKernel {
    return drop ? bn_res::k_res_transform<decltype(v)::value, bn_res::kResDropAdd> : bn_res::k_res_transform<decltype(v)::value, bn_res::kResAdd>;
  });
}
static ResBwdReduceKernel res_bwd_reduce_kernel() { return bn_res::k_res_bwd_reduce; }
template <typename P>
static ResInferKernel<P> res_infer_kernel(int vec, bool add) {
  return with_const<1, kEwVec>(vec, [&](auto v) -> ResInferKernel<P> {
    return add ? bn_res::k_res_infer<decltype(v)::value, bn_res::kResAdd, P> : bn_res::k_res_infer<decltype(v)::value, bn_res::kResPlain, P>;
  });
}

// VGG's stage end (norm_pool2.cuh): the training and eval pooling kernels take 8 channels per thread or 1, the backward
// reduce kBwdVec or 1.
using Pool2FwdKernel = void (*)(const bf16*, bf16*, uint8_t*, const float*, const float*, const float*, const float*, bn_pool2::Dims,
                                int, int);
using Pool2BwdReduceKernel = void (*)(const bf16*, const bf16*, const uint8_t*, const float*, const float*, float*, float*, float*,
                                      float*, volatile float*, int*, bn_pool2::Dims, int, int);
using Pool2BwdElemtKernel = void (*)(const bf16*, const uint8_t*, const bf16*, bf16*, const float*, const float*, const float*,
                                     const float*, const float*, float, bn_pool2::Dims, int, int);
template <typename P>
using Pool2InferKernel = void (*)(const bf16*, bf16*, const P*, const P*, const P*, const P*, float, bn_pool2::Dims, int, int);

static Pool2FwdKernel pool2_fwd_kernel(int vec) {
  return with_const<1, kEwVec>(vec, [](auto v) -> Pool2FwdKernel { return bn_pool2::k_pool2_fwd<decltype(v)::value>; });
}
static Pool2BwdReduceKernel pool2_bwd_reduce_kernel(int vec) {
  return with_const<1, kBwdVec>(vec, [](auto v) -> Pool2BwdReduceKernel { return bn_pool2::k_pool2_bwd_reduce<decltype(v)::value>; });
}
static Pool2BwdElemtKernel pool2_bwd_elemt_kernel(int vec) {
  return with_const<1, kEwVec>(vec, [](auto v) -> Pool2BwdElemtKernel { return bn_pool2::k_pool2_bwd_elemt<decltype(v)::value>; });
}
template <typename P>
static Pool2InferKernel<P> pool2_infer_kernel(int vec) {
  return with_const<1, kEwVec>(vec, [](auto v) -> Pool2InferKernel<P> { return bn_pool2::k_pool2_infer<decltype(v)::value, P>; });
}

// Loads every batch-norm kernel into the context (b200coll.cu's load_kernels explains why a loopback world must not
// load a kernel lazily while a peer's collective waits): every key value goes through the functions above.
cudaError_t load_kernels() {
  cudaFuncAttributes attr;
  cudaError_t e = cudaSuccess;
  auto load = [&](auto kernel) { if (kernel && e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kernel); };
  load(&k_bn_sync_merge);
  load(res_bwd_reduce_kernel());
  load(&bn_cat::k_cat_stats);
  load(&bn_cat::k_cat_transform);
  load(&bn_cat::k_cat_bwd_reduce);
  load(&bn_cat::k_cat_bwd_elemt);
  load(&bn_cat::k_cat_infer<float>);
  load(&bn_cat::k_cat_infer<bf16>);
  load(&bn_slice::k_slice_transform);
  load(&bn_slice::k_slice_bwd_reduce);
  load(&bn_slice::k_slice_bwd_elemt);
  load(&bn_slice::k_slice_infer<float>);
  load(&bn_slice::k_slice_infer<bf16>);
  load(&bn_shuffle::k_shuffle_transform<false>);
  load(&bn_shuffle::k_shuffle_transform<true>);
  load(&bn_shuffle::k_shuffle_bwd_reduce<false>);
  load(&bn_shuffle::k_shuffle_bwd_reduce<true>);
  load(&bn_shuffle::k_shuffle_bwd_elemt<false>);
  load(&bn_shuffle::k_shuffle_bwd_elemt<true>);
  load(&bn_shuffle::k_shuffle_infer<false, float>);
  load(&bn_shuffle::k_shuffle_infer<true, float>);
  load(&bn_shuffle::k_shuffle_infer<false, bf16>);
  load(&bn_shuffle::k_shuffle_infer<true, bf16>);
  for (int vec : {1, kEwVec}) {
    load(pool2_fwd_kernel(vec));
    load(pool2_bwd_elemt_kernel(vec));
    load(pool2_infer_kernel<float>(vec));
    load(pool2_infer_kernel<bf16>(vec));
  }
  load(pool2_bwd_reduce_kernel(1));
  load(pool2_bwd_reduce_kernel(kBwdVec));
  for (int src = 0; src < kGradSrcs; src++) {
    load(bwd_reduce_kernel(src, false));
    load(bwd_reduce_kernel(src, true));
  }
  for (int vec : {1, kStatsVec, kEwVec}) {
    load(stats_kernel(vec));
    load(stats_dual_kernel(vec));
    load(sync_stats_kernel(vec));
    load(pool_fwd_kernel(vec));
    for (int tail = 0; tail < kTails; tail++) load(transform_kernel(vec, tail));
    for (int src = 0; src < kGradSrcs; src++)
      for (bool fct_ptr : {false, true})
        for (bool dual : {false, true}) load(bwd_elemt_kernel(vec, src, fct_ptr, dual));
    load(infer_pool_kernel<float>(vec));
    load(infer_pool_kernel<bf16>(vec));
    for (int tail = 0; tail < kTails; tail++) {
      load(infer_transform_kernel<float>(vec, tail));
      load(infer_transform_kernel<bf16>(vec, tail));
    }
    for (int act : {bn_act::kActRelu6, bn_act::kActSilu, bn_act::kActHardswish}) {
      if (vec == 1) load(act_bwd_reduce_kernel(act));
      load(act_transform_kernel(vec, act));
      load(act_infer_kernel<float>(vec, act));
      load(act_infer_kernel<bf16>(vec, act));
    }
    for (bool b : {false, true}) {
      load(res_transform_kernel(vec, b));
      load(res_infer_kernel<float>(vec, b));
      load(res_infer_kernel<bf16>(vec, b));
    }
  }
  return e;
}

// ---- launchers, shared by the local site and the sync phases ----
// Each returns the launch's error, or kNoKernel when the dispatch has no kernel for the site's keys.
constexpr cudaError_t kNoKernel = cudaErrorInvalidDeviceFunction;

// The statistics: with `sync_row` this rank's row for the allgather (k_bn_sync_stats), else the site's own save and
// running statistics (k_bn_stats).
static cudaError_t launch_stats(const FwdArgs& a, float* sync_row, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const int vec = vec_ok(a.c, &a.x, 1) ? kStatsVec : 1;
  block.x /= vec;
  const size_t smem = vec == kStatsVec ? stats_ring_bytes(block) : 0;
  const bf16* x = static_cast<const bf16*>(a.x);
  if (sync_row) {
    const SyncStatsKernel k = sync_stats_kernel(vec);
    if (!k) return kNoKernel;
    k<<<grid, block, smem, st>>>(x, sync_row, a.eps, s.staging, s.semaphores, a.m, a.c);
  } else {
    const StatsKernel k = stats_kernel(vec);
    if (!k) return kNoKernel;
    StatsOut o{a.save_mean, a.save_invstd, a.running_mean, a.running_var, a.num_batches_tracked, a.momentum,
               (float)((double)a.m / (double)(a.m - 1)), a.eps};
    k<<<grid, block, smem, st>>>(x, o, s.staging, s.semaphores, a.m, a.c);
  }
  return cudaGetLastError();
}

static cudaError_t launch_transform(const FwdArgs& a, cudaStream_t st) {
  const void* ptrs[3] = {a.x, a.y, a.identity ? a.identity : a.x};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const TransformKernel k = transform_kernel(vec, !a.relu ? kTailNone : a.identity ? kTailAddRelu : kTailRelu);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.identity), static_cast<bf16*>(a.y),
                            static_cast<uint8_t*>(a.mask), a.save_mean, a.save_invstd, a.weight, a.bias, nullptr, nullptr, nullptr,
                            nullptr, a.m, a.c);
  return cudaGetLastError();
}

static PoolDims pool_dims(int h, int w) { return PoolDims{h, w, (h - 1) / 2 + 1, (w - 1) / 2 + 1}; }

// The stem's pooling: one thread per pooled element and 8 (or 1) channels.
static cudaError_t launch_pool_fwd(const FwdArgs& a, cudaStream_t st) {
  const PoolDims d = pool_dims(a.pool_h, a.pool_w);
  const int pooled_rows = a.m / (a.pool_h * a.pool_w) * d.oh * d.ow;
  const void* ptrs[3] = {a.x, a.y, a.argmax};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(pooled_rows, a.c, vec, &block, &grid);
  const PoolFwdKernel k = pool_fwd_kernel(vec);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), static_cast<uint8_t*>(a.argmax), a.save_mean,
                            a.save_invstd, a.weight, a.bias, d, pooled_rows, a.c);
  return cudaGetLastError();
}

cudaError_t forward(const FwdArgs& a, cudaStream_t st) {
  const cudaError_t e = launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  return a.pool_h ? launch_pool_fwd(a, st) : launch_transform(a, st);
}

// Where a backward kernel takes g from.  The elementwise kernel runs after the reduce kernel (`reduced`), which at a
// residual site and at the stem has written g to dy_masked.
static GradSrc grad_src(const BwdArgs& a, bool reduced) {
  if (!a.relu) return kGradDy;
  if (reduced && a.dy_masked) return kGradMasked;
  if (a.pool_h) return kGradPool;
  return a.mask ? kGradBits : kGradY;
}

static cudaError_t launch_bwd_reduce(const BwdArgs& a, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  const GradSrc src = grad_src(a, false);
  const void* ptrs[5] = {a.x, a.dy, a.dy2 ? a.dy2 : a.dy, src == kGradY ? a.y : a.dy, a.dy_masked ? a.dy_masked : a.dy};
  const BwdReduceLaunch l = bwd_reduce_launch(a.m, a.c, src, a.dy2 != nullptr, false, ptrs, 5);
  const BwdReduceKernel k = bwd_reduce_kernel(src, false);
  if (!k) return kNoKernel;
  const void* mask = src == kGradPool ? a.argmax : a.mask;
  k<<<l.grid, l.block, l.smem, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.dy), static_cast<const bf16*>(a.dy2),
                            static_cast<const bf16*>(a.y), static_cast<const uint8_t*>(mask), static_cast<bf16*>(a.dy_masked),
                            a.save_mean, a.save_invstd, s.sums, s.sums + a.c, a.grad_weight, a.grad_bias, s.staging, s.semaphores,
                            pool_dims(a.pool_h, a.pool_w), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, a.m, a.c, l.vec);
  return cudaGetLastError();
}

// norm_fct is this call's (float)(1.0 / m) unless the site brings a pointer to its own (a sync site's).
static cudaError_t launch_bwd_elemt(const BwdArgs& a, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  const GradSrc src = grad_src(a, true);
  const void* g = src == kGradMasked ? a.dy_masked : a.dy;
  const void* ptrs[5] = {a.x, a.dx, g, a.dy2 && src != kGradMasked ? a.dy2 : a.dy, a.y};
  const int vec = vec_ok(a.c, ptrs, src == kGradY ? 5 : 4) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const BwdElemtKernel k = bwd_elemt_kernel(vec, src, a.norm_fct != nullptr, false);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(g), static_cast<const bf16*>(a.dy2), static_cast<const bf16*>(a.y),
                            static_cast<const uint8_t*>(a.mask), static_cast<const bf16*>(a.x), static_cast<bf16*>(a.dx), a.save_mean,
                            a.save_invstd, a.weight, s.sums, s.sums + a.c, a.norm_fct, (float)(1.0 / a.m), nullptr, nullptr, nullptr,
                            nullptr, nullptr, nullptr, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t backward(const BwdArgs& a, cudaStream_t st) {
  const cudaError_t e = launch_bwd_reduce(a, st);
  return e == cudaSuccess ? launch_bwd_elemt(a, st) : e;
}

// ---- a tail whose identity is a downsample branch's batch norm (two batch norms of one shape) ----
// The dual scratch is the local one followed by the second statistics plane's staging and the second batch norm's
// sum of g * (x - mean); the semaphores stay in the fixed region at the start, plane 1's after plane 0's, which is
// why a dual site takes at most kMaxChannels / 2 channels.
static size_t dual_extra_offset(int c) { return (scratch_bytes(c) + 15) / 16 * 16; }
size_t dual_scratch_bytes(int c) { return dual_extra_offset(c) + (size_t)3 * c * kMaxHBlock * 4 + (size_t)c * 4; }
static float* dual_staging(void* scratch, int c) { return reinterpret_cast<float*>(static_cast<char*>(scratch) + dual_extra_offset(c)); }
static float* dual_sum_xmu2(void* scratch, int c) { return dual_staging(scratch, c) + (size_t)3 * c * kMaxHBlock; }

// `a` is the tail's batch norm (y, mask), `b` the downsample branch's (its x, weight, bias, statistics); b's y and
// mask are unused.
// The statistics of both: k_bn_stats_dual, plane z taking k_bn_stats's launch shape for its own input.
static cudaError_t launch_stats_dual(const FwdArgs& a, const FwdArgs& b, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const void* xs[2] = {a.x, b.x};
  const int svec = vec_ok(a.c, xs, 2) ? kStatsVec : 1;
  block.x /= svec;
  grid.z = 2;
  const size_t smem = svec == kStatsVec ? stats_ring_bytes(block) : 0;
  const StatsDualKernel ks = stats_dual_kernel(svec);
  if (!ks) return kNoKernel;
  StatsOut oa{a.save_mean, a.save_invstd, a.running_mean, a.running_var, a.num_batches_tracked, a.momentum,
              (float)((double)a.m / (double)(a.m - 1)), a.eps};
  StatsOut ob{b.save_mean, b.save_invstd, b.running_mean, b.running_var, b.num_batches_tracked, b.momentum,
              (float)((double)b.m / (double)(b.m - 1)), b.eps};
  ks<<<grid, block, smem, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(b.x), oa, ob, s.staging,
                             dual_staging(a.scratch, a.c), s.semaphores, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t forward_dual(const FwdArgs& a, const FwdArgs& b, cudaStream_t st) {
  const cudaError_t e = launch_stats_dual(a, b, st);
  if (e != cudaSuccess) return e;
  dim3 block, grid;
  const void* ptrs[3] = {a.x, a.y, b.x};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  ew_config(a.m, a.c, vec, &block, &grid);
  const TransformKernel kt = transform_kernel(vec, kTailBnAddRelu);
  if (!kt) return kNoKernel;
  kt<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(b.x), static_cast<bf16*>(a.y),
                             static_cast<uint8_t*>(a.mask), a.save_mean, a.save_invstd, a.weight, a.bias, b.save_mean, b.save_invstd,
                             b.weight, b.bias, a.m, a.c);
  return cudaGetLastError();
}

// `a` is the tail's batch norm (dy, dy2, y or mask, x, dx), `b` the downsample branch's (x, dx, weight, statistics,
// grad_weight, grad_bias).  Neither writes g: the elementwise kernel derives it again.
cudaError_t backward_dual(const BwdArgs& a, const BwdArgs& b, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  float* sum2 = dual_sum_xmu2(a.scratch, a.c);
  const GradSrc src = a.mask ? kGradBits : kGradY;
  const void* rptrs[5] = {a.x, a.dy, a.dy2 ? a.dy2 : a.dy, src == kGradY ? a.y : a.dy, b.x};
  const BwdReduceLaunch l = bwd_reduce_launch(a.m, a.c, src, a.dy2 != nullptr, true, rptrs, 5);
  const BwdReduceKernel kr = bwd_reduce_kernel(src, true);
  if (!kr) return kNoKernel;
  kr<<<l.grid, l.block, l.smem, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.dy), static_cast<const bf16*>(a.dy2),
                             static_cast<const bf16*>(a.y), static_cast<const uint8_t*>(a.mask), nullptr, a.save_mean, a.save_invstd,
                             s.sums, s.sums + a.c, a.grad_weight, a.grad_bias, s.staging, s.semaphores, pool_dims(0, 0),
                             static_cast<const bf16*>(b.x), b.save_mean, b.save_invstd, sum2, b.grad_weight, b.grad_bias, a.m, a.c, l.vec);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const void* ptrs[7] = {a.x, a.dx, a.dy, a.dy2 ? a.dy2 : a.dy, b.x, b.dx, a.y};
  const int vec = vec_ok(a.c, ptrs, src == kGradY ? 7 : 6) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const BwdElemtKernel ke = bwd_elemt_kernel(vec, src, false, true);
  if (!ke) return kNoKernel;
  ke<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.dy), static_cast<const bf16*>(a.dy2), static_cast<const bf16*>(a.y),
                             static_cast<const uint8_t*>(a.mask), static_cast<const bf16*>(a.x), static_cast<bf16*>(a.dx), a.save_mean,
                             a.save_invstd, a.weight, s.sums, s.sums + a.c, nullptr, (float)(1.0 / a.m), static_cast<const bf16*>(b.x),
                             static_cast<bf16*>(b.dx), b.save_mean, b.save_invstd, b.weight, sum2, a.m, a.c);
  return cudaGetLastError();
}

// ---- eval mode: one kernel per site, launched as the training transform / pool kernels are ----
template <typename P>
static cudaError_t launch_infer(const InferArgs& a, cudaStream_t st) {
  auto p = [](const void* q) { return static_cast<const P*>(q); };
  const bf16* x = static_cast<const bf16*>(a.x);
  bf16* y = static_cast<bf16*>(a.y);
  const InferParams& b = a.bn;
  dim3 block, grid;
  if (a.pool_h) {
    const PoolDims d = pool_dims(a.pool_h, a.pool_w);
    const int pooled_rows = a.m / (a.pool_h * a.pool_w) * d.oh * d.ow;
    const void* ptrs[2] = {a.x, a.y};
    const int vec = vec_ok(a.c, ptrs, 2) ? kEwVec : 1;
    ew_config(pooled_rows, a.c, vec, &block, &grid);
    const InferPoolKernel<P> k = infer_pool_kernel<P>(vec);
    if (!k) return kNoKernel;
    k<<<grid, block, 0, st>>>(x, y, p(b.running_mean), p(b.running_var), p(b.weight), p(b.bias), b.eps, d, pooled_rows, a.c);
    return cudaGetLastError();
  }
  const void* ptrs[3] = {a.x, a.y, a.identity ? a.identity : a.x};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  ew_config(a.m, a.c, vec, &block, &grid);
  const InferTransformKernel<P> k = infer_transform_kernel<P>(vec, a.dual ? kTailBnAddRelu : a.identity ? kTailAddRelu : kTailRelu);
  if (!k) return kNoKernel;
  const InferParams& ds = a.ds;
  k<<<grid, block, 0, st>>>(x, static_cast<const bf16*>(a.identity), y, p(b.running_mean), p(b.running_var), p(b.weight), p(b.bias), b.eps,
                            p(ds.running_mean), p(ds.running_var), p(ds.weight), p(ds.bias), ds.eps, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t infer(const InferArgs& a, cudaStream_t st) { return a.param_bf16 ? launch_infer<bf16>(a, st) : launch_infer<float>(a, st); }

// dx of a local site from a g that is already in memory (the one a reduce kernel wrote, or dy itself where g = dy):
// k_bn_bwd_elemt reads it as kGradMasked, with this call's norm_fct = (float)(1.0 / m).
static cudaError_t launch_elemt_of(const BwdArgs& a, const bf16* g, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  const void* ptrs[3] = {a.x, a.dx, g};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const BwdElemtKernel ke = bwd_elemt_kernel(vec, kGradMasked, false, false);
  if (!ke) return kNoKernel;
  ke<<<grid, block, 0, st>>>(g, nullptr, nullptr, nullptr, static_cast<const bf16*>(a.x), static_cast<bf16*>(a.dx), a.save_mean,
                             a.save_invstd, a.weight, s.sums, s.sums + a.c, nullptr, (float)(1.0 / a.m), nullptr, nullptr, nullptr,
                             nullptr, nullptr, nullptr, a.m, a.c);
  return cudaGetLastError();
}

// ---- batch norm followed by ReLU6, SiLU or Hardswish ----
// The statistics are the local site's (k_bn_stats); the transform, like k_bn_transform, then writes act(t).
cudaError_t forward_act(const FwdArgs& a, int act, cudaStream_t st) {
  const cudaError_t e = launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  const void* ptrs[2] = {a.x, a.y};
  const int vec = vec_ok(a.c, ptrs, 2) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const ActTransformKernel k = act_transform_kernel(vec, act);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), a.save_mean, a.save_invstd, a.weight, a.bias, a.m, a.c);
  return cudaGetLastError();
}

// The reduce recomputes t, derives g from dy and writes it to a.dy_masked, with k_bn_bwd_reduce's launch shape; the
// local site's elementwise kernel then reads g (kGradMasked) with this call's norm_fct = (float)(1.0 / m).
cudaError_t backward_act(const BwdArgs& a, const float* bias, int act, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const ActBwdReduceKernel kr = act_bwd_reduce_kernel(act);
  if (!kr) return kNoKernel;
  const bf16* x = static_cast<const bf16*>(a.x);
  bf16* g = static_cast<bf16*>(a.dy_masked);
  kr<<<grid, block, 0, st>>>(x, static_cast<const bf16*>(a.dy), a.save_mean, a.save_invstd, a.weight, bias, s.sums, s.sums + a.c,
                             a.grad_weight, a.grad_bias, s.staging, s.semaphores, g, a.m, a.c);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_elemt_of(a, g, st);
}

template <typename P>
static cudaError_t launch_infer_act(const InferArgs& a, int act, cudaStream_t st) {
  const void* ptrs[2] = {a.x, a.y};
  const int vec = vec_ok(a.c, ptrs, 2) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const ActInferKernel<P> k = act_infer_kernel<P>(vec, act);
  if (!k) return kNoKernel;
  const InferParams& b = a.bn;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), static_cast<const P*>(b.running_mean),
                            static_cast<const P*>(b.running_var), static_cast<const P*>(b.weight), static_cast<const P*>(b.bias), b.eps,
                            a.m, a.c);
  return cudaGetLastError();
}

cudaError_t infer_act(const InferArgs& a, int act, cudaStream_t st) {
  return a.param_bf16 ? launch_infer_act<bf16>(a, act, st) : launch_infer_act<float>(a, act, st);
}

// ---- batch norm followed by a residual add, with or without stochastic depth ----
// The statistics are the local site's (k_bn_stats).  Without an identity the transform is k_bn_transform<V, kTailNone>.
cudaError_t forward_res(const FwdArgs& a, const void* noise, int rows_per_sample, cudaStream_t st) {
  if (!a.identity) return forward(a, st);
  const cudaError_t e = launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  const void* ptrs[3] = {a.x, a.y, a.identity};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const ResTransformKernel k = res_transform_kernel(vec, noise != nullptr);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.identity), static_cast<const bf16*>(noise),
                            static_cast<bf16*>(a.y), a.save_mean, a.save_invstd, a.weight, a.bias, rows_per_sample, a.m, a.c);
  return cudaGetLastError();
}

// Without noise g = dy: k_bn_bwd_reduce<kGradDy, false> sums dy, and the elementwise kernel reads dy as its g.  With
// noise the reduce derives g = bf16(dy * noise[n]) and writes it to a.dy_masked for the elementwise kernel.
cudaError_t backward_res(const BwdArgs& a, const void* noise, int rows_per_sample, cudaStream_t st) {
  if (!noise) {
    const cudaError_t e = launch_bwd_reduce(a, st);
    return e == cudaSuccess ? launch_elemt_of(a, static_cast<const bf16*>(a.dy), st) : e;
  }
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const ResBwdReduceKernel kr = res_bwd_reduce_kernel();
  bf16* g = static_cast<bf16*>(a.dy_masked);
  kr<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.dy), static_cast<const bf16*>(noise), a.save_mean,
                             a.save_invstd, s.sums, s.sums + a.c, a.grad_weight, a.grad_bias, s.staging, s.semaphores, g, rows_per_sample,
                             a.m, a.c);
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? launch_elemt_of(a, g, st) : e;
}

template <typename P>
static cudaError_t launch_infer_res(const InferArgs& a, cudaStream_t st) {
  const void* ptrs[3] = {a.x, a.y, a.identity ? a.identity : a.x};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const ResInferKernel<P> k = res_infer_kernel<P>(vec, a.identity != nullptr);
  if (!k) return kNoKernel;
  const InferParams& b = a.bn;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.identity), static_cast<bf16*>(a.y),
                            static_cast<const P*>(b.running_mean), static_cast<const P*>(b.running_var), static_cast<const P*>(b.weight),
                            static_cast<const P*>(b.bias), b.eps, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t infer_res(const InferArgs& a, cudaStream_t st) { return a.param_bf16 ? launch_infer_res<bf16>(a, st) : launch_infer_res<float>(a, st); }

// ---- sync batch norm ----
// The sync scratch is the local one followed, from a 16-byte boundary, by W + 1 rows of [mean | invstd | count]:
// this rank's row (the allgather's input) and the W gathered ones.  The backward's 2C sums are the local layout's.
static size_t sync_row_floats(int c) { return ((size_t)2 * c + 1 + 3) / 4 * 4; }
static size_t sync_rows_offset(int c) { return (scratch_bytes(c) + 15) / 16 * 16; }

size_t sync_scratch_bytes(int c, int world) { return sync_rows_offset(c) + (size_t)(world + 1) * sync_row_floats(c) * 4; }

SyncRows sync_rows(void* scratch, int c) {
  SyncRows r;
  r.row_floats = sync_row_floats(c);
  r.local = reinterpret_cast<float*>(static_cast<char*>(scratch) + sync_rows_offset(c));
  r.gathered = r.local + r.row_floats;
  r.sums = carve(scratch, c).sums;
  return r;
}

cudaError_t sync_stats(const FwdArgs& a, cudaStream_t st) {
  SyncRows r = sync_rows(a.scratch, a.c);
  // an empty rank still sends a row: zeros, count 0, which every rank's merge skips
  if (a.m == 0) return cudaMemsetAsync(r.local, 0, ((size_t)2 * a.c + 1) * 4, st);
  return launch_stats(a, r.local, st);
}

cudaError_t sync_apply(const FwdArgs& a, int world, float* norm_fct, cudaStream_t st) {
  SyncRows r = sync_rows(a.scratch, a.c);
  k_bn_sync_merge<<<ceil_div(a.c, kEwThreads), kEwThreads, 0, st>>>(r.gathered, (int)r.row_floats, world, a.save_mean, a.save_invstd,
                                                                    norm_fct, a.running_mean, a.running_var, a.num_batches_tracked,
                                                                    a.momentum, a.eps, a.c);
  return a.m == 0 ? cudaGetLastError() : launch_transform(a, st);
}

cudaError_t sync_bwd_reduce(const BwdArgs& a, cudaStream_t st) {
  if (a.m == 0) {
    // nothing to sum: zero sums for the allreduce, zero dweight and dbias
    cudaMemsetAsync(carve(a.scratch, a.c).sums, 0, (size_t)2 * a.c * 4, st);
    cudaMemsetAsync(a.grad_weight, 0, (size_t)a.c * 4, st);
    cudaMemsetAsync(a.grad_bias, 0, (size_t)a.c * 4, st);
    return cudaGetLastError();
  }
  return launch_bwd_reduce(a, st);
}

cudaError_t sync_bwd_elemt(const BwdArgs& a, cudaStream_t st) { return a.m == 0 ? cudaSuccess : launch_bwd_elemt(a, st); }

// ---- batch norm and ReLU over a channel concatenation (norm_cat.cuh) ----
// Each launch takes its bn:: counterpart's vector launch shape for the concatenation's m and c: the caller has
// checked every segment (C_s % 8 == 0, 16-byte grid) and the outputs onto the 16-byte grid, which is what vec_ok
// decides for a tensor of c % 8 == 0.
static bn_cat::CatSegs cat_segs(const CatSegments& in) {
  bn_cat::CatSegs t{};
  int c = 0;
  for (int s = 0; s < in.n; s++) {
    t.ptr[s] = static_cast<const bf16*>(in.ptrs[s]);
    t.c0[s] = c;
    c += in.channels[s];
  }
  t.c0[in.n] = c;
  t.n = in.n;
  return t;
}

cudaError_t forward_cat(const CatSegments& in, const FwdArgs& a, cudaStream_t st) {
  const bn_cat::CatSegs segs = cat_segs(in);
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  block.x /= kStatsVec;
  StatsOut o{a.save_mean, a.save_invstd, a.running_mean, a.running_var, a.num_batches_tracked, a.momentum,
             (float)((double)a.m / (double)(a.m - 1)), a.eps};
  bn_cat::k_cat_stats<<<grid, block, stats_ring_bytes(block), st>>>(segs, o, s.staging, s.semaphores, a.m, a.c);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  bn_cat::k_cat_transform<<<grid, block, 0, st>>>(segs, static_cast<bf16*>(a.y), static_cast<uint8_t*>(a.mask), a.save_mean,
                                                  a.save_invstd, a.weight, a.bias, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t backward_cat(const CatSegments& in, const BwdArgs& a, cudaStream_t st) {
  const bn_cat::CatSegs segs = cat_segs(in);
  Scratch s = carve(a.scratch, a.c);
  const void* ptrs[1] = {a.dy};
  const BwdReduceLaunch l = bwd_reduce_launch(a.m, a.c, kGradBits, false, false, ptrs, 1);
  if (l.vec != kBwdVec) return kNoKernel;
  bn_cat::k_cat_bwd_reduce<<<l.grid, l.block, l.smem, st>>>(segs, static_cast<const bf16*>(a.dy), static_cast<const uint8_t*>(a.mask),
                                                            a.save_mean, a.save_invstd, s.sums, s.sums + a.c, a.grad_weight,
                                                            a.grad_bias, s.staging, s.semaphores, a.m, a.c);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  dim3 block, grid;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  bn_cat::k_cat_bwd_elemt<<<grid, block, 0, st>>>(segs, static_cast<const bf16*>(a.dy), static_cast<const uint8_t*>(a.mask),
                                                  static_cast<bf16*>(a.dx), a.save_mean, a.save_invstd, a.weight, s.sums, s.sums + a.c,
                                                  (float)(1.0 / a.m), a.m, a.c);
  return cudaGetLastError();
}

template <typename P>
static cudaError_t launch_infer_cat(const CatSegments& in, const InferArgs& a, cudaStream_t st) {
  dim3 block, grid;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  const InferParams& b = a.bn;
  bn_cat::k_cat_infer<P><<<grid, block, 0, st>>>(cat_segs(in), static_cast<bf16*>(a.y), static_cast<const P*>(b.running_mean),
                                                 static_cast<const P*>(b.running_var), static_cast<const P*>(b.weight),
                                                 static_cast<const P*>(b.bias), b.eps, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t infer_cat(const CatSegments& in, const InferArgs& a, cudaStream_t st) {
  return a.param_bf16 ? launch_infer_cat<bf16>(in, a, st) : launch_infer_cat<float>(in, a, st);
}

// ---- batch norm and ReLU into a channel slice of a wider output (norm_slice.cuh) ----
// The statistics are the local site's (k_bn_stats on x); every other launch takes its bn:: counterpart's vector launch
// shape for the branch's m and c: the caller has checked C % 8 == 0 and x, y, dy and dx onto the 16-byte grid, which
// is what vec_ok decides for a tensor of c % 8 == 0.
cudaError_t forward_slice(const FwdArgs& a, int ldy, cudaStream_t st) {
  const cudaError_t e = launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  dim3 block, grid;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  bn_slice::k_slice_transform<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), ldy,
                                                      static_cast<uint8_t*>(a.mask), a.save_mean, a.save_invstd, a.weight, a.bias,
                                                      a.m, a.c);
  return cudaGetLastError();
}

cudaError_t backward_slice(const BwdArgs& a, int lddy, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  const void* ptrs[2] = {a.x, a.dy};
  const BwdReduceLaunch l = bwd_reduce_launch(a.m, a.c, kGradBits, false, false, ptrs, 2);
  if (l.vec != kBwdVec) return kNoKernel;
  bn_slice::k_slice_bwd_reduce<<<l.grid, l.block, l.smem, st>>>(static_cast<const bf16*>(a.x), static_cast<const bf16*>(a.dy), lddy,
                                                                static_cast<const uint8_t*>(a.mask), a.save_mean, a.save_invstd, s.sums,
                                                                s.sums + a.c, a.grad_weight, a.grad_bias, s.staging, s.semaphores, a.m,
                                                                a.c);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  dim3 block, grid;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  bn_slice::k_slice_bwd_elemt<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.dy), lddy, static_cast<const uint8_t*>(a.mask),
                                                      static_cast<const bf16*>(a.x), static_cast<bf16*>(a.dx), a.save_mean, a.save_invstd,
                                                      a.weight, s.sums, s.sums + a.c, (float)(1.0 / a.m), a.m, a.c);
  return cudaGetLastError();
}

template <typename P>
static cudaError_t launch_infer_slice(const InferArgs& a, int ldy, cudaStream_t st) {
  dim3 block, grid;
  ew_config(a.m, a.c, kEwVec, &block, &grid);
  const InferParams& b = a.bn;
  bn_slice::k_slice_infer<P><<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), ldy,
                                                     static_cast<const P*>(b.running_mean), static_cast<const P*>(b.running_var),
                                                     static_cast<const P*>(b.weight), static_cast<const P*>(b.bias), b.eps, a.m, a.c);
  return cudaGetLastError();
}

cudaError_t infer_slice(const InferArgs& a, int ldy, cudaStream_t st) {
  return a.param_bf16 ? launch_infer_slice<bf16>(a, ldy, st) : launch_infer_slice<float>(a, ldy, st);
}

// ---- ShuffleNetV2's block end (norm_shuffle.cuh) ----
// The statistics are the local site's (k_bn_stats on t) or, with u, k_bn_stats_dual on (t, u) in the dual scratch;
// the transform and eval launches cover the [m][B] rows with kTile x kTile tiles; the backward reduce takes
// reduce_config's launch for [m][B] and the elementwise kernel ew_config's with one channel per thread.
size_t shuffle_mask_bytes(int m, int c) { return (size_t)m * bn_shuffle::mask_row_bytes(c); }

static dim3 shuffle_tiles(int m, int c) { return dim3(ceil_div(m, bn_shuffle::kTile), ceil_div(c, bn_shuffle::kTile), 1); }

cudaError_t forward_shuffle(const FwdArgs& a, const FwdArgs* b, const void* x1, int x1_stride, int hw, cudaStream_t st) {
  const cudaError_t e = b ? launch_stats_dual(a, *b, st) : launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  const bn_shuffle::Geometry g{a.m, a.c, hw, static_cast<const bf16*>(x1), x1_stride};
  const bn_shuffle::SavedStats sa{a.save_mean, a.save_invstd, a.weight, a.bias};
  const bf16* t = static_cast<const bf16*>(a.x);
  bf16* y = static_cast<bf16*>(a.y);
  uint8_t* mask = static_cast<uint8_t*>(a.mask);
  if (b) {
    const bn_shuffle::SavedStats sb{b->save_mean, b->save_invstd, b->weight, b->bias};
    bn_shuffle::k_shuffle_transform<true><<<shuffle_tiles(a.m, a.c), kEwThreads, 0, st>>>(t, static_cast<const bf16*>(b->x), y, mask,
                                                                                           static_cast<uint8_t*>(b->mask), sa, sb, g);
  } else {
    bn_shuffle::k_shuffle_transform<false><<<shuffle_tiles(a.m, a.c), kEwThreads, 0, st>>>(t, nullptr, y, mask, nullptr, sa, sa, g);
  }
  return cudaGetLastError();
}

// t's sums go to the local layout (grad_bias holds Σg, sums + c Σg(x - mean)), u's to the dual scratch's second
// staging plane and its sum_xmu2; both backward kernels read dy from a.dy.
cudaError_t backward_shuffle(const BwdArgs& a, const BwdArgs* b, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  auto site = [](const BwdArgs& x, float* sum_xmu, float* staging) {
    return bn_shuffle::BwdSite{static_cast<const bf16*>(x.x), static_cast<const uint8_t*>(x.mask), x.save_mean, x.save_invstd, x.weight,
                               x.grad_weight, x.grad_bias, sum_xmu, staging, static_cast<bf16*>(x.dx)};
  };
  const bn_shuffle::BwdSite sa = site(a, s.sums + a.c, s.staging);
  const bn_shuffle::BwdSite sb = b ? site(*b, dual_sum_xmu2(a.scratch, a.c), dual_staging(a.scratch, a.c)) : sa;
  const bf16* dy = static_cast<const bf16*>(a.dy);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  if (b) bn_shuffle::k_shuffle_bwd_reduce<true><<<grid, block, 0, st>>>(dy, sa, sb, s.semaphores, a.m, a.c);
  else bn_shuffle::k_shuffle_bwd_reduce<false><<<grid, block, 0, st>>>(dy, sa, sb, s.semaphores, a.m, a.c);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  ew_config(a.m, a.c, 1, &block, &grid);
  const float norm_fct = (float)(1.0 / a.m);
  if (b) bn_shuffle::k_shuffle_bwd_elemt<true><<<grid, block, 0, st>>>(dy, sa, sb, norm_fct, a.m, a.c);
  else bn_shuffle::k_shuffle_bwd_elemt<false><<<grid, block, 0, st>>>(dy, sa, sb, norm_fct, a.m, a.c);
  return cudaGetLastError();
}

template <typename P>
static cudaError_t launch_infer_shuffle(const InferArgs& a, const void* x1, int x1_stride, int hw, cudaStream_t st) {
  auto stats = [](const InferParams& q) {
    return bn_shuffle::RunningStats<P>{static_cast<const P*>(q.running_mean), static_cast<const P*>(q.running_var),
                                       static_cast<const P*>(q.weight), static_cast<const P*>(q.bias), q.eps};
  };
  const bn_shuffle::Geometry g{a.m, a.c, hw, static_cast<const bf16*>(x1), x1_stride};
  const bn_shuffle::RunningStats<P> sa = stats(a.bn);
  const bf16* t = static_cast<const bf16*>(a.x);
  bf16* y = static_cast<bf16*>(a.y);
  if (a.dual)
    bn_shuffle::k_shuffle_infer<true, P><<<shuffle_tiles(a.m, a.c), kEwThreads, 0, st>>>(t, static_cast<const bf16*>(a.identity), y, sa,
                                                                                          stats(a.ds), g);
  else
    bn_shuffle::k_shuffle_infer<false, P><<<shuffle_tiles(a.m, a.c), kEwThreads, 0, st>>>(t, nullptr, y, sa, sa, g);
  return cudaGetLastError();
}

cudaError_t infer_shuffle(const InferArgs& a, const void* x1, int x1_stride, int hw, cudaStream_t st) {
  return a.param_bf16 ? launch_infer_shuffle<bf16>(a, x1, x1_stride, hw, st) : launch_infer_shuffle<float>(a, x1, x1_stride, hw, st);
}

// ---- VGG's stage end (norm_pool2.cuh) ----
// The statistics are launch_stats'.  The pooling kernels run one thread per pooled row and 8 (or 1) channels, the
// backward reduce reduce_config's launch for [m][C] with kBwdVec (or 1) channels per hardware thread, and the backward
// elementwise kernel ew_config's launch for [m][C].
static bn_pool2::Dims pool2_dims(int h, int w) { return bn_pool2::Dims{h, w, h / 2, w / 2}; }
static int pool2_rows(int m, int h, int w) { return m / (h * w) * (h / 2) * (w / 2); }

cudaError_t forward_pool2(const FwdArgs& a, cudaStream_t st) {
  cudaError_t e = launch_stats(a, nullptr, st);
  if (e != cudaSuccess) return e;
  const int rows = pool2_rows(a.m, a.pool_h, a.pool_w);
  const void* ptrs[3] = {a.x, a.y, a.argmax};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(rows, a.c, vec, &block, &grid);
  const Pool2FwdKernel k = pool2_fwd_kernel(vec);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), static_cast<uint8_t*>(a.argmax), a.save_mean,
                            a.save_invstd, a.weight, a.bias, pool2_dims(a.pool_h, a.pool_w), rows, a.c);
  return cudaGetLastError();
}

cudaError_t backward_pool2(const BwdArgs& a, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  const bn_pool2::Dims d = pool2_dims(a.pool_h, a.pool_w);
  const bf16* dy = static_cast<const bf16*>(a.dy);
  const bf16* x = static_cast<const bf16*>(a.x);
  const uint8_t* argmax = static_cast<const uint8_t*>(a.argmax);
  const void* ptrs[4] = {a.x, a.dy, a.argmax, a.dx};
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const int rvec = vec_ok(a.c, ptrs, 3) ? kBwdVec : 1;
  block.x /= rvec;
  const Pool2BwdReduceKernel r = pool2_bwd_reduce_kernel(rvec);
  if (!r) return kNoKernel;
  r<<<grid, block, 0, st>>>(x, dy, argmax, a.save_mean, a.save_invstd, s.sums, s.sums + a.c, a.grad_weight, a.grad_bias, s.staging,
                            s.semaphores, d, a.m, a.c);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  const int vec = vec_ok(a.c, ptrs, 4) ? kEwVec : 1;
  ew_config(a.m, a.c, vec, &block, &grid);
  const Pool2BwdElemtKernel k = pool2_bwd_elemt_kernel(vec);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(dy, argmax, x, static_cast<bf16*>(a.dx), a.save_mean, a.save_invstd, a.weight, s.sums, s.sums + a.c,
                            (float)(1.0 / a.m), d, a.m, a.c);
  return cudaGetLastError();
}

template <typename P>
static cudaError_t launch_infer_pool2(const InferArgs& a, cudaStream_t st) {
  auto p = [](const void* q) { return static_cast<const P*>(q); };
  const InferParams& b = a.bn;
  const int rows = pool2_rows(a.m, a.pool_h, a.pool_w);
  const void* ptrs[2] = {a.x, a.y};
  const int vec = vec_ok(a.c, ptrs, 2) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(rows, a.c, vec, &block, &grid);
  const Pool2InferKernel<P> k = pool2_infer_kernel<P>(vec);
  if (!k) return kNoKernel;
  k<<<grid, block, 0, st>>>(static_cast<const bf16*>(a.x), static_cast<bf16*>(a.y), p(b.running_mean), p(b.running_var), p(b.weight),
                            p(b.bias), b.eps, pool2_dims(a.pool_h, a.pool_w), rows, a.c);
  return cudaGetLastError();
}

cudaError_t infer_pool2(const InferArgs& a, cudaStream_t st) {
  return a.param_bf16 ? launch_infer_pool2<bf16>(a, st) : launch_infer_pool2<float>(a, st);
}

}  // namespace bn
}  // namespace b200c
