// Launchers of the fused batch-norm kernels (norm_kernels.cuh); argument checking lives in b200coll.cu.
#include <algorithm>

#include "norm_kernels.cuh"
#include "norm_launch.h"

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

// The transform after the statistics: k_bn_transform (ReLU, optionally after `+= identity`) or, without relu,
// k_bn_sync_transform.
static void launch_transform(const FwdArgs& a, bool relu, cudaStream_t st) {
  const void* ptrs[3] = {a.x, a.y, a.identity ? a.identity : a.x};
  const int vec = vec_ok(a.c, ptrs, 3) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  const bf16* x = static_cast<const bf16*>(a.x);
  const bf16* id = static_cast<const bf16*>(a.identity);
  bf16* y = static_cast<bf16*>(a.y);
  uint8_t* mask = static_cast<uint8_t*>(a.mask);
  if (!relu) {
    if (vec == kEwVec) k_bn_sync_transform<kEwVec><<<grid, block, 0, st>>>(x, y, a.save_mean, a.save_invstd, a.weight, a.bias, a.m, a.c);
    else k_bn_sync_transform<1><<<grid, block, 0, st>>>(x, y, a.save_mean, a.save_invstd, a.weight, a.bias, a.m, a.c);
    return;
  }
#define B200C_BN_TRANSFORM(V, R) \
  k_bn_transform<V, R><<<grid, block, 0, st>>>(x, id, y, mask, a.save_mean, a.save_invstd, a.weight, a.bias, a.m, a.c)
  if (vec == kEwVec) {
    if (id) B200C_BN_TRANSFORM(kEwVec, true); else B200C_BN_TRANSFORM(kEwVec, false);
  } else {
    if (id) B200C_BN_TRANSFORM(1, true); else B200C_BN_TRANSFORM(1, false);
  }
#undef B200C_BN_TRANSFORM
}

cudaError_t forward(const FwdArgs& a, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  StatsOut o{a.save_mean, a.save_invstd, a.running_mean, a.running_var, a.num_batches_tracked, a.momentum,
             (float)((double)a.m / (double)(a.m - 1)), a.eps};
  const bf16* x = static_cast<const bf16*>(a.x);
  if (vec_ok(a.c, &a.x, 1)) {
    k_bn_stats<kStatsVec><<<grid, dim3(block.x / kStatsVec, block.y), 0, st>>>(x, o, s.staging, s.semaphores, a.m, a.c);
  } else {
    k_bn_stats<1><<<grid, block, 0, st>>>(x, o, s.staging, s.semaphores, a.m, a.c);
  }
  launch_transform(a, true, st);
  return cudaGetLastError();
}

// The reduce kernel for g from dy and the ReLU's mask or output, or (relu false) g = dy.
static void launch_bwd_reduce(const BwdArgs& a, bool relu, float* sum_dy, float* sum_dy_xmu, const Scratch& s, cudaStream_t st) {
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const bf16* x = static_cast<const bf16*>(a.x);
  const bf16* dy = static_cast<const bf16*>(a.dy);
  const bf16* dy2 = static_cast<const bf16*>(a.dy2);
  const bf16* y = static_cast<const bf16*>(a.y);
  const uint8_t* mask = static_cast<const uint8_t*>(a.mask);
  bf16* masked = static_cast<bf16*>(a.dy_masked);
  if (!relu)
    k_bn_sync_bwd_reduce<<<grid, block, 0, st>>>(x, dy, dy2, y, mask, masked, a.save_mean, a.save_invstd, sum_dy, sum_dy_xmu,
                                                 a.grad_weight, a.grad_bias, s.staging, s.semaphores, a.m, a.c);
  else if (mask)
    k_bn_bwd_reduce<true><<<grid, block, 0, st>>>(x, dy, dy2, y, mask, masked, a.save_mean, a.save_invstd, sum_dy, sum_dy_xmu,
                                                  a.grad_weight, a.grad_bias, s.staging, s.semaphores, a.m, a.c);
  else
    k_bn_bwd_reduce<false><<<grid, block, 0, st>>>(x, dy, dy2, y, mask, masked, a.save_mean, a.save_invstd, sum_dy, sum_dy_xmu,
                                                   a.grad_weight, a.grad_bias, s.staging, s.semaphores, a.m, a.c);
}

// The elementwise kernel after the reduce: k_bn_bwd_elemt with a norm_fct value, or with norm_fct_ptr set
// k_bn_sync_bwd_elemt, which reads it from the device.
static void launch_bwd_elemt(const BwdArgs& a, bool relu, const float* sum_dy, const float* sum_dy_xmu, float norm_fct,
                             const float* norm_fct_ptr, cudaStream_t st) {
  const bf16* x = static_cast<const bf16*>(a.x);
  const bf16* dy = static_cast<const bf16*>(a.dy);
  const bf16* dy2 = static_cast<const bf16*>(a.dy2);
  const bf16* y = static_cast<const bf16*>(a.y);
  const uint8_t* mask = static_cast<const uint8_t*>(a.mask);
  const bf16* masked = static_cast<const bf16*>(a.dy_masked);
  // g comes from the tensor the reduce kernel wrote (tail), else from dy and the mask or y, or is dy (no ReLU)
  const GradSrc src = !relu ? kGradDy : masked ? kGradMasked : mask ? kGradBits : kGradY;
  const void* ptrs[5] = {a.x, a.dx, masked ? a.dy_masked : a.dy, dy2 && !masked ? a.dy2 : a.dy, a.y};
  const int vec = vec_ok(a.c, ptrs, src == kGradY ? 5 : 4) ? kEwVec : 1;
  dim3 block, grid;
  ew_config(a.m, a.c, vec, &block, &grid);
  bf16* dx = static_cast<bf16*>(a.dx);
#define B200C_BN_ELEMT(V, S, G)                                                                                               \
  if (norm_fct_ptr)                                                                                                          \
    k_bn_sync_bwd_elemt<V, S><<<grid, block, 0, st>>>(G, dy2, y, mask, x, dx, a.save_mean, a.save_invstd, a.weight, sum_dy,  \
                                                      sum_dy_xmu, norm_fct_ptr, a.m, a.c);                                   \
  else                                                                                                                       \
    k_bn_bwd_elemt<V, S><<<grid, block, 0, st>>>(G, dy2, y, mask, x, dx, a.save_mean, a.save_invstd, a.weight, sum_dy,       \
                                                 sum_dy_xmu, norm_fct, a.m, a.c);
#define B200C_BN_ELEMT_SRC(V)                                    \
  if (src == kGradMasked) { B200C_BN_ELEMT(V, kGradMasked, masked) } \
  else if (src == kGradBits) { B200C_BN_ELEMT(V, kGradBits, dy) }    \
  else if (src == kGradY) { B200C_BN_ELEMT(V, kGradY, dy) }          \
  else if (norm_fct_ptr) { k_bn_sync_bwd_elemt<V, kGradDy><<<grid, block, 0, st>>>(dy, dy2, y, mask, x, dx, a.save_mean, \
                             a.save_invstd, a.weight, sum_dy, sum_dy_xmu, norm_fct_ptr, a.m, a.c); }
  if (vec == kEwVec) {
    B200C_BN_ELEMT_SRC(kEwVec)
  } else {
    B200C_BN_ELEMT_SRC(1)
  }
#undef B200C_BN_ELEMT_SRC
#undef B200C_BN_ELEMT
}

cudaError_t backward(const BwdArgs& a, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  float* sum_dy = s.sums;
  float* sum_dy_xmu = s.sums + a.c;
  launch_bwd_reduce(a, true, sum_dy, sum_dy_xmu, s, st);
  launch_bwd_elemt(a, true, sum_dy, sum_dy_xmu, (float)(1.0 / a.m), nullptr, st);
  return cudaGetLastError();
}

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

int sync_stats(const FwdArgs& a, cudaStream_t st) {
  SyncRows r = sync_rows(a.scratch, a.c);
  if (a.m == 0) {
    // an empty rank still sends a row: zeros, count 0, which every rank's merge skips
    cudaMemsetAsync(r.local, 0, ((size_t)2 * a.c + 1) * 4, st);
    return 0;
  }
  Scratch s = carve(a.scratch, a.c);
  dim3 block, grid;
  reduce_config(a.m, a.c, &block, &grid);
  const bf16* x = static_cast<const bf16*>(a.x);
  if (vec_ok(a.c, &a.x, 1))
    k_bn_sync_stats<kStatsVec><<<grid, dim3(block.x / kStatsVec, block.y), 0, st>>>(x, r.local, a.eps, s.staging, s.semaphores, a.m, a.c);
  else
    k_bn_sync_stats<1><<<grid, block, 0, st>>>(x, r.local, a.eps, s.staging, s.semaphores, a.m, a.c);
  return 1;
}

int sync_apply(const FwdArgs& a, bool relu, int world, float* norm_fct, cudaStream_t st) {
  SyncRows r = sync_rows(a.scratch, a.c);
  k_bn_sync_merge<<<ceil_div(a.c, kEwThreads), kEwThreads, 0, st>>>(r.gathered, (int)r.row_floats, world, a.save_mean, a.save_invstd,
                                                                    norm_fct, a.running_mean, a.running_var, a.num_batches_tracked,
                                                                    a.momentum, a.eps, a.c);
  if (a.m == 0) return 1;
  launch_transform(a, relu, st);
  return 2;
}

int sync_bwd_reduce(const BwdArgs& a, bool relu, cudaStream_t st) {
  Scratch s = carve(a.scratch, a.c);
  if (a.m == 0) {
    // nothing to sum: zero sums for the allreduce, zero dweight and dbias
    cudaMemsetAsync(s.sums, 0, (size_t)2 * a.c * 4, st);
    cudaMemsetAsync(a.grad_weight, 0, (size_t)a.c * 4, st);
    cudaMemsetAsync(a.grad_bias, 0, (size_t)a.c * 4, st);
    return 0;
  }
  launch_bwd_reduce(a, relu, s.sums, s.sums + a.c, s, st);
  return 1;
}

// Loads every batch-norm kernel into the context (b200coll.cu's load_kernels explains why a loopback world must not
// load a kernel lazily while a peer's collective waits).
cudaError_t load_kernels() {
  cudaFuncAttributes attr;
  cudaError_t e = cudaSuccess;
  auto load = [&](auto kernel) { if (e == cudaSuccess) e = cudaFuncGetAttributes(&attr, kernel); };
  load(k_bn_stats<1>);
  load(k_bn_stats<kStatsVec>);
  load(k_bn_sync_stats<1>);
  load(k_bn_sync_stats<kStatsVec>);
  load(k_bn_sync_merge);
  load(k_bn_bwd_reduce<false>);
  load(k_bn_bwd_reduce<true>);
  load(k_bn_sync_bwd_reduce);
  load(k_bn_transform<1, false>);
  load(k_bn_transform<1, true>);
  load(k_bn_transform<kEwVec, false>);
  load(k_bn_transform<kEwVec, true>);
  load(k_bn_sync_transform<1>);
  load(k_bn_sync_transform<kEwVec>);
  load(k_bn_bwd_elemt<1, kGradMasked>);
  load(k_bn_bwd_elemt<1, kGradY>);
  load(k_bn_bwd_elemt<1, kGradBits>);
  load(k_bn_bwd_elemt<kEwVec, kGradMasked>);
  load(k_bn_bwd_elemt<kEwVec, kGradY>);
  load(k_bn_bwd_elemt<kEwVec, kGradBits>);
  load(k_bn_sync_bwd_elemt<1, kGradMasked>);
  load(k_bn_sync_bwd_elemt<1, kGradY>);
  load(k_bn_sync_bwd_elemt<1, kGradBits>);
  load(k_bn_sync_bwd_elemt<1, kGradDy>);
  load(k_bn_sync_bwd_elemt<kEwVec, kGradMasked>);
  load(k_bn_sync_bwd_elemt<kEwVec, kGradY>);
  load(k_bn_sync_bwd_elemt<kEwVec, kGradBits>);
  load(k_bn_sync_bwd_elemt<kEwVec, kGradDy>);
  return e;
}

int sync_bwd_elemt(const BwdArgs& a, bool relu, const float* norm_fct, cudaStream_t st) {
  if (a.m == 0) return 0;
  Scratch s = carve(a.scratch, a.c);
  launch_bwd_elemt(a, relu, s.sums, s.sums + a.c, 0.f, norm_fct, st);
  return 1;
}

}  // namespace bn
}  // namespace b200c
