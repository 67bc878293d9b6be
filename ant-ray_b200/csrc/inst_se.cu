// Launchers of the squeeze-and-excitation kernels (se_kernels.cuh); argument checking lives in b200coll.cu.
#include <stdint.h>

#include <algorithm>
#include <initializer_list>

#include "se_kernels.cuh"
#include "se_launch.h"

namespace b200c {
namespace se {

static int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// Reduce.cuh's last_pow2
static int last_pow2(long long n) {
  n |= (n >> 1);
  n |= (n >> 2);
  n |= (n >> 4);
  n |= (n >> 8);
  n |= (n >> 16);
  n |= (n >> 32);
  return (int)std::max<long long>(1, n - (n >> 1));
}

// Torch's output_vec_size for the reduction of a tensor at `ptr` (get_output_vec_size): 4, halved until it divides
// the element address and C (the other strides, C and HW * C, follow from C).
static int output_vec_size(const void* ptr, int c) {
  const unsigned long long elem = reinterpret_cast<unsigned long long>(ptr) / 2;
  int v = 4;
  while (elem % v || c % v) v /= 2;
  return v;
}

struct Config {
  ReduceShape r;
  dim3 block, grid;
  int vec;
};

// setReduceConfig<float, bf16, vt0 = 4> for the mean / sum over (H, W) of a channels-last [n, c, H, W] bf16 tensor,
// the "vectorize along output" case: num_outputs = n * c, inputs_per_output = hw, dim0 = n * c / vec, dim1 = hw.
// num_mp and max_tpm are the device's multiProcessorCount and maxThreadsPerMultiProcessor.
static Config reduce_config(int n, int c, int hw, int vec, int num_mp, int max_tpm) {
  Config k;
  k.vec = vec;
  const long long num_outputs = (long long)n * c;
  const long long dim0 = num_outputs / vec, dim1 = hw;
  const int mnt = kMaxThreads / vec;
  const int d0 = dim0 < mnt ? last_pow2(dim0) : mnt;
  const int d1 = dim1 < mnt ? last_pow2(dim1) : mnt;
  int bw = std::min(d0, 32);
  const int bh = std::min(d1, mnt / bw);
  bw = std::min(d0, mnt / bh);
  const int num_threads = bw * bh;
  // output_mult[0] = split_output(block_width); then the warps take rows (split) or outputs
  int step_output = bw, step_input = 1;
  const bool split = hw >= std::min(bh * 16, 256);
  if (split) step_input = bh;
  else step_output *= bh;
  const int grid_x = div_up(dim0, step_output);
  const int target = num_mp * (max_tpm / num_threads);
  int ctas = 1;
  const int vpt = div_up(hw, step_input);
  if (split && vpt >= 256 && grid_x <= target) {
    const int c1 = div_up(target, grid_x), c2 = div_up(vpt, 16), c3 = div_up(vpt, 256);
    ctas = std::max(std::min(c1, c2), c3);
  }
  k.r = ReduceShape{(int)num_outputs, c, hw, split ? 1 : 0, ctas};
  k.block = dim3(bw, bh, 1);
  k.grid = dim3(grid_x, ctas, 1);
  return k;
}

static size_t staging_floats(const Config& k) {
  return k.r.ctas > 1 ? (size_t)k.grid.x * k.grid.y * k.block.x * k.vec : 0;
}

static cudaError_t device_limits(int* num_mp, int* max_tpm) {
  int dev;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(num_mp, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(max_tpm, cudaDevAttrMaxThreadsPerMultiProcessor, dev);
  return e;
}

size_t scratch_bytes(int n, int c, int hw, cudaError_t* err) {
  int num_mp, max_tpm;
  *err = device_limits(&num_mp, &max_tpm);
  if (*err != cudaSuccess) return 0;
  // the pool's vec follows x's address, the reduce's follows C: take the largest staging of any vec C allows
  size_t floats = 0;
  for (int vec = 4; vec >= 1; vec /= 2)
    if (c % vec == 0) floats = std::max(floats, staging_floats(reduce_config(n, c, hw, vec, num_mp, max_tpm)));
  return (size_t)kSemaphores * 4 + floats * 4;
}

template <bool kProduct>
static cudaError_t launch_reduce(const void* a, const void* b, void* out, float factor, int n, int c, int hw, int vec, void* scratch,
                                 cudaStream_t s) {
  int num_mp, max_tpm;
  cudaError_t e = device_limits(&num_mp, &max_tpm);
  if (e != cudaSuccess) return e;
  const Config k = reduce_config(n, c, hw, vec, num_mp, max_tpm);
  if (k.r.ctas > 1 && k.grid.x > (unsigned)kSemaphores) return cudaErrorInvalidValue;
  int* semaphores = static_cast<int*>(scratch);
  float* staging = reinterpret_cast<float*>(static_cast<char*>(scratch) + (size_t)kSemaphores * 4);
  const bf16* pa = static_cast<const bf16*>(a);
  const bf16* pb = static_cast<const bf16*>(b);
  bf16* po = static_cast<bf16*>(out);
  if (!kProduct) {
    switch (vec) {
      case 4: k_se_pool<4><<<k.grid, k.block, 0, s>>>(pa, po, factor, k.r, staging, semaphores); break;
      case 2: k_se_pool<2><<<k.grid, k.block, 0, s>>>(pa, po, factor, k.r, staging, semaphores); break;
      default: k_se_pool<1><<<k.grid, k.block, 0, s>>>(pa, po, factor, k.r, staging, semaphores); break;
    }
  } else {
    const int bytes = 2 * vec;
    const bool aligned = reinterpret_cast<uintptr_t>(a) % bytes == 0 && reinterpret_cast<uintptr_t>(b) % bytes == 0;
    switch (vec * 2 + aligned) {
      case 9: k_se_bwd_reduce<4, true><<<k.grid, k.block, 0, s>>>(pa, pb, po, k.r, staging, semaphores); break;
      case 8: k_se_bwd_reduce<4, false><<<k.grid, k.block, 0, s>>>(pa, pb, po, k.r, staging, semaphores); break;
      case 5: k_se_bwd_reduce<2, true><<<k.grid, k.block, 0, s>>>(pa, pb, po, k.r, staging, semaphores); break;
      case 4: k_se_bwd_reduce<2, false><<<k.grid, k.block, 0, s>>>(pa, pb, po, k.r, staging, semaphores); break;
      default: k_se_bwd_reduce<1, false><<<k.grid, k.block, 0, s>>>(pa, pb, po, k.r, staging, semaphores); break;
    }
  }
  return cudaGetLastError();
}

cudaError_t pool(const void* x, void* pooled, int n, int c, int hw, void* scratch, cudaStream_t s) {
  // MeanOps' factor: float(num_output_elements) / numel, the int64 numel converted to float
  const long long nc = (long long)n * c;
  const float factor = static_cast<float>(nc) / static_cast<float>(nc * hw);
  return launch_reduce<false>(x, nullptr, pooled, factor, n, c, hw, output_vec_size(x, c), scratch, s);
}

cudaError_t backward_reduce(const void* dy, const void* x, void* ds, int n, int c, int hw, void* scratch, cudaStream_t s) {
  // torch reduces a freshly allocated product tensor, whose address is on every vector grid
  return launch_reduce<true>(dy, x, ds, 1.f, n, c, hw, output_vec_size(nullptr, c), scratch, s);
}

// Elementwise launches: V channels per thread, a block of kEwThreads threads over channel groups and rows, and enough
// blocks for a few waves (each thread strides over the rows).
static void ew_config(int rows, int c, int vec, dim3* block, dim3* grid) {
  const int groups = c / vec;
  const int bx = std::min(groups, kEwThreads);
  const int by = kEwThreads / bx;
  const int gx = div_up(groups, bx);
  const int gy = std::max(1, std::min(div_up(rows, by), 4096 / gx));
  *block = dim3(bx, by, 1);
  *grid = dim3(gx, gy, 1);
}

static bool ew_vec_ok(int c, std::initializer_list<const void*> ptrs) {
  if (c % kEwVec) return false;
  for (const void* p : ptrs)
    if (reinterpret_cast<uintptr_t>(p) % 16) return false;
  return true;
}

cudaError_t scale(const void* x, const void* sc, void* y, int n, int c, int hw, cudaStream_t s) {
  const int rows = n * hw;
  const bf16* px = static_cast<const bf16*>(x);
  const bf16* ps = static_cast<const bf16*>(sc);
  bf16* py = static_cast<bf16*>(y);
  dim3 block, grid;
  if (ew_vec_ok(c, {x, sc, y})) {
    ew_config(rows, c, kEwVec, &block, &grid);
    k_se_scale<kEwVec><<<grid, block, 0, s>>>(px, ps, py, rows, c, hw);
  } else {
    ew_config(rows, c, 1, &block, &grid);
    k_se_scale<1><<<grid, block, 0, s>>>(px, ps, py, rows, c, hw);
  }
  return cudaGetLastError();
}

cudaError_t backward_elemt(const void* dy, const void* sc, const void* gp, void* dx, int n, int c, int hw, cudaStream_t s) {
  const int rows = n * hw;
  // div_true's CPU-scalar path: a multiply by opmath 1 / float(HW)
  const float inv_hw = 1.0f / static_cast<float>(hw);
  const bf16* pd = static_cast<const bf16*>(dy);
  const bf16* ps = static_cast<const bf16*>(sc);
  const bf16* pg = static_cast<const bf16*>(gp);
  bf16* px = static_cast<bf16*>(dx);
  dim3 block, grid;
  if (ew_vec_ok(c, {dy, sc, gp, dx})) {
    ew_config(rows, c, kEwVec, &block, &grid);
    k_se_bwd_elemt<kEwVec><<<grid, block, 0, s>>>(pd, ps, pg, px, inv_hw, rows, c, hw);
  } else {
    ew_config(rows, c, 1, &block, &grid);
    k_se_bwd_elemt<1><<<grid, block, 0, s>>>(pd, ps, pg, px, inv_hw, rows, c, hw);
  }
  return cudaGetLastError();
}

}  // namespace se
}  // namespace b200c
