// The end of torchvision's ShuffleNetV2 block, `channel_shuffle(torch.cat((a, relu(bn_t(t))), 1), 2)` with a either the
// block input's first half x1 (stride 1: one batch norm) or relu(bn_u(u)) (stride 2: two batch norms), in training and
// eval, with the shuffled output written directly: no branch output and no concatenation exists.
//
// Shapes.  t and u are the branches' channels-last (NHWC) bf16 [m][B], m = n * hw rows, any B >= 1.  The output y is
// contiguous NCHW bf16 [n][2B][hw], as channel_shuffle's `.contiguous()` leaves it: channel 2c is a's channel c and
// channel 2c + 1 is relu(bn_t(t))'s channel c.  x1 is read as NCHW planes, element (n, c, p) at x1 + n * x1_stride +
// c * hw + p (x1_stride = 2B * hw where x1 is x.chunk(2, 1)[0] of a contiguous x).  The backward reads dy, the
// output's gradient, channels-last [m][2B]: a's gradient at channel 2c, t's at 2c + 1, so one 4-byte load feeds both
// batch norms of the two-batch-norm form.
//
// Mask.  The ReLU's predicate !(y <= 0) of each batch norm is kept as bits, for every B: row r of [m][B] takes
// mask_row_bytes(B) = ceil(B / 8) bytes, channel c is bit c % 8 of byte r * ceil(B / 8) + c / 8, and the bits of a
// row's padding channels are 0.  With B % 8 == 0 this is the bn:: kernels' layout.
//
// Bits.  The statistics are bn::k_bn_stats (one batch norm) or bn::k_bn_stats_dual (two).  The transform and eval
// kernels compute each element as bn::k_bn_transform<V, kTailRelu> and bn_infer::k_infer_transform<V, kTailRelu, P>
// do; they only route the result through a shared-memory tile to store NCHW planes.  The backward reduce is
// bn::k_bn_bwd_reduce<kGradBits, false>'s register walk (V = 1) with torch's launch shape for [m][B]: the same
// per-thread row sequence, block tree and grid merge, so every sum is torch's.  Each batch norm's sums are
// accumulated, merged over the block and over the grid as their own launch would merge them.  The backward
// elementwise kernel is bn::k_bn_bwd_elemt<1, kGradBits, false, false>'s expression per element.
#pragma once
#include "norm_infer.cuh"
#include "norm_kernels.cuh"

namespace b200c {
namespace bn_shuffle {

using bn::bf16;
using bn::kEwThreads;
using bn::kMaxBlock;
using bn::kParallelLoads;

__host__ __device__ constexpr int mask_row_bytes(int channels) { return (channels + 7) / 8; }

// The output tile: kTile rows of the input by kTile channels per block of kEwThreads threads.  The first pass reads
// a row's channels (warp = one row, lanes = channels) and packs each 8-channel mask byte with a ballot; the second
// writes each output plane's kTile consecutive rows (warp = one channel, lanes = rows).
constexpr int kTile = 32;
constexpr int kTileRowsPerPass = kEwThreads / kTile;

struct Geometry {
  int m, c, hw;
  const bf16* x1;    // the stride-1 form's pass-through, or null: the two-batch-norm form
  int x1_stride;     // x1's sample stride in elements
};

// Per-channel affine form of a batch norm: y = relu(bf16(w * (x - mean) * inv_std + s)).
struct Affine {
  float mean, inv_std, w, s;
  __device__ __forceinline__ bf16 relu_bn(bf16 x) const {
    auto tmp = w * (__bfloat162float(x) - mean) * inv_std + s;
    return tmp <= 0.f ? __float2bfloat16(0.f) : __float2bfloat16(tmp);
  }
};

// One block's tile.  chan_t(c) / chan_u(c) give channel c's Affine; mask_t / mask_u, where set, receive the bits.
template <bool TWO, typename ChanT, typename ChanU>
__device__ __forceinline__ void shuffle_tile(const bf16* __restrict__ t, const bf16* __restrict__ u, bf16* __restrict__ out,
                                             uint8_t* __restrict__ mask_t, uint8_t* __restrict__ mask_u, const Geometry g,
                                             ChanT chan_t, ChanU chan_u) {
  __shared__ bf16 tile_t[kTile][kTile + 1];
  __shared__ bf16 tile_u[TWO ? kTile : 1][kTile + 1];
  const int lane = threadIdx.x % kTile, row_in = threadIdx.x / kTile;
  const int r0 = blockIdx.x * kTile, c0 = blockIdx.y * kTile;
  const int mb = mask_row_bytes(g.c);
  {
    const int c = c0 + lane;
    const bool c_ok = c < g.c;
    bn_shuffle::Affine at{}, au{};
    if (c_ok) {
      at = chan_t(c);
      if (TWO) au = chan_u(c);
    }
    for (int rr = row_in; rr < kTile; rr += kTileRowsPerPass) {
      const int r = r0 + rr;
      if (r >= g.m) break;   // warp-uniform: a warp holds one row
      bf16 yt = __float2bfloat16(0.f), yu = __float2bfloat16(0.f);
      if (c_ok) {
        yt = at.relu_bn(t[(size_t)r * g.c + c]);
        if (TWO) yu = au.relu_bn(u[(size_t)r * g.c + c]);
      }
      tile_t[lane][rr] = yt;
      if (TWO) tile_u[lane][rr] = yu;
      const unsigned bt = __ballot_sync(0xffffffffu, c_ok && !(__bfloat162float(yt) <= 0.f));
      const unsigned bu = TWO ? __ballot_sync(0xffffffffu, c_ok && !(__bfloat162float(yu) <= 0.f)) : 0u;
      if (lane % 8 == 0 && c_ok) {
        const size_t at_byte = (size_t)r * mb + c / 8;
        if (mask_t) mask_t[at_byte] = (uint8_t)(bt >> lane);
        if (TWO && mask_u) mask_u[at_byte] = (uint8_t)(bu >> lane);
      }
    }
  }
  __syncthreads();
  const int r = r0 + lane;
  if (r >= g.m) return;
  const int n = r / g.hw, p = r - n * g.hw;
  bf16* const base = out + (size_t)n * 2 * g.c * g.hw + p;
  for (int cc = row_in; cc < kTile; cc += kTileRowsPerPass) {
    const int c = c0 + cc;
    if (c >= g.c) break;
    base[(size_t)(2 * c + 1) * g.hw] = tile_t[cc][lane];
    base[(size_t)(2 * c) * g.hw] = TWO ? tile_u[cc][lane] : g.x1[(size_t)n * g.x1_stride + (size_t)c * g.hw + p];
  }
}

struct SavedStats {
  const float* mean;
  const float* inv_std;
  const float* weight;
  const float* bias;
  __device__ __forceinline__ Affine operator()(int c) const { return Affine{mean[c], inv_std[c], weight[c], bias[c]}; }
};

// Training: y from t (and u) with the saved statistics, and each batch norm's mask.  grid (ceil(m / kTile),
// ceil(B / kTile)), block kEwThreads.
template <bool TWO>
__global__ void __launch_bounds__(kEwThreads) k_shuffle_transform(const bf16* __restrict__ t, const bf16* __restrict__ u,
                                                                  bf16* __restrict__ out, uint8_t* __restrict__ mask_t,
                                                                  uint8_t* __restrict__ mask_u, const SavedStats st, const SavedStats su,
                                                                  const Geometry g) {
  shuffle_tile<TWO>(t, u, out, mask_t, mask_u, g, st, su);
}

template <typename P>
struct RunningStats {
  const P* running_mean;
  const P* running_var;
  const P* weight;
  const P* bias;
  float eps;
  __device__ __forceinline__ Affine operator()(int c) const {
    const bn_infer::Channel<P> k(running_mean, running_var, weight, bias, eps, c);
    return Affine{k.mean, k.inv_std, k.w, k.s};
  }
};

// Eval: y from t (and u) with the running statistics, nothing else written.  Launched as k_shuffle_transform.
template <bool TWO, typename P>
__global__ void __launch_bounds__(kEwThreads) k_shuffle_infer(const bf16* __restrict__ t, const bf16* __restrict__ u,
                                                              bf16* __restrict__ out, const RunningStats<P> st, const RunningStats<P> su,
                                                              const Geometry g) {
  shuffle_tile<TWO>(t, u, out, nullptr, nullptr, g, st, su);
}

// What the backward kernels read and write of one batch norm.
struct BwdSite {
  const bf16* x;          // t or u, [m][B]
  const uint8_t* mask;
  const float* mean;
  const float* inv_std;
  const float* weight;
  float* grad_weight;
  float* grad_bias;       // also the sum of g, which the elementwise kernel reads
  float* sum_dy_xmu;
  volatile float* staging;
  bf16* dx;
};

// bn::k_bn_bwd_reduce<kGradBits, false> with V = 1 for t (dy's odd channels) and, in the two-batch-norm form, u (its
// even channels) from the same walk: per thread and batch norm torch's PARALLEL_LOADS accumulators, block tree and
// grid merge.  Each batch norm stages in its own region; the last block of a column (one semaphore per column) merges
// both.
template <bool TWO>
__global__ void __launch_bounds__(kMaxBlock) k_shuffle_bwd_reduce(const bf16* __restrict__ grad_output, const BwdSite st, const BwdSite su,
                                                                  int* semaphores, const int reduction_size, const int stride) {
  constexpr int PARALLEL_LOADS = kParallelLoads;
  constexpr int S = TWO ? 2 : 1;   // batch norms: 0 is t's, 1 is u's
  __shared__ float shmem_sum_dy[kMaxBlock];
  __shared__ float shmem_sum_dy_xmu[kMaxBlock];
  __shared__ bool is_last_block_done;

  float sum_dy[S][PARALLEL_LOADS];
  float sum_dy_xmu[S][PARALLEL_LOADS];
#pragma unroll
  for (int s = 0; s < S; s++)
#pragma unroll
    for (int i = 0; i < PARALLEL_LOADS; i++) {
      sum_dy[s][i] = float(0);
      sum_dy_xmu[s][i] = float(0);
    }
  int inner_loop_stride = blockDim.y * gridDim.y;
  int m_offset = blockIdx.y * blockDim.y + threadIdx.y;
  const int c_offset = blockIdx.x * blockDim.x + threadIdx.x;
  if (c_offset >= stride || m_offset >= reduction_size) return;

  const int loop_count = 1 + (reduction_size - 1) / (inner_loop_stride * PARALLEL_LOADS);
  const int mb = mask_row_bytes(stride);
  const unsigned bit = c_offset & 7;
  float r_mean[S];
  r_mean[0] = st.mean[c_offset];
  if (TWO) r_mean[S - 1] = su.mean[c_offset];

  for (int i = 0; i < loop_count; i++) {
    // all rows of the iteration are loaded before any sum uses one
    __nv_bfloat162 dy_v[PARALLEL_LOADS];
    bf16 x_v[S][PARALLEL_LOADS];
    uint8_t mask_v[S][PARALLEL_LOADS];
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
      const int m = m_offset + j * inner_loop_stride;
      if (m < reduction_size) {
        dy_v[j] = *reinterpret_cast<const __nv_bfloat162*>(grad_output + ((size_t)m * 2 * stride + 2 * c_offset));
        x_v[0][j] = st.x[(size_t)m * stride + c_offset];
        mask_v[0][j] = st.mask[(size_t)m * mb + (c_offset >> 3)];
        if (TWO) {
          x_v[S - 1][j] = su.x[(size_t)m * stride + c_offset];
          mask_v[S - 1][j] = su.mask[(size_t)m * mb + (c_offset >> 3)];
        }
      }
    }
#pragma unroll
    for (int j = 0; j < PARALLEL_LOADS; j++) {
#pragma unroll
      for (int s = 0; s < S; s++) {
        float x_input = float(0), x_grad_output = float(0);
        if (m_offset < reduction_size) {
          const bf16 dy = s == 0 ? dy_v[j].y : dy_v[j].x;
          x_input = __bfloat162float(x_v[s][j]);
          x_grad_output = __bfloat162float(bn::relu_grad_bit(dy, (mask_v[s][j] >> bit) & 1u));
        }
        sum_dy[s][j] += x_grad_output;
        sum_dy_xmu[s][j] = __fmaf_rn(x_grad_output, x_input - r_mean[s], sum_dy_xmu[s][j]);
      }
      m_offset += inner_loop_stride;
    }
  }

  float sum_dy_th[S], sum_dy_xmu_th[S];
#pragma unroll
  for (int s = 0; s < S; s++) {
#pragma unroll
    for (int j = 1; j < PARALLEL_LOADS; j++) {
      sum_dy[s][0] += sum_dy[s][j];
      sum_dy_xmu[s][0] += sum_dy_xmu[s][j];
    }
    sum_dy_th[s] = sum_dy[s][0];
    sum_dy_xmu_th[s] = sum_dy_xmu[s][0];
  }
  // each batch norm's values take the tree in turn (each value's tree is independent of the others)
  auto merge = [&]() {
#pragma unroll
    for (int s = 0; s < S; s++) {
      if (s) __syncthreads();
      bn::merge_block_vertical_backward(sum_dy_th[s], sum_dy_xmu_th[s], shmem_sum_dy, shmem_sum_dy_xmu);
    }
  };
  merge();

  auto write_sums = [&]() {
#pragma unroll
    for (int s = 0; s < S; s++) {
      const BwdSite& b = s == 0 ? st : su;
      b.grad_bias[c_offset] = sum_dy_th[s];
      b.grad_weight[c_offset] = sum_dy_xmu_th[s] * b.inv_std[c_offset];
      b.sum_dy_xmu[c_offset] = sum_dy_xmu_th[s];
    }
  };
  if (gridDim.y > 1) {
    if (threadIdx.y == 0) {
#pragma unroll
      for (int s = 0; s < S; s++) {
        volatile float* staging = s == 0 ? st.staging : su.staging;
        staging[c_offset + blockIdx.y * stride] = sum_dy_th[s];
        staging[stride * gridDim.y + c_offset + blockIdx.y * stride] = sum_dy_xmu_th[s];
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
      for (int s = 0; s < S; s++) {
        volatile float* staging = s == 0 ? st.staging : su.staging;
        sum_dy_th[s] = float(0.0);
        sum_dy_xmu_th[s] = float(0.0);
        for (int y = threadIdx.y; y < gridDim.y; y += blockDim.y) {
          sum_dy_th[s] += staging[c_offset + y * stride];
          sum_dy_xmu_th[s] += staging[stride * gridDim.y + c_offset + y * stride];
        }
      }
      merge();
      if (threadIdx.y == 0) write_sums();
    }
  } else {
    if (blockIdx.y == 0 && threadIdx.y == 0) write_sums();
  }
}

// bn::k_bn_bwd_elemt<1, kGradBits, false, false> per batch norm: dt (and du) with g = mask ? dy : 0, dy read at its
// channel 2c + 1 (2c), and this call's norm_fct = 1 / m.  ew_config's launch for [m][B] with one channel per thread.
template <bool TWO>
__global__ void __launch_bounds__(kEwThreads) k_shuffle_bwd_elemt(const bf16* __restrict__ grad_output, const BwdSite st,
                                                                  const BwdSite su, const float norm_fct, const int reduction_size,
                                                                  const int stride) {
  constexpr int S = TWO ? 2 : 1;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= stride) return;
  float m_c[S], m_dy_c[S], factor_1_c[S], factor_2_c[S];
#pragma unroll
  for (int s = 0; s < S; s++) {
    const BwdSite& b = s == 0 ? st : su;
    m_c[s] = b.mean[c];
    m_dy_c[s] = b.grad_bias[c] * norm_fct;
    factor_1_c[s] = b.inv_std[c];
    factor_2_c[s] = b.weight[c] * factor_1_c[s];
    factor_1_c[s] = factor_1_c[s] * factor_1_c[s] * b.sum_dy_xmu[c] * norm_fct;
  }
  const int mb = mask_row_bytes(stride);
  const int row_step = blockDim.y * gridDim.y;
  for (int m = blockIdx.y * blockDim.y + threadIdx.y; m < reduction_size; m += row_step) {
    const __nv_bfloat162 gv = *reinterpret_cast<const __nv_bfloat162*>(grad_output + ((size_t)m * 2 * stride + 2 * c));
    const size_t a = (size_t)m * stride + c;
#pragma unroll
    for (int s = 0; s < S; s++) {
      const BwdSite& b = s == 0 ? st : su;
      const unsigned bit = (b.mask[(size_t)m * mb + (c >> 3)] >> (c & 7)) & 1u;
      const float g = __bfloat162float(bn::relu_grad_bit(s == 0 ? gv.y : gv.x, bit));
      b.dx[a] = __float2bfloat16((g - m_dy_c[s] - (__bfloat162float(b.x[a]) - m_c[s]) * factor_1_c[s]) * factor_2_c[s]);
    }
  }
}

}  // namespace bn_shuffle
}  // namespace b200c
