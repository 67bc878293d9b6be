// Host-side interface between the C-ABI (b200coll.cu) and the fused batch-norm launchers (inst_norm.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace b200c {
namespace bn {

struct FwdArgs {
  const void* x;         // bf16 [m][c]
  const void* identity;  // bf16 [m][c], or null: no residual add
  void* y;               // bf16 [m][c]
  void* mask;            // uint8 [m * c / 8], or null: receives the ReLU's predicate, one bit per element (c % 8 == 0)
  bool relu;             // a ReLU follows the batch norm (and the residual add); without one, no identity and no mask
  const float* weight;
  const float* bias;
  float* running_mean;
  float* running_var;
  long long* num_batches_tracked;  // may be null
  float* save_mean;
  float* save_invstd;
  int m, c;
  float momentum, eps;
  void* scratch;
  // The stem (pool_h > 0): y is relu(bn(x)) max-pooled 3x3 / stride 2 / padding 1 over m / (pool_h * pool_w)
  // images of pool_h x pool_w rows, and argmax receives one byte per pooled element; identity and mask are null.
  void* argmax;
  int pool_h, pool_w;
};

struct BwdArgs {
  const void* dy;        // bf16 [m][c], gradient of the ReLU's output
  const void* dy2;       // bf16 [m][c], or null: a second gradient of the ReLU's output, added to dy
  const void* y;         // bf16 [m][c], the ReLU's output (read when mask is null)
  const void* mask;      // uint8 [m * c / 8], or null: the forward's mask, read instead of y (c % 8 == 0)
  const void* x;         // bf16 [m][c], the batch norm's input
  void* dy_masked;       // bf16 [m][c], or null: receives the ReLU's input gradient (residual site)
  void* dx;              // bf16 [m][c]
  bool relu;             // as in FwdArgs; without one, dy is the batch norm's output gradient: no y, mask, dy2 or dy_masked
  const float* weight;
  const float* save_mean;
  const float* save_invstd;
  const float* norm_fct;  // device, 1 / float(rows of all ranks) of a sync site, or null: 1 / m
  float* grad_weight;
  float* grad_bias;
  int m, c;
  void* scratch;
  // The stem (pool_h > 0): dy is the pooled output's gradient, argmax the forward's, and dy_masked receives g;
  // y, mask and dy2 are null.
  const void* argmax;
  int pool_h, pool_w;
};

// Largest channel count the kernels take: it bounds the semaphore region at the start of every scratch buffer.
constexpr int kMaxChannels = 1 << 17;

size_t scratch_bytes(int c);
cudaError_t forward(const FwdArgs& a, cudaStream_t s);   // 2 kernels, the stem's included
cudaError_t backward(const BwdArgs& a, cudaStream_t s);  // 2 kernels, the stem's included

// A tail whose identity is a downsample branch's batch norm: `a` the tail's batch norm, `b` the branch's, of the
// same m and c (c <= kMaxChannels / 2).  2 kernels per direction; scratch of dual_scratch_bytes(c).
size_t dual_scratch_bytes(int c);
cudaError_t forward_dual(const FwdArgs& a, const FwdArgs& b, cudaStream_t s);
cudaError_t backward_dual(const BwdArgs& a, const BwdArgs& b, cudaStream_t s);

// Sync batch norm: the local phases around the two collectives, which b200coll.cu runs between them.
//   forward:  sync_stats -> allgather of `local` (2c + 1 floats) into the W `gathered` rows -> sync_apply
//   backward: sync_bwd_reduce -> allreduce SUM of `sums` (2c floats, in place) -> sync_bwd_elemt
// FwdArgs.save_mean / save_invstd receive the global statistics, which the backward reads.  m may be 0: the rank
// then sends zeros and launches only the merge; otherwise each phase launches one kernel, and sync_apply two.
struct SyncRows {
  float* local;       // [mean (c) | invstd (c) | count], 16-byte aligned
  float* gathered;    // W rows like `local`, row_floats apart (16-byte aligned)
  size_t row_floats;
  float* sums;        // [sum_dy (c) | sum_dy_xmu (c)], 16-byte aligned
};
size_t sync_scratch_bytes(int c, int world);
SyncRows sync_rows(void* scratch, int c);
cudaError_t sync_stats(const FwdArgs& a, cudaStream_t s);
cudaError_t sync_apply(const FwdArgs& a, int world, float* norm_fct, cudaStream_t s);
cudaError_t sync_bwd_reduce(const BwdArgs& a, cudaStream_t s);
cudaError_t sync_bwd_elemt(const BwdArgs& a, cudaStream_t s);
cudaError_t load_kernels();   // every batch-norm kernel, into the current context

// Eval-mode sites (norm_infer.cuh): one kernel each, no scratch, nothing written but y.  Weight, bias and running
// statistics of each batch norm are [c] of fp32, or of bf16 with param_bf16.
struct InferParams {
  const void* weight;
  const void* bias;
  const void* running_mean;
  const void* running_var;
  float eps;
};
struct InferArgs {
  const void* x;         // bf16 [m][c]
  const void* identity;  // bf16 [m][c], or null: no residual add; with `ds`, the downsample branch's batch-norm input
  void* y;               // bf16 [m][c], or the pooled rows of the stem
  InferParams bn;
  InferParams ds;        // the downsample branch's batch norm (dual), else unused
  bool dual, param_bf16;
  int m, c;
  int pool_h, pool_w;    // the stem (pool_h > 0): y = max_pool2d(relu(bn(x)), 3, 2, 1) over m / (pool_h * pool_w) images
};
cudaError_t infer(const InferArgs& a, cudaStream_t s);

// Batch norm followed by ReLU6, SiLU or Hardswish (norm_act.cuh; act is b200c_act_t).  A local training site: the
// forward reads FwdArgs without identity, mask or stem (2 kernels), the backward BwdArgs.dy / x / dx / weight, the
// statistics, sums and scratch, and `bias` to recompute the batch norm's output, and writes the activation's gradient g
// to BwdArgs.dy_masked (2 kernels).  The eval site reads
// InferArgs without identity, downsample or stem (1 kernel).
bool act_ok(int act);
cudaError_t forward_act(const FwdArgs& a, int act, cudaStream_t s);
cudaError_t backward_act(const BwdArgs& a, const float* bias, int act, cudaStream_t s);
cudaError_t infer_act(const InferArgs& a, int act, cudaStream_t s);

// Batch norm followed by a residual add, with or without stochastic depth (norm_res.cuh).  A local training site: the
// forward reads FwdArgs without mask or stem (relu false), an optional identity and, with it, optional bf16 noise of
// one value per rows_per_sample rows (2 kernels); the backward reads BwdArgs.dy / x / dx / weight, the statistics,
// sums and scratch, and with noise writes g = bf16(dy * noise) to BwdArgs.dy_masked (2 kernels).  The eval site reads
// InferArgs without downsample or stem (1 kernel).
cudaError_t forward_res(const FwdArgs& a, const void* noise, int rows_per_sample, cudaStream_t s);
cudaError_t backward_res(const BwdArgs& a, const void* noise, int rows_per_sample, cudaStream_t s);
cudaError_t infer_res(const InferArgs& a, cudaStream_t s);

// Batch norm followed by ReLU over the channel concatenation of `n` channels-last segments, read in place (norm_cat.cuh):
// segment s is bf16 [m][channels[s]], channels[s] % 8 == 0, on the 16-byte grid, and the segments' channels sum to
// the site's c.  A local training site: the forward reads FwdArgs without x, identity or stem and writes y and the
// mask (2 kernels); the backward reads BwdArgs.dy and .mask instead of .x, .dy2, .y or .dy_masked, and writes the whole
// [m][c] dx (2 kernels).  The eval site reads InferArgs without x, identity, downsample or stem (1 kernel).
// densenet201's last block concatenates 49 segments.
constexpr int kMaxCatSegs = 64;
struct CatSegments {
  const void* const* ptrs;
  const int* channels;
  int n;
};
cudaError_t forward_cat(const CatSegments& segs, const FwdArgs& a, cudaStream_t s);
cudaError_t backward_cat(const CatSegments& segs, const BwdArgs& a, cudaStream_t s);
cudaError_t infer_cat(const CatSegments& segs, const InferArgs& a, cudaStream_t s);

// Batch norm followed by ReLU whose output y is a channel slice of a wider channels-last tensor (norm_slice.cuh): x is
// the branch's bf16 [m][c], y row r sits at y + r * ldy, and the backward's dy at dy + r * lddy; c, ldy and lddy are
// multiples of 8 and x, y, dy and dx sit on the 16-byte grid.  A local training site: the forward reads FwdArgs
// without identity or stem and writes y's slice and the branch's mask (2 kernels); the backward reads BwdArgs.dy, .mask
// and .x instead of .dy2, .y or .dy_masked and writes dx (2 kernels).  The eval site reads InferArgs without identity,
// downsample or stem (1 kernel).
cudaError_t forward_slice(const FwdArgs& a, int ldy, cudaStream_t s);
cudaError_t backward_slice(const BwdArgs& a, int lddy, cudaStream_t s);
cudaError_t infer_slice(const InferArgs& a, int ldy, cudaStream_t s);

// ShuffleNetV2's block end, channel_shuffle(torch.cat((x1 or relu(bn_u(u)), relu(bn_t(t))), 1), 2) (norm_shuffle.cuh):
// t and u are bf16 [m][c] rows (m = n * hw), y the contiguous NCHW [n][2c][hw] output, x1 NCHW planes x1_stride
// elements apart per sample.  Each mask takes shuffle_mask_bytes(m, c).  A local training site: the forward reads `a`
// (t's batch norm: x, y, mask, parameters, statistics, scratch) and with `b` u's (x, mask, parameters, statistics;
// the dual scratch) instead of x1 (2 kernels); the backward reads a.dy, the channels-last [m][2c] gradient of y, and
// each batch norm's x, mask, weight and statistics, and writes dx, grad_weight and grad_bias (2 kernels).  The eval
// site reads InferArgs x (t), y and bn, and with `dual` identity (u) and ds instead of x1 (1 kernel).
size_t shuffle_mask_bytes(int m, int c);
cudaError_t forward_shuffle(const FwdArgs& a, const FwdArgs* b, const void* x1, int x1_stride, int hw, cudaStream_t s);
cudaError_t backward_shuffle(const BwdArgs& a, const BwdArgs* b, cudaStream_t s);
cudaError_t infer_shuffle(const InferArgs& a, const void* x1, int x1_stride, int hw, cudaStream_t s);

// VGG's stage end, max_pool2d(relu(bn(x)), 2, 2) (norm_pool2.cuh): FwdArgs, BwdArgs and InferArgs as at the stem (pool_h
// by pool_w images, h, w >= 2), with n * (h / 2) * (w / 2) pooled rows and one argmax byte per pooled element.  The
// backward writes no g (BwdArgs.dy_masked is unused).  2 kernels per training direction, 1 in eval.
cudaError_t forward_pool2(const FwdArgs& a, cudaStream_t s);
cudaError_t backward_pool2(const BwdArgs& a, cudaStream_t s);
cudaError_t infer_pool2(const InferArgs& a, cudaStream_t s);

}  // namespace bn
}  // namespace b200c
