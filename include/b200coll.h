/*
 * b200coll.h — C-ABI of the B200 peer-memory collective / tensor-transport library.
 *
 * This is the drop-in boundary for the hot path (SURVEY.md §8b).
 * The reference has no C seam of its own on this path: its only native boundary is
 * cupy's NcclCommunicator, which takes raw integer device pointers, element counts,
 * NCCL dtype / redop enums and a raw stream pointer.  Every entry point below replaces
 * one of those call sites and keeps that call shape (plain pointers and sizes, no torch
 * or cupy types).  Enum values are the ncclDataType_t / ncclRedOp_t numbering so the
 * reference's dtype/op maps (nccl_util.py:22-87) carry over unchanged.
 *
 * All collective / p2p calls are asynchronous: they enqueue work on `stream` and return.
 * Return value: 0 on success, a negative B200C_E* code otherwise; b200c_last_error()
 * returns a thread-local human-readable message for the last failure.
 *
 * Threading: a communicator is NOT thread-safe (same contract as the reference:
 * nccl_collective_group.py:127 "we need a lock here", nccl_group.py:26 "not thread-safe").
 */
#ifndef B200COLL_H_
#define B200COLL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200C_VERSION 200 /* 0.2.0 */
#define B200C_MAX_RANKS 8 /* one NVSwitch domain (SURVEY.md §8e) */

/* ncclDataType_t numbering (reference: nccl_util.py:30-71 maps numpy/torch dtypes onto these). */
typedef enum {
  B200C_INT8 = 0,
  B200C_UINT8 = 1,
  B200C_INT32 = 2,
  B200C_UINT32 = 3,
  B200C_INT64 = 4,
  B200C_UINT64 = 5,
  B200C_FLOAT16 = 6,
  B200C_FLOAT32 = 7,
  B200C_FLOAT64 = 8,
  B200C_BFLOAT16 = 9,
  B200C_NUM_DTYPES = 10
} b200c_dtype_t;

/* ncclRedOp_t numbering.  ray.experimental.util.types.ReduceOp passes its .value raw
 * (nccl_group.py:304,325); ray.util.collective.types.ReduceOp goes through
 * NCCL_REDUCE_OP_MAP (nccl_util.py:22-27).
 *
 * Semantics at the edges (pinned by tests/test_oracle.py and tests/test_gpu_value_edges.py):
 *  - Ranks are folded in order 0..W-1.  MIN / MAX fold with `acc = a < b ? a : b` /
 *    `acc = a > b ? a : b` (a = the fold so far, b = the next rank).  That rule decides NaN and
 *    signed zeros: whenever the comparison is false (a NaN on either side, or +0 against -0) the
 *    next rank's value is taken, so MAX over ranks [NaN, 1] is 1, over [1, NaN] is NaN, and over
 *    [+0, -0] is -0.
 *  - Integer SUM / PROD wrap around (two's complement, modulo 2^bits).  Integer AVG is that
 *    wrapped sum divided by W with truncation toward zero (ncclAvg).
 *  - f16 / bf16 accumulate in fp32.  A scaled sum (AVG, b200c_allreduce_scaled) multiplies the
 *    fp32 accumulator by the scale and rounds once, after the scale, to the element (or wire) type;
 *    f64 AVG divides in fp64.  A contribution is rounded to the wire type before it is summed. */
typedef enum {
  B200C_SUM = 0,
  B200C_PROD = 1,
  B200C_MAX = 2,
  B200C_MIN = 3,
  B200C_AVG = 4,
  B200C_NUM_OPS = 5
} b200c_redop_t;

/* Algorithm selector for allreduce. AUTO picks by message size (thresholds in b200c_config_t). */
typedef enum {
  B200C_ALGO_AUTO = 0,
  B200C_ALGO_ONESHOT = 1, /* every rank pushes its whole buffer to every peer, reduces locally */
  B200C_ALGO_TWOSHOT = 2, /* push reduce-scatter + pull all-gather over peer memory */
  B200C_ALGO_NVLS = 3,    /* multimem.ld_reduce / multimem.st on the NVSwitch multicast object */
  B200C_ALGO_NVLS_PIPE = 4,/* same, staged copies overlapped with the switch traffic (per-round flags, software-pipelined blocks) */
  B200C_ALGO_LL = 5,       /* packed {data, flag} 8-byte stores, one NVLink hop, no fence: small messages */
  B200C_ALGO_NVLS_LANES = 6,/* staged NVLS in lanes: few switch-only CTAs + many copy-only CTAs over an L2-resident staging ring */
  B200C_ALGO_NVLS_STREAMS = 7 /* staged NVLS as a pipeline of kernels on internal streams: copy-in | 32-CTA zero-copy NVLS | copy-out per piece */
} b200c_algo_t;

typedef enum {
  B200C_OK = 0,
  B200C_EINVAL = -1,      /* bad argument (maps to ValueError / RuntimeError on the Python side) */
  B200C_ECUDA = -2,       /* CUDA runtime / driver call failed */
  B200C_ESTATE = -3,      /* communicator not ready / already destroyed */
  B200C_EUNSUPPORTED = -4,/* dtype/op/algorithm combination not available on this device */
  B200C_ETIMEOUT = -5,    /* a kernel gave up waiting for a peer flag (dead or mismatched peer) */
  B200C_EABORTED = -6,    /* b200c_comm_abort() was called while kernels were waiting */
  B200C_EMISMATCH = -7,   /* peers disagreed on op / dtype / count for the same sequence number */
  B200C_ENOMEM = -8
} b200c_status_t;

/* How a rank's arena is shared with its peers. */
typedef enum {
  B200C_SHARE_VMM_FD = 0,     /* cuMemCreate + POSIX fd (SCM_RIGHTS side channel); multicast capable */
  B200C_SHARE_LEGACY_IPC = 1  /* cudaMalloc + 64-byte cudaIpcMemHandle_t (plain bytes, object store) */
} b200c_share_mode_t;

typedef struct {
  uint32_t struct_size;        /* sizeof(b200c_config_t), for forward compatibility */
  int32_t share_mode;          /* b200c_share_mode_t */
  uint64_t staging_bytes;      /* bytes of ONE staging half (two halves are allocated) */
  uint64_t symmetric_bytes;    /* user-visible symmetric region (0 = none) */
  uint64_t p2p_slot_bytes;     /* bytes of one p2p ring slot */
  uint32_t p2p_slots;          /* ring slots per ordered (src,dst) pair */
  uint32_t max_blocks;         /* upper bound on CTAs per collective kernel (<= 2048) */
  uint64_t oneshot_max_bytes;  /* AUTO: message <= this -> one-shot */
  uint64_t nvls_min_bytes;     /* AUTO: message >= this and multicast bound -> NVLS */
  uint64_t nvls_pipe_min_bytes;/* AUTO: staged NVLS pieces >= this use the round-pipelined kernel (0 = never) */
  uint64_t timeout_ms;         /* device-side bounded spin; 0 = default (600 s; NCCL's watchdog default is of that order) */
  uint64_t granule_bytes;      /* block-cyclic granule of the large-message kernels (multiple of 16 KiB; 0 = 32 KiB) */
  uint64_t ll_max_bytes;       /* AUTO: same-type allreduce <= this goes by the LL kernel; also sizes the LL region (0 = no LL) */
  uint64_t bcast_rounds_min_bytes; /* broadcast >= this uses scatter + multicast-allgather rounds (0 = never) */
  uint32_t nvls_blocks;        /* CTAs of the zero-copy NVLS kernel (0 = max_blocks) */
  uint32_t nvls_lanes;         /* lane kernel: lanes (each 1 switch CTA + (max_blocks / lanes - 1 <= 7) copy CTAs) */
  uint64_t lane_granule_bytes; /* lane kernel: bytes of one rank chunk's granule per round (multiple of 8 KiB) */
  uint64_t nvls_lanes_min_bytes; /* AUTO: staged NVLS messages >= this use the lane kernel (0 = never) */
  uint32_t nvls_unroll;        /* reserved (ignored): round-2 experiment, 8 instead of 4 multimem vectors in flight - no gain, removed */
  uint32_t rounds_order;       /* reserved (ignored): round-2 experiment, copy-out before the switch stage - slower, removed */
  uint64_t nvls_streams_min_bytes; /* AUTO: staged NVLS messages >= this use the multi-stream pipeline (0 = never) */
  uint64_t nvls_streams_piece_bytes; /* bytes (on the wire) per pipeline piece; at least 3 pieces must fit 2 * staging_bytes */
} b200c_config_t;

typedef struct {
  int32_t device;              /* CUDA ordinal queried */
  int32_t sm_count;
  int32_t cc_major, cc_minor;
  int32_t vmm_supported;       /* CU_DEVICE_ATTRIBUTE_VIRTUAL_MEMORY_MANAGEMENT_SUPPORTED */
  int32_t posix_fd_supported;  /* CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED */
  int32_t multicast_supported; /* CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED */
  int32_t reserved;
  uint64_t total_mem;
} b200c_props_t;

/* Opaque bytes a rank publishes so that peers can map its arena.  With SHARE_VMM_FD the
 * `fd` must travel by SCM_RIGHTS (the Python host side does this over a Unix socket);
 * with SHARE_LEGACY_IPC `ipc` is self-contained and can go through Ray's object store
 * (north_star: "CUDA-IPC handles exchanged through the object store"). */
typedef struct {
  int32_t share_mode;
  int32_t fd;                  /* -1 unless SHARE_VMM_FD */
  uint64_t arena_bytes;
  uint64_t layout_hash;        /* peers must agree on the arena layout */
  int32_t pid;
  int32_t device_uuid_lo;      /* low 32 bits of the device UUID, diagnostics only */
  uint8_t ipc[64];             /* cudaIpcMemHandle_t when SHARE_LEGACY_IPC */
} b200c_export_t;

typedef struct b200c_comm b200c_comm_t;
typedef void* b200c_stream_t;  /* cudaStream_t / CUstream, passed as intptr like cupy's stream.ptr */

/* ---- library ---- */
int b200c_version(void);
const char* b200c_last_error(void);
const char* b200c_status_string(int status);
size_t b200c_dtype_size(int dtype);
int b200c_device_props(int device, b200c_props_t* out);
void b200c_default_config(b200c_config_t* cfg);

/* ---- communicator lifecycle ----
 * Replaces NcclCommunicator(world, uid, rank) (nccl_util.py:107-118; nccl_group.py:90) and the
 * Rendezvous around it (nccl_collective_group.py:29-118).  The rendezvous transport itself
 * (named actor / internal KV / torch store / Unix socket) lives on the host side; the library
 * only produces and consumes the bytes.
 *
 * Order: create -> export (publish) -> import x (world-1) -> [multicast: mc_create on rank 0,
 * mc_import elsewhere, mc_add_device everywhere, <barrier>, mc_bind everywhere, <barrier>]
 * -> ready.  Host-side barriers between the steps are the caller's job. */
int b200c_comm_create(int rank, int world, int device, const b200c_config_t* cfg, b200c_comm_t** out);
int b200c_comm_export(b200c_comm_t* comm, b200c_export_t* out);
int b200c_comm_import(b200c_comm_t* comm, int peer, const b200c_export_t* peer_export);
int b200c_comm_mc_create(b200c_comm_t* comm, int* fd_out);   /* rank 0 */
int b200c_comm_mc_import(b200c_comm_t* comm, int fd);        /* ranks != 0 */
int b200c_comm_mc_add_device(b200c_comm_t* comm);
int b200c_comm_mc_bind(b200c_comm_t* comm);
/* Drop the multicast mapping (called on every rank when any rank failed to bind). */
int b200c_comm_mc_disable(b200c_comm_t* comm);
int b200c_comm_ready(b200c_comm_t* comm);
/* Replaces comm.abort() (nccl_group.py:347-365): makes every kernel of this communicator that is
 * spinning on a peer flag give up; safe to call from another thread. */
int b200c_comm_abort(b200c_comm_t* comm);
int b200c_comm_destroy(b200c_comm_t* comm);
/* Non-blocking: returns B200C_OK, or the first error a kernel of this communicator recorded
 * (ETIMEOUT / EABORTED / EMISMATCH).  Reads host-pinned memory; does not synchronise. */
int b200c_comm_check(b200c_comm_t* comm);
int b200c_comm_rank(const b200c_comm_t* comm);
int b200c_comm_world(const b200c_comm_t* comm);
int b200c_comm_has_multicast(const b200c_comm_t* comm);
uint64_t b200c_comm_seq(const b200c_comm_t* comm);

/* Symmetric region: the same offset names the same logical buffer on every rank.  A tensor
 * living there takes the zero-copy paths (NVLS reads/writes it in place). */
void* b200c_comm_symmetric_base(b200c_comm_t* comm);
uint64_t b200c_comm_symmetric_bytes(const b200c_comm_t* comm);

/* Symmetric pool: allocator entry points in the shape torch.cuda.memory.CUDAPluggableAllocator expects
 * (alloc(size, device, stream) / free(ptr, size, device, stream)), carving 2 MiB-granular segments out of
 * the symmetric region of the communicator selected by b200c_pool_bind (one per process; NULL unbinds).
 * Tensors allocated from a torch.cuda.MemPool built on them are peer-mapped and multicast-bound, so
 * collectives on them are zero-copy.  First fit over a sorted free list: the same allocation sequence on
 * every rank yields the same offsets. */
int b200c_pool_bind(b200c_comm_t* comm);
void* b200c_pool_malloc(size_t size, int device, void* stream);
void b200c_pool_free(void* ptr, size_t size, int device, void* stream);

/* ---- collectives (K1-K7, K10-K13 in SURVEY.md §2d) ---- */

/* allReduce(sendptr, recvptr, count, dtype, op, stream): nccl_collective_group.py:181-188,
 * nccl_group.py:293-312.  send == recv (in place) is allowed. */
int b200c_allreduce(b200c_comm_t* comm, const void* send, void* recv, size_t count, int dtype,
                    int op, int algo, b200c_stream_t stream);

/* Fused gradient allreduce for the DDP bucket hook (K13): reads `count` elements of `dtype`
 * from every rank's bucket, moves `wire_dtype` over NVLink (FLOAT32 bucket + BFLOAT16 wire is
 * the bf16-compress case), accumulates in fp32 in rank order, multiplies by `scale`
 * (1/world for the mean) and writes `dtype` back in place.  One launch per piece; replaces
 * div_() + ncclAllReduce (+ to(bf16)/copy_() in bf16_compress_hook). */
int b200c_allreduce_scaled(b200c_comm_t* comm, const void* send, void* recv, size_t count, int dtype,
                           int wire_dtype, float scale, int algo, b200c_stream_t stream);

/* reduce(sendptr, recvptr, count, dtype, op, root, stream): nccl_collective_group.py:226-234.
 * Only `root` writes `recv`; other ranks' buffers are left untouched (gloo semantics,
 * torch_gloo_collective_group.py:170-179). */
int b200c_reduce(b200c_comm_t* comm, const void* send, void* recv, size_t count, int dtype, int op,
                 int root, b200c_stream_t stream);

/* broadcast(ptr, ptr, count, dtype, root, stream): nccl_collective_group.py:253-260. */
int b200c_broadcast(b200c_comm_t* comm, void* buf, size_t count, int dtype, int root,
                    b200c_stream_t stream);

/* allGather: nccl_collective_group.py:278-284 + the W copy_tensor calls of postprocess_fn
 * (:292-296).  `recv_ptrs` holds `world` device pointers (the caller's W output tensors, or
 * base + j*count*size for a contiguous output as in nccl_group.py:274-291); rank j's data lands
 * in recv_ptrs[j].  No flat temp buffer, no extra D2D copies. */
int b200c_allgather(b200c_comm_t* comm, const void* send, void* const* recv_ptrs, size_t count,
                    int dtype, b200c_stream_t stream);

/* reduceScatter: nccl_collective_group.py:319-326 + the W copy_tensor calls of preprocess_fn
 * (:334-337).  `send_ptrs[j]` is this rank's contribution to rank j (`count` elements each). */
int b200c_reducescatter(b200c_comm_t* comm, const void* const* send_ptrs, void* recv, size_t count,
                        int dtype, int op, b200c_stream_t stream);

/* Fused gradient mean as a reduceScatter (the FSDP gradient reduce-scatter, K13): `send_ptrs[j]`
 * is this rank's contribution to rank j (`count` elements of `dtype` each).  Every contribution is
 * rounded to `wire_dtype` and moved as `wire_dtype` (FLOAT32 buffers + BFLOAT16 / FLOAT16 wire, or
 * wire == dtype), the W contributions are summed in fp32 in rank order, multiplied once by `scale`
 * (1/world for the mean), rounded to `wire_dtype` and written to `recv` as `dtype`.  Buffers are
 * f32 / bf16 / f16, anything else is B200C_EUNSUPPORTED.  `recv` may alias send_ptrs[rank].
 * Pieces are sized by the staging capacity in wire bytes.  The wire is part of the op signature:
 * a peer that entered b200c_reducescatter (or another wire) instead gets B200C_EMISMATCH.  With one
 * rank only the wire rounding and the scale are applied. */
int b200c_reducescatter_scaled(b200c_comm_t* comm, const void* const* send_ptrs, void* recv, size_t count,
                               int dtype, int wire_dtype, float scale, b200c_stream_t stream);

/* send / recv: nccl_collective_group.py:355-363, 381-389; nccl_group.py:178-184, 217-237.
 * Sender writes the receiver's HBM (ring of slots) and raises a flag; receiver copies out. */
int b200c_send(b200c_comm_t* comm, const void* buf, size_t bytes, int peer, b200c_stream_t stream);
int b200c_recv(b200c_comm_t* comm, void* buf, size_t bytes, int peer, b200c_stream_t stream);

/* Multi-reader send: torch_tensor_accelerator_channel.py:586-590 sends the same tensor once per reader
 * ("TODO: If there are multiple readers, can replace with a broadcast").  One call delivers `bytes` to
 * every rank in `peers`; with a bound multicast object the payload leaves this GPU once (multimem.st)
 * and the NVSwitch replicates it.  Every reader receives with b200c_recv_multi(src = the sender).
 * A source rank multi-sends to ONE reader set for the lifetime of the communicator (ring positions are
 * counted per source); another reader set -> B200C_EUNSUPPORTED, use per-reader b200c_send.  With a
 * single reader, or a world of two, both calls are the pairwise b200c_send / b200c_recv. */
int b200c_send_multi(b200c_comm_t* comm, const void* buf, size_t bytes, const int* peers, int npeers,
                     b200c_stream_t stream);
int b200c_recv_multi(b200c_comm_t* comm, void* buf, size_t bytes, int src, b200c_stream_t stream);

/* barrier: nccl_collective_group.py:192-210 (an allreduce of [1] in the reference). */
int b200c_barrier(b200c_comm_t* comm, b200c_stream_t stream);

/* Profiling aid: set every flag of this rank's signal pad to `value`.  With value = 0x7fffffff every
 * wait of every later op is already satisfied, so ONE rank's kernel can run without its peers —
 * which is what Nsight Compute's kernel replay needs (it re-runs a kernel in isolation, so a kernel
 * that waits for a concurrently running peer kernel would never finish).  Results are garbage;
 * memory traffic and instruction mix are those of the real run.  The LL region is stamped with the
 * flag of the next LL op (one LL launch per call).  Never call it on a live group. */
int b200c_debug_fill_flags(b200c_comm_t* comm, uint32_t value);

/* ---- fused batch norm (training) over channels-last bf16 activations ----
 * A ResNet block's batch norm and what follows it, in one call per direction: x -> relu(bn(x)), or, with
 * `identity` set, x -> relu(bn(x) + identity).  Activations are bf16 rows of `channels` values (NHWC memory order,
 * m = N*H*W rows); weight, bias and the statistics are fp32 [channels].  The results are bit-identical to eager
 * torch's native channels-last batch norm (its statistics, running-statistics update, transform, backward reduce
 * and backward elementwise kernels) followed by the bf16 residual add and ReLU, and their backward.
 * `scratch` holds at least b200c_bn_scratch_bytes(channels) bytes, zero-filled before its first use.  Its
 * semaphores sit in a fixed region at its start that no call's staging overlaps, and every call leaves them at
 * zero, so one buffer, sized for the largest channel count, serves calls of any channel count.  Calls sharing a
 * scratch buffer must be ordered (one stream).  channels <= 131072; b200c_bn_scratch_bytes returns 0 outside
 * 1..131072.
 *
 * Forward: writes y, save_mean, save_invstd (1 / sqrt(biased var + eps)), updates running_mean / running_var
 * with `momentum` (unbiased variance) and adds 1 to *num_batches_tracked (may be NULL).  2 kernels.
 * Backward: from dy (the gradient of y), y and x writes dx, grad_weight and grad_bias; `dy_masked` (may be NULL)
 * receives the gradient of the ReLU's input, the identity branch's gradient.  2 kernels.
 *
 * The _mask variants (channels % 8 == 0 only; EINVAL otherwise, and for a NULL mask) replace the backward's
 * 2-byte read of y by a 1-bit read.  Forward: as b200c_bn_forward, and also writes `mask`, m * channels / 8 bytes:
 * element e = row * channels + channel is bit e % 8 of byte e / 8, set where y > 0 or y is NaN (the ReLU passes
 * the gradient).  Backward: as b200c_bn_backward with that mask in place of y.  `dy2` (may be NULL) is a second
 * gradient of y, for a y with two consumers: the kernels use bf16(float(dy) + float(dy2)), autograd's sum of the
 * two; with dy2 NULL, dy is used as it is.  2 kernels each.  b200c_bn_forward and b200c_bn_backward run the same
 * kernels without a mask and without dy2. */
size_t b200c_bn_scratch_bytes(int channels);
int b200c_bn_forward(const void* x, const void* identity, void* y, const float* weight, const float* bias,
                     float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                     float* save_invstd, int m, int channels, float momentum, float eps, void* scratch,
                     b200c_stream_t stream);
int b200c_bn_forward_mask(const void* x, const void* identity, void* y, uint8_t* mask, const float* weight,
                          const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked,
                          float* save_mean, float* save_invstd, int m, int channels, float momentum, float eps,
                          void* scratch, b200c_stream_t stream);
int b200c_bn_backward(const void* dy, const void* y, const void* x, void* dy_masked, void* dx, const float* weight,
                      const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int m,
                      int channels, void* scratch, b200c_stream_t stream);
int b200c_bn_backward_mask(const void* dy, const void* dy2, const uint8_t* mask, const void* x, void* dy_masked, void* dx,
                           const float* weight, const float* save_mean, const float* save_invstd, float* grad_weight,
                           float* grad_bias, int m, int channels, void* scratch, b200c_stream_t stream);

/* A block tail whose identity is a downsample branch's batch norm: y = relu(bn(x) + bn_ds(x_ds)), the two batch
 * norms' outputs each rounded to bf16 before the bf16 add, as eager torch computes
 * `out = bn3(conv3); out += downsample(x); relu(out)`.  x and x_ds have the same m rows of `channels`; each batch
 * norm has its own weight, bias, statistics, momentum and eps, with the results of b200c_bn_forward for each.
 * bn_ds(x_ds) is never written.  `mask` (may be NULL; channels % 8 == 0) as in b200c_bn_forward_mask.
 * Backward: both batch norms take g, the ReLU's gradient of dy (or of bf16(dy + dy2) with `dy2` set); writes dx,
 * dx_ds and both dweight / dbias, reading the mask, or y where mask is NULL.  g is not written.
 * `scratch` holds at least b200c_bn_dual_scratch_bytes(channels) bytes, with the contract of b200c_bn_scratch_bytes;
 * channels <= 65536 (0 outside 1..65536).  2 kernels per direction; every argument is checked before the first
 * launch. */
size_t b200c_bn_dual_scratch_bytes(int channels);
int b200c_bn_forward_dual(const void* x, const void* x_ds, void* y, uint8_t* mask, const float* weight, const float* bias,
                          float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                          float* save_invstd, float momentum, float eps, const float* weight_ds, const float* bias_ds,
                          float* running_mean_ds, float* running_var_ds, int64_t* num_batches_tracked_ds,
                          float* save_mean_ds, float* save_invstd_ds, float momentum_ds, float eps_ds, int m, int channels,
                          void* scratch, b200c_stream_t stream);
int b200c_bn_backward_dual(const void* dy, const void* dy2, const void* y, const uint8_t* mask, const void* x,
                           const void* x_ds, void* dx, void* dx_ds, const float* weight, const float* save_mean,
                           const float* save_invstd, float* grad_weight, float* grad_bias, const float* weight_ds,
                           const float* save_mean_ds, const float* save_invstd_ds, float* grad_weight_ds,
                           float* grad_bias_ds, int m, int channels, void* scratch, b200c_stream_t stream);

/* The ResNet stem, maxpool(relu(bn(x))) with torch's nn.MaxPool2d(3, stride=2, padding=1), over n images of h x w
 * rows (m = n * h * w), bit-identical to eager torch's batch norm, ReLU and channels-last max_pool2d.  Scratch,
 * statistics and their contract are those of b200c_bn_forward; any channel count.
 * Forward: y receives the pooled output, n * oh * ow rows with oh = (h - 1) / 2 + 1, ow = (w - 1) / 2 + 1, and
 * `argmax` one byte per pooled element: the position (row * 3 + column) in its window of the element it selected
 * (rows first, the first maximum and the last NaN win), or 255 where the maximum is 0 and the ReLU passes no
 * gradient.  relu(bn(x)) itself is not written.  2 kernels.
 * Backward: from dy (the gradient of y), argmax and x writes dx, grad_weight and grad_bias; `g` (m rows, required)
 * receives the batch norm's output gradient, torch's max_pool2d backward followed by the ReLU's.  2 kernels. */
int b200c_bn_forward_pool(const void* x, void* y, uint8_t* argmax, const float* weight, const float* bias,
                          float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                          float* save_invstd, int n, int h, int w, int channels, float momentum, float eps, void* scratch,
                          b200c_stream_t stream);
int b200c_bn_backward_pool(const void* dy, const uint8_t* argmax, const void* x, void* g, void* dx, const float* weight,
                           const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int n,
                           int h, int w, int channels, void* scratch, b200c_stream_t stream);

/* VGG-BN's stage end, maxpool(relu(bn(x))) with torch's nn.MaxPool2d(2, stride=2) (floor mode), over n images of h x w
 * rows (m = n * h * w), bit-identical to eager torch's batch norm, ReLU and channels-last max_pool2d.  Scratch,
 * statistics and their contract are those of b200c_bn_forward (b200c_bn_scratch_bytes(channels)).  h >= 2, w >= 2,
 * channels 1..131072 and n * h * w * channels below 2^31; bf16 operands sit on the 2-byte grid and fp32 ones on the
 * 4-byte grid (8 channels per thread where channels % 8 == 0 and every operand is on the 16-byte grid).  Every
 * argument is checked before the first launch.
 * Forward: y receives the pooled output, n * (h / 2) * (w / 2) channels-last rows (an odd h or w leaves its last row
 * or column out of every window), and `argmax` one byte per pooled element: the position ((row & 1) * 2 + (column &
 * 1)) in its window of the element it selected (rows first, the first maximum and the last NaN win), or 255 where the
 * maximum is <= 0 and the ReLU passes no gradient.  relu(bn(x)) itself is not written.  2 kernels.
 * Backward: from dy (the gradient of y, channels-last), argmax and x writes dx, grad_weight and grad_bias.  An element's
 * batch-norm output gradient is its window's dy as it is where the window selected it, else +0; it is rebuilt by both
 * kernels and never written.  2 kernels.
 * b200c_bn_infer_pool2: eval, y = max_pool2d(relu(bn(x)), 2, 2) from the running statistics, fp32 (param_bf16 0) or
 * bf16 (1) parameters, as b200c_bn_infer; writes the pooled rows only (no argmax).  1 kernel. */
int b200c_bn_forward_pool2(const void* x, void* y, uint8_t* argmax, const float* weight, const float* bias,
                           float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                           float* save_invstd, int n, int h, int w, int channels, float momentum, float eps, void* scratch,
                           b200c_stream_t stream);
int b200c_bn_backward_pool2(const void* dy, const uint8_t* argmax, const void* x, void* dx, const float* weight,
                            const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int n,
                            int h, int w, int channels, void* scratch, b200c_stream_t stream);
int b200c_bn_infer_pool2(const void* x, void* y, const void* weight, const void* bias, const void* running_mean,
                         const void* running_var, int param_bf16, float eps, int n, int h, int w, int channels,
                         b200c_stream_t stream);

/* ---- fused batch norm (eval) over channels-last bf16 activations ----
 * An eval-mode batch norm with its running statistics and what follows it in a ResNet, in one kernel, bit-identical
 * to eager torch's batch_norm (train = false: invstd = rsqrt(float(running_var) + eps), then w * (x - mean) * invstd
 * + bias) followed by the bf16 ops after it.  weight, bias, running_mean and running_var are [channels] of fp32, or of
 * bf16 with param_bf16 = 1 (widened to fp32, as torch widens them).  Only y is written: no running statistic, no
 * num_batches_tracked, no mask and no scratch.  m >= 1 rows of `channels` (NHWC memory order), fewer than 2^31
 * elements; every argument is checked before the launch.  1 kernel each.
 *
 * b200c_bn_infer: y = relu(bn(x)), or with `identity` (may be NULL) y = relu(bn(x) + identity).
 * b200c_bn_infer_dual: y = relu(bn(x) + bn_ds(x_ds)), a block tail whose identity is a downsample branch's batch norm;
 * each batch norm has its own parameters and eps, of the one parameter type.
 * b200c_bn_infer_pool: the stem, y = max_pool2d(relu(bn(x)), 3, stride 2, padding 1) over n images of h x w rows,
 * selected as b200c_bn_forward_pool selects; writes the pooled rows only (no argmax). */
int b200c_bn_infer(const void* x, const void* identity, void* y, const void* weight, const void* bias, const void* running_mean,
                   const void* running_var, int param_bf16, float eps, int m, int channels, b200c_stream_t stream);
int b200c_bn_infer_dual(const void* x, const void* x_ds, void* y, const void* weight, const void* bias, const void* running_mean,
                        const void* running_var, float eps, const void* weight_ds, const void* bias_ds, const void* running_mean_ds,
                        const void* running_var_ds, float eps_ds, int param_bf16, int m, int channels, b200c_stream_t stream);
int b200c_bn_infer_pool(const void* x, void* y, const void* weight, const void* bias, const void* running_mean,
                        const void* running_var, int param_bf16, float eps, int n, int h, int w, int channels,
                        b200c_stream_t stream);

/* ---- fused batch norm followed by ReLU6, SiLU or Hardswish (torchvision's Conv2dNormActivation) ----
 * y = act(bn(x)) over channels-last bf16 activations, bit-identical to eager torch's batch norm followed by its
 * activation module: the batch norm's output t is rounded to bf16, the activation computed in fp32 as torch's CUDA
 * kernels compute it and rounded to bf16.  t itself is never written.  `act` is a b200c_act_t; EINVAL for any other.
 * Channels 1..131072, m >= 1 rows, fewer than 2^31 elements; every argument is checked before the first launch.
 *
 * b200c_bn_forward_act: the training forward of b200c_bn_forward (statistics, running statistics, num_batches_tracked,
 * scratch of b200c_bn_scratch_bytes(channels)) without identity, writing act(t).  2 kernels.
 * b200c_bn_backward_act: from dy (the gradient of y), x, weight, bias and the saved statistics, writes dx, grad_weight
 * and grad_bias; the activation's gradient g is derived from dy and t recomputed from x, as torch's
 * silu_backward / hardswish_backward / hardtanh_backward derive it from the saved t, rounded to bf16, and written to
 * `g` (m rows, required), which the batch norm's elementwise backward reads.  2 kernels.
 * b200c_bn_infer_act: the eval site of b200c_bn_infer without identity, writing act(t).  1 kernel. */
typedef enum { B200C_ACT_RELU6 = 1, B200C_ACT_SILU = 2, B200C_ACT_HARDSWISH = 3 } b200c_act_t;
int b200c_bn_forward_act(const void* x, void* y, const float* weight, const float* bias, float* running_mean, float* running_var,
                         int64_t* num_batches_tracked, float* save_mean, float* save_invstd, int act, int m, int channels,
                         float momentum, float eps, void* scratch, b200c_stream_t stream);
int b200c_bn_backward_act(const void* dy, const void* x, void* g, void* dx, const float* weight, const float* bias, const float* save_mean,
                          const float* save_invstd, float* grad_weight, float* grad_bias, int act, int m, int channels, void* scratch,
                          b200c_stream_t stream);
int b200c_bn_infer_act(const void* x, void* y, const void* weight, const void* bias, const void* running_mean, const void* running_var,
                       int param_bf16, float eps, int act, int m, int channels, b200c_stream_t stream);

/* ---- fused batch norm followed by a residual add, with or without stochastic depth (inverted-residual blocks) ----
 * y = bn(x), y = bn(x) + identity or y = stochastic_depth(bn(x)) + identity over channels-last bf16 activations,
 * bit-identical to eager torch: the batch norm's output t is rounded to bf16; stochastic depth multiplies it by
 * noise[n] (bf16, one value per sample n = row / rows_per_sample, as torchvision's "row" mode builds it) and rounds to
 * bf16; the add sums in fp32 and rounds to bf16.  `identity` may be null (no add); `noise` may be null (no stochastic
 * depth) and needs an identity and a rows_per_sample >= 1 that divides m.  Channels 1..131072, m >= 1 rows, fewer than
 * 2^31 elements; every argument is checked before the first launch.
 *
 * b200c_bn_forward_res: the training forward of b200c_bn_forward (statistics, running statistics,
 * num_batches_tracked, scratch of b200c_bn_scratch_bytes(channels)) without ReLU.  2 kernels.
 * b200c_bn_backward_res: from dy (the gradient of y), x, weight and the saved statistics, writes dx, grad_weight and
 * grad_bias.  The identity's gradient is dy itself.  With noise, g = bf16(dy * noise[n]) (stochastic depth's backward)
 * is written to `g` (m rows, required then, null otherwise), which the batch norm's elementwise backward reads.
 * 2 kernels.
 * b200c_bn_infer_res: the eval site, y = bf16(bn(x)) or bf16(bf16(bn(x)) + identity) (stochastic depth is the
 * identity in eval), with weight, bias and running statistics of fp32, or of bf16 with param_bf16.  1 kernel. */
int b200c_bn_forward_res(const void* x, const void* identity, const void* noise, int rows_per_sample, void* y, const float* weight,
                         const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                         float* save_invstd, int m, int channels, float momentum, float eps, void* scratch, b200c_stream_t stream);
int b200c_bn_backward_res(const void* dy, const void* noise, int rows_per_sample, const void* x, void* g, void* dx, const float* weight,
                          const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int m, int channels,
                          void* scratch, b200c_stream_t stream);
int b200c_bn_infer_res(const void* x, const void* identity, void* y, const void* weight, const void* bias, const void* running_mean,
                       const void* running_var, int param_bf16, float eps, int m, int channels, b200c_stream_t stream);

/* ---- fused batch norm and ReLU over a channel concatenation (DenseNet) ----
 * y = relu(bn(cat(segs, 1))) over channels-last bf16 activations without the cat: segment s is bf16 [m][seg_channels[s]]
 * (channels-last rows, m = N * H * W alike for every segment), with seg_channels[s] % 8 == 0 and segs[s] on the 16-byte
 * grid; the nsegs (1..64) segments' channels sum to `channels` (1..131072); m * channels < 2^31.  Results have the bits
 * of b200c_bn_forward_mask / b200c_bn_backward_mask / b200c_bn_infer over the concatenated tensor, which are eager
 * torch's.  y, mask, dy and dx are whole [m][channels] tensors; y, dy and dx sit on the 16-byte grid.  Every argument
 * is checked before the first launch.
 *
 * b200c_bn_forward_cat: the training forward of b200c_bn_forward_mask (statistics, running statistics,
 * num_batches_tracked, mask bits, scratch of b200c_bn_scratch_bytes(channels)), m >= 2.  2 kernels.
 * b200c_bn_backward_cat: from dy (the gradient of y), the mask, the segments, weight and the saved statistics, writes
 * the whole dx, grad_weight and grad_bias; a segment's gradient is its channels of dx.  2 kernels.
 * b200c_bn_infer_cat: the eval site of b200c_bn_infer without identity, with weight, bias and running statistics of
 * fp32, or of bf16 with param_bf16.  1 kernel. */
int b200c_bn_forward_cat(const void* const* segs, const int* seg_channels, int nsegs, void* y, uint8_t* mask, const float* weight,
                         const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                         float* save_invstd, int m, int channels, float momentum, float eps, void* scratch, b200c_stream_t stream);
int b200c_bn_backward_cat(const void* dy, const uint8_t* mask, const void* const* segs, const int* seg_channels, int nsegs, void* dx,
                          const float* weight, const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias,
                          int m, int channels, void* scratch, b200c_stream_t stream);
int b200c_bn_infer_cat(const void* const* segs, const int* seg_channels, int nsegs, void* y, const void* weight, const void* bias,
                       const void* running_mean, const void* running_var, int param_bf16, float eps, int m, int channels,
                       b200c_stream_t stream);

/* ---- fused batch norm and ReLU into a channel slice of a wider output (Inception, GoogLeNet) ----
 * y = relu(bn(x)) over a branch's channels-last bf16 x of [m][channels] (channels 1..131072, a multiple of 8), written
 * into a channel slice of a wider channels-last output: row r of the branch lands at y + r * ldy, y pointing at the
 * slice's first channel, so the branch outputs of a concatenation are written in place and never copied.  ldy (and
 * the backward's lddy) is a multiple of 8 of at least `channels`, with m * ldy and m * channels below 2^31.  x, y, dy
 * and dx sit on the 16-byte grid; the mask is the branch's own m * channels / 8 bytes.  Nothing outside the slice is
 * written.  Results have the bits of b200c_bn_forward_mask / b200c_bn_backward_mask / b200c_bn_infer over the branch,
 * which are eager torch's.  Every argument is checked before the first launch.
 *
 * b200c_bn_forward_slice: the training forward of b200c_bn_forward_mask without identity (statistics, running
 * statistics, num_batches_tracked, mask bits, scratch of b200c_bn_scratch_bytes(channels)), m >= 2.  2 kernels.
 * b200c_bn_backward_slice: from dy (the gradient of y, rows lddy apart), the mask, x, weight and the saved statistics,
 * writes dx, grad_weight and grad_bias.  2 kernels.
 * b200c_bn_infer_slice: the eval site of b200c_bn_infer without identity, with weight, bias and running statistics of
 * fp32, or of bf16 with param_bf16, m >= 1.  1 kernel. */
int b200c_bn_forward_slice(const void* x, void* y, int ldy, uint8_t* mask, const float* weight, const float* bias, float* running_mean,
                           float* running_var, int64_t* num_batches_tracked, float* save_mean, float* save_invstd, int m, int channels,
                           float momentum, float eps, void* scratch, b200c_stream_t stream);
int b200c_bn_backward_slice(const void* dy, int lddy, const uint8_t* mask, const void* x, void* dx, const float* weight,
                            const float* save_mean, const float* save_invstd, float* grad_weight, float* grad_bias, int m, int channels,
                            void* scratch, b200c_stream_t stream);
int b200c_bn_infer_slice(const void* x, void* y, int ldy, const void* weight, const void* bias, const void* running_mean,
                         const void* running_var, int param_bf16, float eps, int m, int channels, b200c_stream_t stream);

/* ---- fused batch norms and ReLU into ShuffleNetV2's shuffled block output ----
 * The end of torchvision's ShuffleNetV2 InvertedResidual, channel_shuffle(torch.cat((a, relu(bn(t))), 1), 2), with a
 * either the block input's first half x1 (stride 1: one batch norm) or relu(bn_u(u)) (stride 2: a second batch norm
 * on u), written straight into its bf16 output y, contiguous NCHW [n][2 * channels][hw]: channel 2c is a's channel c,
 * channel 2c + 1 is relu(bn(t))'s.  t and u are channels-last bf16 [m][channels], m = n * hw, any channels in
 * 1..65536 with n * 2 * channels * hw below 2^31; x1 is NCHW planes, element (n, c, p) at x1 + n * x1_stride + c * hw +
 * p.  Exactly one of x1 and u is given.  Every result has the bits of eager torch's modules, cat and channel_shuffle
 * (bf16 autocast); no branch output or concatenation is written.
 *
 * Each batch norm's ReLU predicate is kept as bits in b200c_bn_shuffle_mask_bytes(m, channels) bytes (ceil(channels /
 * 8) per row; 0 for a bad shape); the layout is private to these calls.  A site's scratch is b200c_bn_scratch_bytes
 * (one batch norm) or b200c_bn_dual_scratch_bytes (two) of channels.
 *
 * b200c_bn_forward_shuffle: training forward, m >= 2: statistics, running statistics and num_batches_tracked (may be
 *   null) of each batch norm, y and the masks.  2 launches.
 * b200c_bn_backward_shuffle: from dy, y's gradient as channels-last bf16 [m][2 * channels] on the 4-byte grid, each
 *   batch norm's mask, input, weight and saved statistics: dt (and du), grad_weight and grad_bias.  u null: the
 *   one-batch-norm form, whose x1 gradient is dy's even channels.  2 launches.
 * b200c_bn_infer_shuffle: eval, m >= 1, weight, bias and running statistics all fp32 (param_bf16 0) or all bf16 (1):
 *   y alone.  1 launch. */
size_t b200c_bn_shuffle_mask_bytes(int m, int channels);
int b200c_bn_forward_shuffle(const void* x1, int x1_stride, const void* u, uint8_t* mask_u, const float* weight_u, const float* bias_u,
                             float* running_mean_u, float* running_var_u, int64_t* num_batches_tracked_u, float* save_mean_u,
                             float* save_invstd_u, float momentum_u, float eps_u, const void* t, uint8_t* mask, const float* weight,
                             const float* bias, float* running_mean, float* running_var, int64_t* num_batches_tracked, float* save_mean,
                             float* save_invstd, float momentum, float eps, void* y, int n, int hw, int channels, void* scratch,
                             b200c_stream_t stream);
int b200c_bn_backward_shuffle(const void* dy, const void* u, const uint8_t* mask_u, void* du, const float* weight_u, const float* save_mean_u,
                              const float* save_invstd_u, float* grad_weight_u, float* grad_bias_u, const void* t, const uint8_t* mask,
                              void* dt, const float* weight, const float* save_mean, const float* save_invstd, float* grad_weight,
                              float* grad_bias, int m, int channels, void* scratch, b200c_stream_t stream);
int b200c_bn_infer_shuffle(const void* x1, int x1_stride, const void* u, const void* weight_u, const void* bias_u, const void* running_mean_u,
                           const void* running_var_u, float eps_u, const void* t, const void* weight, const void* bias,
                           const void* running_mean, const void* running_var, float eps, void* y, int param_bf16, int n, int hw,
                           int channels, b200c_stream_t stream);

/* ---- squeeze-and-excitation (torchvision's SqueezeExcitation without its squeeze path) ----
 * Over channels-last bf16 activations x, y, dy, dx of n samples, hw = H * W rows per sample and `channels` channels
 * ([n][hw][channels]), and bf16 per-sample vectors pooled, s, ds, gp of [n][channels]; bit-identical to eager torch:
 *
 * b200c_se_pool: pooled = x.mean((-1, -2)) = bf16(sum_hw float(x) * factor), factor = float(n * c) / (n * c * hw), summed
 * in the order of torch's reduce kernel for that tensor: its launch follows from the shape, x's address and the
 * current device's multiProcessorCount and maxThreadsPerMultiProcessor.  1 kernel.
 * b200c_se_scale: y = bf16(float(s[n, c]) * float(x)).  1 kernel.
 * b200c_se_backward_reduce: ds = bf16(sum_hw float(bf16(float(dy) * float(x)))), summed as torch sums a freshly allocated
 * product tensor of x's shape (the gradient of s in y = s * x); with hw == 1 torch reduces nothing and ds is that
 * product itself, -0.0 included.  1 kernel.
 * b200c_se_backward_elemt: dx = bf16(float(bf16(float(dy) * float(s))) + float(bf16(float(gp) * (1 / float(hw))))), the
 * gradient of x from y = s * x plus the mean's, gp being pooled's gradient.  1 kernel.
 *
 * n, channels, hw >= 1 with n * channels * hw < 2^31; the reducing calls also reject channels == 1 with hw > 1 (torch
 * reduces that along the fastest dimension, another order).  Torch sums in one launch, the order restated here, up to
 * 2^30 elements.  The reducing calls take `scratch` of at least b200c_se_scratch_bytes(n, channels, hw) bytes
 * (`scratch_bytes` its size), zero-filled before its first use; every call leaves its semaphores at zero, so one buffer
 * of the largest size serves every site on one stream.  b200c_se_scratch_bytes returns 0 for a bad shape.  Every
 * argument is checked before the launch. */
size_t b200c_se_scratch_bytes(int n, int channels, int hw);
int b200c_se_pool(const void* x, void* pooled, int n, int channels, int hw, void* scratch, size_t scratch_bytes, b200c_stream_t stream);
int b200c_se_scale(const void* x, const void* s, void* y, int n, int channels, int hw, b200c_stream_t stream);
int b200c_se_backward_reduce(const void* dy, const void* x, void* ds, int n, int channels, int hw, void* scratch, size_t scratch_bytes,
                             b200c_stream_t stream);
int b200c_se_backward_elemt(const void* dy, const void* s, const void* gp, void* dx, int n, int channels, int hw,
                            b200c_stream_t stream);

/* Sync batch norm: torch.nn.SyncBatchNorm's training-mode forward and backward over the ranks of `comm`, with the
 * same fusions as the calls above, bit-identical to torch's sync functions (batch_norm_stats,
 * batch_norm_gather_stats_with_counts, batch_norm_elemt, batch_norm_backward_reduce, batch_norm_backward_elemt)
 * whose all_gather stacks the ranks in order and whose all_reduce folds them in rank order.  Every rank calls both
 * functions for every site, in the same order, with its own rows: `m` may differ between ranks and may be 0 (the
 * rank then contributes count 0 and zero sums, and its dweight / dbias are written as zeros; torch's SyncBatchNorm
 * has no gradient there, which is what fused_norm returns for such a rank).
 *
 * `relu` != 0: y = relu(bn(x)) or, with `identity`, relu(bn(x) + identity), as b200c_bn_forward; `mask` (may be
 * NULL; channels % 8 == 0) as in b200c_bn_forward_mask.  relu == 0: y = bn(x); identity, mask, dy2 and dy_masked
 * must then be NULL.
 *
 * Forward: local statistics -> b200c_allgather of [mean, invstd, count] (2 * channels + 1 floats) -> merge of the
 * ranks with count >= 1 -> transform, in stream order.  Writes save_mean / save_invstd (the global statistics),
 * norm_fct (one float: 1 / the global row count, which the backward reads), y and mask, updates running_mean /
 * running_var with the unbiased global variance and adds 1 to num_batches_tracked (may be NULL).
 * Backward: local sums of g and g * (x - mean) and dweight / dbias (kept local, as torch keeps them) ->
 * b200c_allreduce SUM of the 2 * channels sums -> dx (and dy_masked as in b200c_bn_backward).
 *
 * `scratch` holds at least b200c_bn_sync_scratch_bytes(channels, world) bytes, zero-filled before its first use,
 * with the same contract as b200c_bn_scratch_bytes: it serves sites of any channel count on one stream, and its
 * semaphores are left at zero.  b200c_bn_sync_scratch_bytes returns 0 for channels outside 1..131072 or world
 * outside 1..8.  Every argument is checked before the first launch. */
size_t b200c_bn_sync_scratch_bytes(int channels, int world);
int b200c_bn_sync_forward(b200c_comm_t* comm, const void* x, const void* identity, void* y, uint8_t* mask, int relu,
                          const float* weight, const float* bias, float* running_mean, float* running_var,
                          int64_t* num_batches_tracked, float* save_mean, float* save_invstd, float* norm_fct, int m,
                          int channels, float momentum, float eps, void* scratch, b200c_stream_t stream);
int b200c_bn_sync_backward(b200c_comm_t* comm, const void* dy, const void* dy2, const void* y, const uint8_t* mask, int relu,
                           const void* x, void* dy_masked, void* dx, const float* weight, const float* save_mean,
                           const float* save_invstd, const float* norm_fct, float* grad_weight, float* grad_bias, int m,
                           int channels, void* scratch, b200c_stream_t stream);

/* Launch statistics (bench.py's gpu_launches claim). */
uint64_t b200c_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200COLL_H_ */
