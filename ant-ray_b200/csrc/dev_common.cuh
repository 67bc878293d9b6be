// Device-side building blocks of the peer-memory collectives.
//
// Memory model notes (PTX ISA, scope .sys):
//  * data moves with weak 16-byte ld/st; a block publishes them with
//        __syncthreads();  (CTA-scope happens-before from every thread to the signaller)
//        st.release.sys    (cumulative: covers the other threads' earlier stores)
//    and a consumer observes them with ld.acquire.sys followed by __syncthreads().
//  * flags are monotonically increasing 32-bit sequence numbers (never reset), compared with
//    a signed difference so wrap-around is harmless.
//  * peer (NVLink) loads bypass the local L2 but may allocate in L1; staging is re-used every
//    second op, so every read of
//    staging / peer memory is an L1-bypassing ld.volatile / ld.relaxed.sys.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200coll.h"

namespace b200c {

constexpr int kMaxRanks = B200C_MAX_RANKS;
constexpr int kMaxBlocks = 2048;
constexpr int kThreads = 512;

// ---- arena layout (identical on every rank; offsets in bytes from the arena base) ----
constexpr size_t kPadBytes = 2ull << 20;                      // signal pad = one VMM granule
constexpr size_t kOffFlagA = 0;                               // u32 [kMaxBlocks][8]
constexpr size_t kOffFlagB = kOffFlagA + kMaxBlocks * 8 * 4;  // u32 [kMaxBlocks][8]
constexpr size_t kOffArrive = kOffFlagB + kMaxBlocks * 8 * 4; // u32 [8]   arrive[src] = seq
constexpr size_t kOffOpSig = kOffArrive + 256;                // u64 [2][8] opsig[seq&1][src] = seq << 32 | signature (block 0)
constexpr size_t kOffPipeA = kOffOpSig + 256;                 // u32 [kMaxBlocks][8]  pipelined kernels: sub-tile staged in
constexpr size_t kOffPipeB = kOffPipeA + kMaxBlocks * 8 * 4;  // u32 [kMaxBlocks][8]  pipelined kernels: sub-tile reduced
constexpr size_t kOffP2PReady = kOffPipeB + kMaxBlocks * 8 * 4;  // u32 [8 src][kMaxCells]
constexpr int kMaxCells = 1024;
constexpr size_t kOffP2PAck = kOffP2PReady + 8 * kMaxCells * 4;  // u32 [8 dst][kMaxCells]
constexpr size_t kOffMReady = kOffP2PAck + 8 * kMaxCells * 4;  // u32 [8 src][kMaxCells]  multi-reader ring: cell ready (on each reader)
constexpr size_t kOffMAck = kOffMReady + 8 * kMaxCells * 4;    // u32 [8 dst][kMaxCells]  multi-reader ring: cell consumed (on the source)
constexpr size_t kOffLaneIn = kOffMAck + 8 * kMaxCells * 4;     // u32 [kMaxBlocks lanes][8 copy CTAs]  lane kernel: "my share of round q is staged" (local)
constexpr size_t kPadUsed = kOffLaneIn + kMaxBlocks * 8 * 4;
static_assert(kPadUsed <= kPadBytes, "signal pad overflow");

// What a failed wait was waiting for (Status::err_phase; b200c_comm_check names them in this order).
// kWaitFlagA / kWaitFlagB also cover the round flags pipeA / pipeB and the lane kernel's laneIn.
enum WaitPhase : int { kWaitArrive, kWaitFlagA, kWaitFlagB, kWaitP2PReady, kWaitP2PAck, kWaitLL, kNumWaitPhases };

// host-pinned, device-mapped status block
struct Status {
  volatile int abort_flag;   // host sets to 1: every spinning kernel gives up
  volatile int error;        // first error recorded by a kernel (b200c_status_t), 0 = none
  volatile unsigned err_seq; // sequence number of the op that failed
  volatile int err_peer;     // peer the kernel was waiting for
  volatile int err_phase;    // WaitPhase
  volatile unsigned err_a, err_b;  // mismatch: signature seen / expected
};

struct DevComm {
  int rank, world;
  char* arena[kMaxRanks];   // arena[rank] is this rank's own mapping
  char* mc_arena;           // multicast mapping of the arenas (nullptr when unavailable)
  Status* status;           // device pointer of the mapped status block
  unsigned long long timeout_ns;
  size_t staging_bytes;     // one half
  size_t off_staging;       // arena offset of half 0 (half 1 follows)
  size_t off_p2p;           // arena offset of the p2p rings [8 src][cells][cell_bytes]
  size_t p2p_cell_bytes;
  int p2p_cells;
  size_t off_mring;         // arena offset of the multi-reader rings [8 src][mcells][cell_bytes]
  int mcells;
  size_t off_ll;            // arena offset of the LL (packed data+flag) region: [2 halves][8 src][ll_words] u64
  size_t ll_words;          // 32-bit payload words per source slot (one u64 {data, flag} each)
};

struct CollArgs {
  DevComm c;
  const void* in;
  void* out;
  size_t n;        // elements in this piece
  size_t chunk;    // elements per rank chunk (multiple of the 16-byte vector width)
  size_t tile;     // elements per granule (multiple of the 16-byte vector width).  Block b owns granules
                   // b, b + grid, b + 2*grid, ... of every rank chunk (block-cyclic: at any time the grid
                   // touches one contiguous window of each chunk, which keeps DRAM pages / TLB entries hot on
                   // the serving side of peer and multimem reads)
  uint32_t seq;    // this op's sequence number (>= 1)
  uint32_t sig;    // op signature for mismatch detection
  int root;
  int has_scale;
  float scale;
  uint32_t pipe_base;  // round-pipelined kernels: flag value of round q is pipe_base + q + 1
  uint32_t ll_seq;     // LL kernels: per-communicator LL op counter (flag value; half = ll_seq & 1)
  int lane_copy;       // lane kernel: copy CTAs per lane (each lane = 1 switch CTA + lane_copy copy CTAs)
  int symmetric;   // NVLS: in/out already live at the same offset of the symmetric region
  size_t sym_off;  // arena offset of that buffer
  const void* in_ptrs[kMaxRanks];
  void* out_ptrs[kMaxRanks];
};

// ---------------------------------------------------------------------------------------------
// scoped loads / stores
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// 16-byte L1-bypassing load (staging written by peers, or peer memory over NVLink)
__device__ __forceinline__ uint4 ld_bypass16(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
// predicated form: a single @p LDG, no branch — keeps a compile-time-indexed batch of loads in registers
// when one of them (the rank's own slot) has to be skipped at run time
__device__ __forceinline__ uint4 ld_bypass16_if(const void* p, bool cond) {
  uint4 v = make_uint4(0, 0, 0, 0);
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.s32 q, %5, 0;\n\t@q ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];\n\t}"
      : "+r"(v.x), "+r"(v.y), "+r"(v.z), "+r"(v.w)
      : "l"(p), "r"((int)cond)
      : "memory");
  return v;
}
template <int N> struct RawInt;
template <> struct RawInt<1> { using type = uint8_t; };
template <> struct RawInt<2> { using type = uint16_t; };
template <> struct RawInt<4> { using type = uint32_t; };
template <> struct RawInt<8> { using type = uint64_t; };
template <typename T>
__device__ __forceinline__ T ld_bypass(const T* p) {
  using R = typename RawInt<sizeof(T)>::type;
  R raw = *reinterpret_cast<const volatile R*>(p);
  T v;
  memcpy(&v, &raw, sizeof(T));
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------------------------------------
// bounded wait.  One thread per awaited flag.  Returns false on abort / timeout (and records it).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void record_error(Status* st, int code, uint32_t seq, int peer, WaitPhase phase) {
  if (st->error == 0) { st->error = code; st->err_seq = seq; st->err_peer = peer; st->err_phase = phase; }
}
static __device__ __noinline__ bool wait_slow(const uint32_t* flag, uint32_t seq, Status* st, unsigned long long timeout_ns,
                                       int peer, WaitPhase phase) {
  unsigned long long t0 = globaltimer_ns();
  unsigned spins = 0;
  for (;;) {
    if ((int32_t)(ld_acquire_sys(flag) - seq) >= 0) return true;
    if ((++spins & 0xff) == 0) {
      if (st->abort_flag) { record_error(st, B200C_EABORTED, seq, peer, phase); return false; }
      if (globaltimer_ns() - t0 > timeout_ns) {
        record_error(st, B200C_ETIMEOUT, seq, peer, phase);
        st->abort_flag = 1;  // the op has failed: let this rank's other blocks (and queued kernels) stop waiting too
        return false;
      }
      __nanosleep(64);
    }
  }
}
__device__ __forceinline__ bool wait_flag(const uint32_t* flag, uint32_t seq, const DevComm& c, int peer,
                                          WaitPhase phase) {
#pragma unroll 1
  for (int i = 0; i < 64; i++)
    if ((int32_t)(ld_acquire_sys(flag) - seq) >= 0) return true;
  return wait_slow(flag, seq, c.status, c.timeout_ns, peer, phase);
}

// Flag [slot][src] of the u32 [kMaxBlocks][8] flag array at pad offset `off` in rank x's arena.  The slot is
// the block index (the lane in the lane kernel); arrive[8] is an array of one slot.
__device__ __forceinline__ uint32_t* flag_at(const DevComm& c, int x, size_t off, size_t slot, int src) {
  return reinterpret_cast<uint32_t*>(c.arena[x] + off) + slot * 8 + src;
}

// All threads call.  Thread t < world, t != rank waits for own flag [block][t] >= seq of the array at
// `flag_off`.  Returns block-uniform ok.
__device__ __forceinline__ bool block_wait_all(size_t flag_off, uint32_t seq, const DevComm& c, WaitPhase phase) {
  const uint32_t* f = flag_at(c, c.rank, flag_off, blockIdx.x, 0);
  int ok = 1;
  int t = threadIdx.x;
  if (t < c.world && t != c.rank) ok = wait_flag(f + t, seq, c, t, phase);
  return __syncthreads_and(ok) != 0;
}
// wait for a single peer's flag
__device__ __forceinline__ bool block_wait_one(const uint32_t* flag, uint32_t seq, const DevComm& c, int peer,
                                               WaitPhase phase) {
  int ok = 1;
  if (threadIdx.x == 0) ok = wait_flag(flag, seq, c, peer, phase);
  return __syncthreads_and(ok) != 0;
}
// All threads call (contains the publishing __syncthreads).  Writes `seq` into slot
// [block][rank] of the given flag array in every peer's pad.
__device__ __forceinline__ void block_signal_all(size_t flag_off, uint32_t seq, const DevComm& c) {
  __syncthreads();
  int t = threadIdx.x;
  if (t < c.world && t != c.rank) st_release_sys(flag_at(c, t, flag_off, blockIdx.x, c.rank), seq);
}
__device__ __forceinline__ void block_signal_one(size_t flag_off, uint32_t seq, const DevComm& c, int peer) {
  __syncthreads();
  if (threadIdx.x == 0) st_release_sys(flag_at(c, peer, flag_off, blockIdx.x, c.rank), seq);
}

// Mismatch detection (diagnostic).  Each rank announces (seq, signature) to every peer in one atomic
// 8-byte store.  A peer's announcement is compared only if it carries exactly this op's sequence
// number; anything else (the peer is still behind, or — a producer-only rank such as a broadcast
// root — already ahead) is not evidence of a mismatch and is ignored, so the check can never raise a
// false alarm.  On mismatch the communicator is poisoned: the error is recorded and the abort flag
// raised so this rank's other blocks stop waiting.
__device__ __forceinline__ void announce_signature(const CollArgs& a, int peer) {
  const DevComm& c = a.c;
  unsigned long long* sig = reinterpret_cast<unsigned long long*>(c.arena[peer] + kOffOpSig) + (a.seq & 1) * 8 + c.rank;
  unsigned long long tagged = ((unsigned long long)a.seq << 32) | a.sig;  // one atomic 8-byte store
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(sig), "l"(tagged) : "memory");
}
// Compares what `peer` announced with this op; a mismatch is recorded and raises the abort flag.
__device__ __forceinline__ void compare_signature(const CollArgs& a, int peer, WaitPhase phase) {
  const DevComm& c = a.c;
  const unsigned long long* slot = reinterpret_cast<const unsigned long long*>(c.arena[c.rank] + kOffOpSig) + (a.seq & 1) * 8 + peer;
  unsigned long long v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(slot) : "memory");
  uint32_t s = (uint32_t)v;
  if ((uint32_t)(v >> 32) == a.seq && s != a.sig) {
    if (c.status->error == 0) { c.status->err_a = s; c.status->err_b = a.sig; }
    record_error(c.status, B200C_EMISMATCH, a.seq, peer, phase);
    c.status->abort_flag = 1;
  }
}

// Kernel prologue shared by every collective:
//  (1) block 0 publishes the op signature and arrive[rank] = seq to every peer;
//  (2) every block waits until every peer has arrived at op seq-1, i.e. has finished op seq-2 and
//      therefore no longer touches the staging half this op is about to overwrite.
// Returns block-uniform ok.
__device__ __forceinline__ bool coll_prologue(const CollArgs& a) {
  const DevComm& c = a.c;
  int t = threadIdx.x;
  if (blockIdx.x == 0 && t < c.world && t != c.rank) {
    announce_signature(a, t);
    st_release_sys(flag_at(c, t, kOffArrive, 0, c.rank), a.seq);
  }
  const uint32_t* arrive = flag_at(c, c.rank, kOffArrive, 0, 0);
  int ok = 1;
  if (t < c.world && t != c.rank) ok = wait_flag(arrive + t, a.seq - 1, c, t, kWaitArrive);
  return __syncthreads_and(ok) != 0;
}
// Block 0 compares each peer's announcement once that peer has arrived at this op.
__device__ __forceinline__ void check_signature(const CollArgs& a) {
  const DevComm& c = a.c;
  int t = threadIdx.x;
  if (blockIdx.x == 0 && t < c.world && t != c.rank) {
    if (wait_flag(flag_at(c, c.rank, kOffArrive, 0, t), a.seq, c, t, kWaitArrive)) compare_signature(a, t, kWaitArrive);
  }
}

// k-th rank after r in ring order (0 <= k < W): the order in which a rank visits its peers
__device__ __forceinline__ int peer_at(int r, int k, int W) {
  int j = r + k;
  if (j >= W) j -= W;
  return j;
}
// clip [lo, hi) against n, return count
__device__ __forceinline__ size_t clip_count(size_t lo, size_t hi, size_t n) {
  if (lo >= n) return 0;
  return (hi < n ? hi : n) - lo;
}
struct Span {
  size_t lo, cnt;
};
// granule [g0, g1) of rank chunk j: first element and element count inside the piece (0 past its end)
__device__ __forceinline__ Span chunk_span(const CollArgs& a, int j, size_t g0, size_t g1) {
  const size_t lo = (size_t)j * a.chunk + g0;
  return {lo, clip_count(lo, (size_t)j * a.chunk + g1, a.n)};
}
// The granules a block owns in the round-pipelined kernels: round q < count() is the granule [lo(q), hi(q))
// of every rank chunk, the same granules B200C_FOR_GRANULES walks.  An empty() block owns none.
struct BlockRounds {
  const CollArgs& a;
  size_t first, step;
  __device__ __forceinline__ explicit BlockRounds(const CollArgs& args)
      : a(args), first((size_t)blockIdx.x * args.tile), step((size_t)gridDim.x * args.tile) {}
  __device__ __forceinline__ bool empty() const { return first >= a.chunk; }
  __device__ __forceinline__ int count() const { return (int)((a.chunk - first + step - 1) / step); }
  __device__ __forceinline__ size_t lo(int q) const { return first + (size_t)q * step; }
  __device__ __forceinline__ size_t hi(int q) const { size_t h = first + (size_t)q * step + a.tile; return h < a.chunk ? h : a.chunk; }
};

// ---------------------------------------------------------------------------------------------
// dtype traits: R = storage type, A = accumulator type
// ---------------------------------------------------------------------------------------------
struct f16_t { uint16_t raw; };
struct bf16_t { uint16_t raw; };

template <typename T> struct Traits {
  using A = T;
  static __device__ __forceinline__ A to_acc(T v) { return v; }
  static __device__ __forceinline__ T from_acc(A v) { return v; }
};
template <> struct Traits<f16_t> {
  using A = float;
  static __device__ __forceinline__ float to_acc(f16_t v) { return __half2float(__ushort_as_half(v.raw)); }
  static __device__ __forceinline__ f16_t from_acc(float v) { f16_t r; r.raw = __half_as_ushort(__float2half_rn(v)); return r; }
};
template <> struct Traits<bf16_t> {
  using A = float;
  static __device__ __forceinline__ float to_acc(bf16_t v) { return __uint_as_float(((uint32_t)v.raw) << 16); }
  static __device__ __forceinline__ bf16_t from_acc(float v) { bf16_t r; r.raw = __bfloat16_as_ushort(__float2bfloat16_rn(v)); return r; }
};

template <int OP, typename A> struct Red;
template <typename A> struct Red<B200C_SUM, A> { static __device__ __forceinline__ A f(A a, A b) { return a + b; } };
template <typename A> struct Red<B200C_PROD, A> { static __device__ __forceinline__ A f(A a, A b) { return a * b; } };
template <typename A> struct Red<B200C_MAX, A> { static __device__ __forceinline__ A f(A a, A b) { return a > b ? a : b; } };
template <typename A> struct Red<B200C_MIN, A> { static __device__ __forceinline__ A f(A a, A b) { return a < b ? a : b; } };
// float min/max propagate like torch/gloo for finite inputs; NaN handling follows the comparison.
// signed-integer SUM/PROD wrap (two's complement), same as gloo's plain C arithmetic.
template <> struct Red<B200C_SUM, int8_t> { static __device__ __forceinline__ int8_t f(int8_t a, int8_t b) { return (int8_t)((uint8_t)a + (uint8_t)b); } };
template <> struct Red<B200C_PROD, int8_t> { static __device__ __forceinline__ int8_t f(int8_t a, int8_t b) { return (int8_t)((uint8_t)a * (uint8_t)b); } };
template <> struct Red<B200C_SUM, int32_t> { static __device__ __forceinline__ int32_t f(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); } };
template <> struct Red<B200C_PROD, int32_t> { static __device__ __forceinline__ int32_t f(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); } };
template <> struct Red<B200C_SUM, int64_t> { static __device__ __forceinline__ int64_t f(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); } };
template <> struct Red<B200C_PROD, int64_t> { static __device__ __forceinline__ int64_t f(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); } };

// post-scale in the accumulator domain (AVG, DDP mean)
template <typename A> __device__ __forceinline__ A apply_scale(A v, float s, int world) { return (A)(v / (A)world); }
template <> __device__ __forceinline__ float apply_scale<float>(float v, float s, int) { return v * s; }
template <> __device__ __forceinline__ double apply_scale<double>(double v, float s, int world) { return v / (double)world; }

template <typename T> union Pack16 {
  uint4 u;
  T e[16 / sizeof(T)];
  __device__ Pack16() {}
};

// a 16-byte vector of TW, multiplied element-wise by a.scale when the op has one (the NVLS kernels' AVG / mean)
template <typename TW>
__device__ __forceinline__ uint4 scale_vector(uint4 v, const CollArgs& a) {
  if (a.has_scale) {
    Pack16<TW> p; p.u = v;
#pragma unroll
    for (int e = 0; e < 16 / (int)sizeof(TW); e++) p.e[e] = Traits<TW>::from_acc(Traits<TW>::to_acc(p.e[e]) * a.scale);
    v = p.u;
  }
  return v;
}

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---------------------------------------------------------------------------------------------
// tile primitives: the whole block cooperates on `n` contiguous elements.
// ---------------------------------------------------------------------------------------------
constexpr int kUnroll = 4;

// Plain byte copy of n elements of T.  SRC_BYPASS: source is staging / peer memory.
template <typename T, bool SRC_BYPASS>
__device__ __forceinline__ void copy_tile(T* __restrict__ dst, const T* __restrict__ src, size_t n) {
  constexpr int V = 16 / sizeof(T);
  const int t = threadIdx.x;
  if (aligned16(dst) && aligned16(src)) {
    size_t nv = n / V;
    uint4* d = reinterpret_cast<uint4*>(dst);
    const uint4* s = reinterpret_cast<const uint4*>(src);
    size_t i = t;
    for (; i + (size_t)(kUnroll - 1) * kThreads < nv; i += (size_t)kUnroll * kThreads) {
      uint4 v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) v[u] = SRC_BYPASS ? ld_bypass16(s + i + (size_t)u * kThreads) : s[i + (size_t)u * kThreads];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) d[i + (size_t)u * kThreads] = v[u];
    }
    for (; i < nv; i += kThreads) d[i] = SRC_BYPASS ? ld_bypass16(s + i) : s[i];
    for (size_t k = nv * V + t; k < n; k += kThreads) dst[k] = SRC_BYPASS ? ld_bypass(src + k) : src[k];
  } else {
    for (size_t k = t; k < n; k += kThreads) dst[k] = SRC_BYPASS ? ld_bypass(src + k) : src[k];
  }
}

// Converting copy TS -> TD through the accumulator domain (fp32 for half types).
template <typename TS, typename TD, bool SRC_BYPASS>
__device__ __forceinline__ void convert_tile(TD* __restrict__ dst, const TS* __restrict__ src, size_t n) {
  // vector step = number of elements in 16 bytes of the narrower type
  constexpr int VS = 16 / sizeof(TS), VD = 16 / sizeof(TD);
  constexpr int V = VS > VD ? VS : VD;
  const int t = threadIdx.x;
  if (aligned16(dst) && aligned16(src)) {
    size_t nv = n / V;
    constexpr int NS = V / VS, ND = V / VD;   // 16-byte loads / stores per vector step
    for (size_t i = t; i < nv; i += kThreads) {
      uint4 raw[NS];
      const uint4* s = reinterpret_cast<const uint4*>(src + i * V);
#pragma unroll
      for (int q = 0; q < NS; q++) raw[q] = SRC_BYPASS ? ld_bypass16(s + q) : s[q];
      TD dv[V];
#pragma unroll
      for (int q = 0; q < NS; q++) {
        Pack16<TS> p;
        p.u = raw[q];
#pragma unroll
        for (int e = 0; e < VS; e++) dv[q * VS + e] = Traits<TD>::from_acc((typename Traits<TD>::A)Traits<TS>::to_acc(p.e[e]));
      }
      uint4* d = reinterpret_cast<uint4*>(dst + i * V);
#pragma unroll
      for (int q = 0; q < ND; q++) {
        Pack16<TD> p;
#pragma unroll
        for (int e = 0; e < VD; e++) p.e[e] = dv[q * VD + e];
        d[q] = p.u;
      }
    }
    for (size_t k = nv * V + t; k < n; k += kThreads)
      dst[k] = Traits<TD>::from_acc((typename Traits<TD>::A)Traits<TS>::to_acc(SRC_BYPASS ? ld_bypass(src + k) : src[k]));
  } else {
    for (size_t k = t; k < n; k += kThreads)
      dst[k] = Traits<TD>::from_acc((typename Traits<TD>::A)Traits<TS>::to_acc(SRC_BYPASS ? ld_bypass(src + k) : src[k]));
  }
}

template <typename TS, typename TD, bool SRC_BYPASS> struct Mover {
  static __device__ __forceinline__ void run(TD* dst, const TS* src, size_t n) { convert_tile<TS, TD, SRC_BYPASS>(dst, src, n); }
};
template <typename T, bool SRC_BYPASS> struct Mover<T, T, SRC_BYPASS> {
  static __device__ __forceinline__ void run(T* dst, const T* src, size_t n) { copy_tile<T, SRC_BYPASS>(dst, src, n); }
};
template <typename TS, typename TD, bool SRC_BYPASS>
__device__ __forceinline__ void move_tile(TD* dst, const TS* src, size_t n) {
  Mover<TS, TD, SRC_BYPASS>::run(dst, src, n);
}

// Zero-fills elements [end, end rounded up to the 16-byte vector) of dst when that stays below `limit`, so
// that the switch reduces defined values in the message's last vector.
template <typename TW>
__device__ __forceinline__ void zero_pad_vector(TW* dst, size_t lo, size_t cnt, size_t limit) {
  constexpr int V = 16 / sizeof(TW);
  size_t end = lo + cnt, padded = (end + V - 1) / V * V;
  if (cnt && padded > end && padded <= limit) {
    TW z = Traits<TW>::from_acc((typename Traits<TW>::A)0);
    for (size_t k = end + threadIdx.x; k < padded; k += kThreads) dst[k] = z;
  }
}

// ---------------------------------------------------------------------------------------------
// 1-byte element types.  The accumulator domain of int8 / uint8 is the 8-bit type itself (SUM and PROD wrap, like the
// C arithmetic of the reference's CPU path), so the 16 elements of a vector stay packed four to a register and are folded
// with per-byte SIMD arithmetic: same bits as 16 scalar accumulators, 4 registers instead of 16.
// ---------------------------------------------------------------------------------------------
template <int OP, bool SIGNED>
__device__ __forceinline__ uint32_t red_bytes4(uint32_t x, uint32_t y) {
  if (OP == B200C_SUM) return __vadd4(x, y);
  if (OP == B200C_MAX) return SIGNED ? __vmaxs4(x, y) : __vmaxu4(x, y);
  if (OP == B200C_MIN) return SIGNED ? __vmins4(x, y) : __vminu4(x, y);
  uint32_t r = 0;  // PROD: the low 8 bits of each product (identical for signed and unsigned operands)
#pragma unroll
  for (int q = 0; q < 4; q++) r |= ((((x >> (8 * q)) & 0xffu) * ((y >> (8 * q)) & 0xffu)) & 0xffu) << (8 * q);
  return r;
}
template <bool SIGNED>
__device__ __forceinline__ uint32_t div_bytes4(uint32_t v, int world) {
  uint32_t r = 0;  // integer AVG: truncating division of every element by the world size
#pragma unroll
  for (int q = 0; q < 4; q++) {
    int x = SIGNED ? (int)(int8_t)(v >> (8 * q)) : (int)((v >> (8 * q)) & 0xffu);
    r |= ((uint32_t)(x / world) & 0xffu) << (8 * q);
  }
  return r;
}
template <int OP, bool SIGNED>
__device__ __forceinline__ uint4 red_bytes16(uint4 x, uint4 y) {
  return make_uint4(red_bytes4<OP, SIGNED>(x.x, y.x), red_bytes4<OP, SIGNED>(x.y, y.y), red_bytes4<OP, SIGNED>(x.z, y.z),
                    red_bytes4<OP, SIGNED>(x.w, y.w));
}
template <typename T, int OP, int WT>
__device__ __forceinline__ void reduce_vectors_bytes(const CollArgs& a, const T* src0, size_t src_stride, int own_idx,
                                                     const T* own, T* dst_w, T* dst_i, size_t nv) {
  constexpr bool SG = (T)(-1) < (T)0;
  const int W = WT > 0 ? WT : a.c.world;
  for (size_t i = threadIdx.x; i < nv; i += kThreads) {
    const uint4 ownv = reinterpret_cast<const uint4*>(own)[i];
    uint4 acc = make_uint4(0, 0, 0, 0);
    if (WT > 0) {
      constexpr int B = WT < 4 ? (WT > 0 ? WT : 1) : 4;
#pragma unroll
      for (int s0 = 0; s0 < WT; s0 += B) {
        uint4 raw[B];
#pragma unroll
        for (int k = 0; k < B; k++)
          raw[k] = ld_bypass16_if(reinterpret_cast<const uint4*>(src0 + (size_t)(s0 + k) * src_stride + i * 16), s0 + k != own_idx);
#pragma unroll
        for (int k = 0; k < B; k++) {
          const uint4 x = (s0 + k == own_idx) ? ownv : raw[k];
          acc = (s0 + k == 0) ? x : red_bytes16<OP, SG>(acc, x);
        }
      }
    } else {
#pragma unroll 1
      for (int s = 0; s < W; s++) {
        const uint4 ld = ld_bypass16_if(reinterpret_cast<const uint4*>(src0 + (size_t)s * src_stride + i * 16), s != own_idx);
        const uint4 x = (s == own_idx) ? ownv : ld;
        acc = (s == 0) ? x : red_bytes16<OP, SG>(acc, x);
      }
    }
    if (a.has_scale) acc = make_uint4(div_bytes4<SG>(acc.x, W), div_bytes4<SG>(acc.y, W), div_bytes4<SG>(acc.z, W), div_bytes4<SG>(acc.w, W));
    if (dst_w) reinterpret_cast<uint4*>(dst_w)[i] = acc;
    if (dst_i) reinterpret_cast<uint4*>(dst_i)[i] = acc;
  }
}

// Reduce `world` sources in rank order into up to two destinations.
//   src0 + s * src_stride points at rank s's contribution (TW, staging -> bypass loads) except
//   s == own_idx which is `own` (TI, user memory, rounded through TW so every rank's contribution is
//   treated alike).
//   dst_w (TW, may be nullptr): result for peers to pull.  dst_i (TI, may be nullptr): user output.
// WT > 0: the world size is a compile-time constant, so the W in-flight vectors live in registers
// (a runtime-indexed array would be demoted to local memory); WT == 0 handles the odd world sizes
// (3, 5, 6, 7) by folding each contribution as it is loaded.
template <typename TI, typename TW, int OP, int WT>
__device__ __forceinline__ void reduce_vectors(const CollArgs& a, const TW* src0, size_t src_stride, int own_idx,
                                               const TI* own, TW* dst_w, TI* dst_i, size_t nv) {
  using A = typename Traits<TW>::A;
  constexpr int V = 16 / sizeof(TW);
  constexpr int VI = 16 / sizeof(TI);
  const int W = WT > 0 ? WT : a.c.world;
  if constexpr (sizeof(TW) == 1) {
    reduce_vectors_bytes<TW, OP, WT>(a, src0, src_stride, own_idx, own, dst_w, dst_i, nv);
  } else
  for (size_t i = threadIdx.x; i < nv; i += kThreads) {
    // 8-byte elements: an opaque per-iteration copy of the slot stride keeps the compiler from hoisting all W slot
    // addresses (two registers each) out of the loop, which cost the W = 8 kernels a spill
    size_t stride_i = src_stride;
    if (sizeof(TW) == 8) asm volatile("" : "+l"(stride_i));
    A acc[V];
    TI ownv[V];
    if (!(WT > 0 && sizeof(TI) > sizeof(TW))) {
      const uint4* o = reinterpret_cast<const uint4*>(own + i * V);
#pragma unroll
      for (int q = 0; q < V / VI; q++) {
        Pack16<TI> po;
        po.u = o[q];
#pragma unroll
        for (int e = 0; e < VI; e++) ownv[q * VI + e] = po.e[e];
      }
    }
    if (WT > 0) {
      // loads are issued in batches of up to four sources (memory-level parallelism without exceeding
      // the 64-register budget of two 512-thread CTAs per SM), then folded in rank order
      constexpr int B = WT < 4 ? (WT > 0 ? WT : 1) : 4;
#pragma unroll
      for (int s0 = 0; s0 < WT; s0 += B) {
        uint4 raw[B];
#pragma unroll
        for (int k = 0; k < B; k++)
          raw[k] = ld_bypass16_if(reinterpret_cast<const uint4*>(src0 + (size_t)(s0 + k) * stride_i + i * V), s0 + k != own_idx);
#pragma unroll
        for (int k = 0; k < B; k++) {
          const int s = s0 + k;
          Pack16<TW> p;
          p.u = raw[k];
          if constexpr (sizeof(TI) > sizeof(TW)) {
            // a wire narrower than the buffer: the own contribution (V elements of TI) is loaded where it is
            // folded instead of being held across the batches, which keeps sm_90a's allocation out of local memory
            if (s == own_idx) {
              const uint4* o = reinterpret_cast<const uint4*>(own + i * V);
#pragma unroll
              for (int q = 0; q < V / VI; q++) {
                Pack16<TI> po;
                po.u = o[q];
#pragma unroll
                for (int e = 0; e < VI; e++) {
                  const A x = Traits<TW>::to_acc(Traits<TW>::from_acc((A)Traits<TI>::to_acc(po.e[e])));
                  acc[q * VI + e] = (s == 0) ? x : Red<OP, A>::f(acc[q * VI + e], x);
                }
              }
              continue;
            }
          }
#pragma unroll
          for (int e = 0; e < V; e++) {
            A x;
            if (s == own_idx) x = Traits<TW>::to_acc(Traits<TW>::from_acc((A)Traits<TI>::to_acc(ownv[e])));
            else x = Traits<TW>::to_acc(p.e[e]);
            acc[e] = (s == 0) ? x : Red<OP, A>::f(acc[e], x);
          }
        }
      }
    } else {
#pragma unroll 1
      for (int s = 0; s < W; s++) {
        Pack16<TW> p;
        p.u = ld_bypass16_if(reinterpret_cast<const uint4*>(src0 + (size_t)s * stride_i + i * V), s != own_idx);
#pragma unroll
        for (int e = 0; e < V; e++) {
          A x;
          if (s == own_idx) x = Traits<TW>::to_acc(Traits<TW>::from_acc((A)Traits<TI>::to_acc(ownv[e])));
          else x = Traits<TW>::to_acc(p.e[e]);
          acc[e] = (s == 0) ? x : Red<OP, A>::f(acc[e], x);
        }
      }
    }
    Pack16<TW> r;
#pragma unroll
    for (int e = 0; e < V; e++) {
      A v = acc[e];
      if (a.has_scale) v = apply_scale<A>(v, a.scale, W);
      r.e[e] = Traits<TW>::from_acc(v);
    }
    if (dst_w) *reinterpret_cast<uint4*>(dst_w + i * V) = r.u;
    if (dst_i) {
      uint4* d = reinterpret_cast<uint4*>(dst_i + i * V);
#pragma unroll
      for (int q = 0; q < V / VI; q++) {
        Pack16<TI> po;
#pragma unroll
        for (int e = 0; e < VI; e++) po.e[e] = Traits<TI>::from_acc((typename Traits<TI>::A)Traits<TW>::to_acc(r.e[q * VI + e]));
        d[q] = po.u;
      }
    }
  }
}

template <typename TI, typename TW, int OP, int WT>
__device__ __forceinline__ void reduce_tile(const CollArgs& a, const TW* src0, size_t src_stride, int own_idx,
                                            const TI* own, TW* dst_w, TI* dst_i, size_t n) {
  using A = typename Traits<TW>::A;
  constexpr int V = 16 / sizeof(TW);
  const int W = WT > 0 ? WT : a.c.world;
  const int t = threadIdx.x;
  static_assert(sizeof(TI) >= sizeof(TW), "wire type must not be wider than the buffer type");
  bool vec = aligned16(own) && (dst_i == nullptr || aligned16(dst_i));
  size_t nv = vec ? n / V : 0;
  reduce_vectors<TI, TW, OP, WT>(a, src0, src_stride, own_idx, own, dst_w, dst_i, nv);
  for (size_t k = nv * V + t; k < n; k += kThreads) {
    A acc = A();
#pragma unroll 1
    for (int s = 0; s < W; s++) {
      A x;
      if (s == own_idx) x = Traits<TW>::to_acc(Traits<TW>::from_acc((A)Traits<TI>::to_acc(own[k])));
      else x = Traits<TW>::to_acc(ld_bypass(src0 + (size_t)s * src_stride + k));
      acc = (s == 0) ? x : Red<OP, A>::f(acc, x);
    }
    if (a.has_scale) acc = apply_scale<A>(acc, a.scale, W);
    TW r = Traits<TW>::from_acc(acc);
    if (dst_w) dst_w[k] = r;
    if (dst_i) dst_i[k] = Traits<TI>::from_acc((typename Traits<TI>::A)Traits<TW>::to_acc(r));
  }
}

}  // namespace b200c
