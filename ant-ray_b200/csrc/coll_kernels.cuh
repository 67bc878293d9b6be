// Collective kernels over peer-mapped arenas (hand-written for sm_90a; no NCCL on this path).
//
// Partitioning (SURVEY.md §8e): a piece of n elements is cut into `world` rank chunks of
// `chunk` elements; each chunk is cut into granules of `tile` elements.  Block b of every rank
// works on granules b, b + grid, b + 2*grid, ... of every chunk (block-cyclic), so
//   * cross-rank dependencies exist only between blocks with the same index and are carried by
//     the flag pair [block][src] in the signal pad — no intra-grid synchronisation, blocks need
//     not be co-resident;
//   * at any time the whole grid touches one contiguous window of each chunk (grid * tile
//     elements), which keeps DRAM pages and TLB entries hot on the side that serves peer /
//     multimem reads, instead of `grid` streams spread over the whole message.
//
// Staging is double-buffered by sequence parity (a.seq & 1); coll_prologue() makes the reuse
// safe for asymmetric ops as well.
#pragma once
#include "dev_common.cuh"

namespace b200c {

template <typename T>
__device__ __forceinline__ T* staging_ptr(const DevComm& c, int rank, uint32_t seq, size_t byte_off) {
  return reinterpret_cast<T*>(c.arena[rank] + c.off_staging + (size_t)(seq & 1) * c.staging_bytes + byte_off);
}
// granules of a chunk of `extent` elements owned by this block: [g0, g1) for g0 = first, first + step, ...
#define B200C_FOR_GRANULES(g0, g1, a, extent)                                                                 \
  for (size_t g0 = (size_t)blockIdx.x * (a).tile, g1 = g0 + (a).tile < (extent) ? g0 + (a).tile : (extent); \
       g0 < (extent);                                                                                          \
       g0 += (size_t)gridDim.x * (a).tile, g1 = g0 + (a).tile < (extent) ? g0 + (a).tile : (extent))

// The reducing kernels are compiled once per world size (WT = 2, 4, 8; WT = 0 takes the world size at run time for
// 3, 5, 6, 7): with the four reduce loops in one kernel the register allocator spilled loop invariants into local
// memory under the 64-register budget; one loop per kernel keeps most of them free of a stack (tests/test_sass_hygiene.py).
// ---------------------------------------------------------------------------------------------
// one-shot allreduce: push the whole buffer to every peer, reduce locally.  One flag round.
// staging slot s (n_pad elements of TW) on rank j holds rank s's data.
// ---------------------------------------------------------------------------------------------
template <typename TI, typename TW, int OP, int WT>
__global__ void __launch_bounds__(kThreads, 2) k_allreduce_oneshot(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world;
  if (!coll_prologue(a)) return;
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  const size_t slot_bytes = a.chunk * sizeof(TW);  // chunk == padded n for one-shot
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    for (int k = 1; k < W; k++)
      move_tile<TI, TW, false>(staging_ptr<TW>(c, peer_at(r, k, W), a.seq, (size_t)r * slot_bytes) + t0, in + t0, t1 - t0);
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    reduce_tile<TI, TW, OP, WT>(a, staging_ptr<TW>(c, r, a.seq, 0) + t0, a.chunk, r, in + t0, nullptr, out + t0, t1 - t0);
  }
}

// ---------------------------------------------------------------------------------------------
// LL one-shot allreduce for small messages (latency-bound): every 32-bit payload word travels in
// one naturally aligned 8-byte store {data, flag} (single-copy atomic), so there is no separate
// flag round and no release fence between data and flag — the receiver polls the slot itself.
// flag = a.ll_seq (per-communicator LL op counter, never 0); the region is double-buffered by
// ll_seq & 1.  Reuse is safe without the arrive rule: a peer can only write LL op k+2 after it
// finished op k+1, which needed this rank's op k+1 data, which this rank sends after its op k
// kernel (which read every slot) has completed.
// Layout on rank j: half h, source s, vector i  ->  4 consecutive u64 {word, flag}.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void st_ll2(void* p, uint32_t d0, uint32_t d1, uint32_t flag) {
  asm volatile("st.relaxed.sys.global.v2.b64 [%0], {%1, %2};" ::"l"(p), "l"((unsigned long long)d0 | ((unsigned long long)flag << 32)),
               "l"((unsigned long long)d1 | ((unsigned long long)flag << 32))
               : "memory");
}
__device__ __forceinline__ void ld_ll2(const void* p, unsigned long long& a0, unsigned long long& a1) {
  asm volatile("ld.relaxed.sys.global.v2.b64 {%0, %1}, [%2];" : "=l"(a0), "=l"(a1) : "l"(p) : "memory");
}
__device__ __forceinline__ char* ll_slot(const DevComm& c, int on_rank, uint32_t ll_seq, int src) {
  return c.arena[on_rank] + c.off_ll + ((size_t)(ll_seq & 1) * kMaxRanks + src) * c.ll_words * 8;
}

template <typename T, int OP, int WT>
__device__ __forceinline__ void ll_allreduce_body(const CollArgs& a) {
  using A = typename Traits<T>::A;
  constexpr int V = 16 / sizeof(T);
  const DevComm& c = a.c;
  const int r = c.rank;
  const int W = WT > 0 ? WT : c.world;
  const T* in = static_cast<const T*>(a.in);
  T* out = static_cast<T*>(a.out);
  const size_t nv = (a.n + V - 1) / V;  // 16-byte vectors, the last one possibly partial
  const bool vec_ok = aligned16(in) && aligned16(out);
  const uint32_t flag = a.ll_seq;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nv; i += (size_t)gridDim.x * blockDim.x) {
    const size_t e0 = i * V;
    const bool full = vec_ok && e0 + V <= a.n;
    Pack16<T> mine;
    if (full) {
      mine.u = *reinterpret_cast<const uint4*>(in + e0);
    } else {
      mine.u = make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int e = 0; e < V; e++)
        if (e0 + e < a.n) mine.e[e] = in[e0 + e];
    }
    // the peer order and the signature compare below are spelled out here rather than through peer_at() /
    // compare_signature(): through the helpers sm_90a allocates the LL bodies differently (local memory at W = 4)
    for (int k = 1; k < W; k++) {
      int j = r + k; if (j >= W) j -= W;
      char* dst = ll_slot(c, j, flag, r) + i * 32;
      st_ll2(dst, mine.u.x, mine.u.y, flag);
      st_ll2(dst + 16, mine.u.z, mine.u.w, flag);
    }
    uint4 raw[WT > 0 ? WT : kMaxRanks];
    bool ok = true;
#pragma unroll
    for (int s = 0; s < (WT > 0 ? WT : kMaxRanks); s++) {
      if (s >= W || s == r) continue;
      const char* src = ll_slot(c, r, flag, s) + i * 32;
      unsigned long long q0, q1, q2, q3;
      unsigned spins = 0;
      unsigned long long t_start = 0;
      for (;;) {
        ld_ll2(src, q0, q1);
        ld_ll2(src + 16, q2, q3);
        if ((uint32_t)(q0 >> 32) == flag && (uint32_t)(q1 >> 32) == flag && (uint32_t)(q2 >> 32) == flag && (uint32_t)(q3 >> 32) == flag) break;
        if ((++spins & 0x3ff) == 0) {
          if (t_start == 0) t_start = globaltimer_ns();
          // a peer that entered the same op with different arguments will never fill this slot: compare signatures
          const unsigned long long* sl = reinterpret_cast<const unsigned long long*>(c.arena[r] + kOffOpSig) + (a.seq & 1) * 8 + s;
          unsigned long long sv;
          asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(sv) : "l"(sl) : "memory");
          if ((uint32_t)(sv >> 32) == a.seq && (uint32_t)sv != a.sig) {
            if (c.status->error == 0) { c.status->err_a = (uint32_t)sv; c.status->err_b = a.sig; }
            record_error(c.status, B200C_EMISMATCH, a.seq, s, kWaitLL);
            c.status->abort_flag = 1;
            ok = false; break;
          }
          if (c.status->abort_flag) { record_error(c.status, B200C_EABORTED, a.seq, s, kWaitLL); ok = false; break; }
          if (globaltimer_ns() - t_start > c.timeout_ns) { record_error(c.status, B200C_ETIMEOUT, a.seq, s, kWaitLL); ok = false; break; }
        }
      }
      raw[s] = make_uint4((uint32_t)q0, (uint32_t)q1, (uint32_t)q2, (uint32_t)q3);
    }
    if (!ok) return;
    A acc[V];
#pragma unroll
    for (int s = 0; s < (WT > 0 ? WT : kMaxRanks); s++) {
      if (s >= W) continue;
      Pack16<T> p;
      p.u = (s == r) ? mine.u : raw[s];
#pragma unroll
      for (int e = 0; e < V; e++) {
        A x = Traits<T>::to_acc(p.e[e]);
        acc[e] = (s == 0) ? x : Red<OP, A>::f(acc[e], x);
      }
    }
    Pack16<T> res;
#pragma unroll
    for (int e = 0; e < V; e++) {
      A v = acc[e];
      if (a.has_scale) v = apply_scale<A>(v, a.scale, W);
      res.e[e] = Traits<T>::from_acc(v);
    }
    if (full) {
      *reinterpret_cast<uint4*>(out + e0) = res.u;
    } else {
#pragma unroll
      for (int e = 0; e < V; e++)
        if (e0 + e < a.n) out[e0 + e] = res.e[e];
    }
  }
}

constexpr int kLLThreads = 256;
// one kernel per world size (WT = 2, 4, 8; 0 = the others), like the other reducers: with the four bodies in one
// kernel the register allocator kept the in-flight vectors of the wider bodies in local memory
template <typename T, int OP, int WT>
__global__ void __launch_bounds__(kLLThreads) k_allreduce_ll(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int t = threadIdx.x;
  // announce (seq, signature) first — a plain store, no fence — so a peer that entered this op with
  // different arguments is diagnosed instead of both sides timing out
  if (blockIdx.x == 0 && t < c.world && t != c.rank) announce_signature(a, t);
  ll_allreduce_body<T, OP, WT>(a);
  // arrival (the op after this one may start: arrive rule) goes last so that the fence of the release
  // does not sit in front of the data stores
  if (blockIdx.x == 0 && t < c.world && t != c.rank) {
    st_release_sys(flag_at(c, t, kOffArrive, 0, c.rank), a.seq);
    // a rank whose message is the SHORTER one receives everything it waits for and would not notice a
    // peer that passed other arguments: compare the announcement that peer made at the start of its kernel
    // (no waiting: if it has not landed yet the check is skipped, the longer side reports the mismatch)
    compare_signature(a, t, kWaitLL);
  }
}

// ---------------------------------------------------------------------------------------------
// two-shot allreduce.
//   A: push granule of chunk j to rank j's staging slot [r]          (NVLink egress, stores)
//   B: reduce the W contributions of the own chunk in rank order; result -> own slot [r] + out
//   C: pull every other rank's reduced granule                       (NVLink ingress, loads)
// ---------------------------------------------------------------------------------------------
template <typename TI, typename TW, int OP, int WT>
__global__ void __launch_bounds__(kThreads, 2) k_allreduce_twoshot(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world;
  if (!coll_prologue(a)) return;
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  const size_t slot_bytes = a.chunk * sizeof(TW);
  // ---- A
  B200C_FOR_GRANULES(t0, t1, a, a.chunk) {
    for (int k = 1; k < W; k++) {
      const int j = peer_at(r, k, W);
      const auto [lo, cnt] = chunk_span(a, j, t0, t1);
      if (cnt) move_tile<TI, TW, false>(staging_ptr<TW>(c, j, a.seq, (size_t)r * slot_bytes) + t0, in + lo, cnt);
    }
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  // ---- B
  B200C_FOR_GRANULES(t0, t1, a, a.chunk) {
    const auto [lo, cnt] = chunk_span(a, r, t0, t1);
    if (cnt)
      reduce_tile<TI, TW, OP, WT>(a, staging_ptr<TW>(c, r, a.seq, 0) + t0, a.chunk, r, in + lo, staging_ptr<TW>(c, r, a.seq, (size_t)r * slot_bytes) + t0, out + lo, cnt);
  }
  block_signal_all(kOffFlagB, a.seq, c);
  if (!block_wait_all(kOffFlagB, a.seq, c, kWaitFlagB)) return;
  // ---- C
  B200C_FOR_GRANULES(t0, t1, a, a.chunk) {
    for (int k = 1; k < W; k++) {
      const int j = peer_at(r, k, W);
      const auto [lo, cnt] = chunk_span(a, j, t0, t1);
      if (cnt) move_tile<TW, TI, true>(out + lo, staging_ptr<TW>(c, j, a.seq, (size_t)j * slot_bytes) + t0, cnt);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// reducescatter: in_ptrs[j] (n elements) is this rank's contribution to rank j.
// reduce (root): every non-root pushes to root; root folds; root then releases the others.
// Both are phases A+B of two-shot with full-size chunks.
// ---------------------------------------------------------------------------------------------
template <typename T, int OP, int WT>
__global__ void __launch_bounds__(kThreads, 2) k_reducescatter(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world;
  if (!coll_prologue(a)) return;
  const size_t slot_bytes = a.chunk * sizeof(T);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    for (int k = 1; k < W; k++) {
      const int j = peer_at(r, k, W);
      copy_tile<T, false>(staging_ptr<T>(c, j, a.seq, (size_t)r * slot_bytes) + t0, static_cast<const T*>(a.in_ptrs[j]) + t0, t1 - t0);
    }
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    reduce_tile<T, T, OP, WT>(a, staging_ptr<T>(c, r, a.seq, 0) + t0, a.chunk, r, static_cast<const T*>(a.in_ptrs[r]) + t0, nullptr, static_cast<T*>(a.out) + t0, t1 - t0);
  }
}

// Fused gradient mean as a reducescatter (FSDP): phases A+B of two-shot reading in_ptrs[j].  Each contribution
// travels as TW, the fold accumulates in fp32 in rank order and scales once, the result is stored as TI.
// At W = 8 with a wire narrower than the buffer the fold also writes the TW result into the rank's own staging
// slot, which no peer writes in a reducescatter.  That store is not needed for the result; it is the form of the
// W = 8 fold that sm_90a allocates without a stack under the 64-register budget (tests/test_sass_hygiene.py), like
// the phase B of two-shot, and costs 2 bytes of local HBM writes per element.  The other world sizes fit without it.
template <typename TI, typename TW, int WT>
__global__ void __launch_bounds__(kThreads, 2) k_reducescatter_scaled(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world;
  if (!coll_prologue(a)) return;
  const size_t slot_bytes = a.chunk * sizeof(TW);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    for (int k = 1; k < W; k++) {
      const int j = peer_at(r, k, W);
      move_tile<TI, TW, false>(staging_ptr<TW>(c, j, a.seq, (size_t)r * slot_bytes) + t0, static_cast<const TI*>(a.in_ptrs[j]) + t0, t1 - t0);
    }
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    TW* own_slot = WT == 8 && sizeof(TI) > sizeof(TW) ? staging_ptr<TW>(c, r, a.seq, (size_t)r * slot_bytes) + t0 : nullptr;
    reduce_tile<TI, TW, B200C_SUM, WT>(a, staging_ptr<TW>(c, r, a.seq, 0) + t0, a.chunk, r, static_cast<const TI*>(a.in_ptrs[r]) + t0, own_slot,
                                       static_cast<TI*>(a.out) + t0, t1 - t0);
  }
}

template <typename T, int OP, int WT>
__global__ void __launch_bounds__(kThreads, 2) k_reduce(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, root = a.root;
  if (!coll_prologue(a)) return;
  const size_t slot_bytes = a.chunk * sizeof(T);
  if (r != root) {
    B200C_FOR_GRANULES(t0, t1, a, a.n) {
      copy_tile<T, false>(staging_ptr<T>(c, root, a.seq, (size_t)r * slot_bytes) + t0, static_cast<const T*>(a.in) + t0, t1 - t0);
    }
    block_signal_one(kOffFlagA, a.seq, c, root);
    // wait for root's release: completion of any rank then implies every rank has arrived
    block_wait_one(flag_at(c, r, kOffFlagB, blockIdx.x, root), a.seq, c, root, kWaitFlagB);
  } else {
    if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
    check_signature(a);
    B200C_FOR_GRANULES(t0, t1, a, a.n) {
      reduce_tile<T, T, OP, WT>(a, staging_ptr<T>(c, r, a.seq, 0) + t0, a.chunk, r, static_cast<const T*>(a.in) + t0, nullptr, static_cast<T*>(a.out) + t0, t1 - t0);
    }
    block_signal_all(kOffFlagB, a.seq, c);
  }
}

// ---------------------------------------------------------------------------------------------
// NVLS allreduce (SUM; f32 / bf16 / f16): the NVSwitch reduces (multimem.ld_reduce) and
// broadcasts (multimem.st).  Data must sit at the same arena offset on every rank:
//   staged   : A copies the user tensor into staging, C copies the result back;
//   symmetric: the tensor already lives in the symmetric region, A and C are flag-only.
// ---------------------------------------------------------------------------------------------
template <typename T> struct Multimem;
template <> struct Multimem<float> {
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
template <> struct Multimem<bf16_t> {
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
template <> struct Multimem<f16_t> {
  static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
  }
};
__device__ __forceinline__ void multimem_st16(void* p, uint4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// in-switch reduce of nv 16-byte vectors at multicast address `mc`, broadcast back in place.
// U = 4 vectors are in flight per thread.
template <typename TW, int U>
__device__ __forceinline__ void nvls_reduce_bcast_u(char* mc, size_t nv, const CollArgs& a, size_t i) {
  for (; i + (U - 1) * kThreads < nv; i += U * kThreads) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) v[u] = Multimem<TW>::ld_reduce(mc + (i + u * kThreads) * 16);
#pragma unroll
    for (int u = 0; u < U; u++) multimem_st16(mc + (i + u * kThreads) * 16, scale_vector<TW>(v[u], a));
  }
  for (; i < nv; i += kThreads) multimem_st16(mc + i * 16, scale_vector<TW>(Multimem<TW>::ld_reduce(mc + i * 16), a));
}
template <typename TW>
__device__ __forceinline__ void nvls_reduce_bcast(char* mc, size_t nv, const CollArgs& a) {
  nvls_reduce_bcast_u<TW, kUnroll>(mc, nv, a, threadIdx.x);
}
// user tensor -> staging for the granule [g0, g1) of every rank chunk (zero-pad the last vector so the
// switch reduces defined values)
template <typename TI, typename TW>
__device__ __forceinline__ void nvls_stage_in(const CollArgs& a, TW* mine, const TI* in, size_t g0, size_t g1) {
  const int W = a.c.world;
  for (int j = 0; j < W; j++) {
    const auto [lo, cnt] = chunk_span(a, j, g0, g1);
    if (cnt) move_tile<TI, TW, false>(mine + lo, in + lo, cnt);
    zero_pad_vector(mine, lo, cnt, lo + (g1 - g0));
  }
}
template <typename TI, typename TW>
__device__ __forceinline__ void nvls_stage_out(const CollArgs& a, const TW* mine, TI* out, size_t g0, size_t g1) {
  const int W = a.c.world;
  for (int j = 0; j < W; j++) {
    const auto [lo, cnt] = chunk_span(a, j, g0, g1);
    if (cnt) move_tile<TW, TI, true>(out + lo, mine + lo, cnt);
  }
}

template <typename TI, typename TW>
__global__ void __launch_bounds__(kThreads, 2) k_allreduce_nvls(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank;
  if (!coll_prologue(a)) return;
  constexpr int V = 16 / sizeof(TW);
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  // byte offset (inside the arena) of element 0 of the buffer the switch works on
  const size_t base_off = a.symmetric ? a.sym_off : c.off_staging + (size_t)(a.seq & 1) * c.staging_bytes;
  TW* mine = reinterpret_cast<TW*>(c.arena[r] + base_off);
  // ---- A: stage in
  if (!a.symmetric) {
    B200C_FOR_GRANULES(g0, g1, a, a.chunk) nvls_stage_in<TI, TW>(a, mine, in, g0, g1);
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  // ---- B: in-switch reduce of the own chunk's granules, broadcast back in place
  B200C_FOR_GRANULES(g0, g1, a, a.chunk) {
    const auto [lo, cnt] = chunk_span(a, r, g0, g1);
    if (cnt) nvls_reduce_bcast<TW>(c.mc_arena + base_off + lo * sizeof(TW), (cnt + V - 1) / V, a);
  }
  block_signal_all(kOffFlagB, a.seq, c);
  if (!block_wait_all(kOffFlagB, a.seq, c, kWaitFlagB)) return;
  // ---- C: stage out
  if (!a.symmetric) {
    B200C_FOR_GRANULES(g0, g1, a, a.chunk) nvls_stage_out<TI, TW>(a, mine, out, g0, g1);
  }
}

// ---------------------------------------------------------------------------------------------
// Round-pipelined staged NVLS allreduce (large plain tensors).  Same data flow as k_allreduce_nvls,
// but the three stages are synchronised per ROUND (one granule of every chunk per block) instead of
// per phase, and software-pipelined inside each block:
//
//     in(q+1) -> signalA(q+1) -> waitA(q) -> switch(q) -> signalB(q) -> waitB(q-1) -> out(q-1)
//
// so every wait has a full stage of local work in front of it, and — because a block only ever
// depends on the same-index block of its peers, never on the rest of its own grid — blocks drift out
// of phase as soon as the switch becomes the bottleneck: while some blocks queue on the switch the
// others run their local HBM copies.  (The plain kernel keeps the whole grid in lock step: all copy
// in, then all reduce, then all copy out — the link idles during both copies.)
// Round flags live in pipeA / pipeB [block][src]; the value of round q is pipe_base + q + 1, and the
// host advances pipe_base by the number of rounds of every such op.
// ---------------------------------------------------------------------------------------------
template <typename TI, typename TW>
__global__ void __launch_bounds__(kThreads, 2) k_allreduce_nvls_rounds(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank;
  if (!coll_prologue(a)) return;
  check_signature(a);
  constexpr int V = 16 / sizeof(TW);
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  const size_t base_off = c.off_staging + (size_t)(a.seq & 1) * c.staging_bytes;
  TW* mine = reinterpret_cast<TW*>(c.arena[r] + base_off);
  const BlockRounds rd(a);
  if (rd.empty()) return;
  const int R = rd.count();
  nvls_stage_in<TI, TW>(a, mine, in, rd.lo(0), rd.hi(0));
  block_signal_all(kOffPipeA, a.pipe_base + 1, c);
  for (int q = 0; q < R; q++) {
    if (q + 1 < R) {
      nvls_stage_in<TI, TW>(a, mine, in, rd.lo(q + 1), rd.hi(q + 1));
      block_signal_all(kOffPipeA, a.pipe_base + q + 2, c);
    }
    if (!block_wait_all(kOffPipeA, a.pipe_base + q + 1, c, kWaitFlagA)) return;
    {  // clipped by hand: chunk_span() here changes this kernel's register allocation
      size_t lo = (size_t)r * a.chunk + rd.lo(q);
      size_t cnt = clip_count(lo, (size_t)r * a.chunk + rd.hi(q), a.n);
      if (cnt) nvls_reduce_bcast<TW>(c.mc_arena + base_off + lo * sizeof(TW), (cnt + V - 1) / V, a);
    }
    block_signal_all(kOffPipeB, a.pipe_base + q + 1, c);
    if (q >= 1) {
      if (!block_wait_all(kOffPipeB, a.pipe_base + q, c, kWaitFlagB)) return;
      nvls_stage_out<TI, TW>(a, mine, out, rd.lo(q - 1), rd.hi(q - 1));
    }
  }
  if (!block_wait_all(kOffPipeB, a.pipe_base + R, c, kWaitFlagB)) return;
  nvls_stage_out<TI, TW>(a, mine, out, rd.lo(R - 1), rd.hi(R - 1));
}

// ---------------------------------------------------------------------------------------------
// Lane-structured staged NVLS allreduce (the largest plain tensors).  The grid is cut into L lanes of
// 1 + Kc CTAs.  CTA 0 of a lane only talks to the switch (multimem.ld_reduce / multimem.st and the two
// cross-GPU flags of its lane); the other Kc CTAs only move data locally (user tensor -> ring, ring ->
// user tensor).  Roles meet through flags in LOCAL memory, so
//   * the system-scope release fences (expensive on an SM that streams stores) sit in the switch CTAs,
//     where nothing else streams, and never stall
//     a copy;
//   * few CTAs issue multimem traffic (the switch saturates with ~32 CTAs; more only scatter the access
//     pattern) while many CTAs drive the local HBM copies;
//   * staging is a small ring — lane l, slot q % 3, chunk j, T elements — that is rewritten every three
//     rounds and therefore stays in L2: the switch reads it from L2, the results land in L2, the copy-out
//     reads L2; HBM only sees the user tensor once in and once out.  (It also removes the staging-capacity
//     limit: one launch handles a message of any size.)
// Lane l owns granules l, l + L, l + 2L, ... (T elements) of every rank chunk; round q of lane l is granule
// q*L + l.  Order inside a copy CTA: in(q), out(q-2) — three ring slots make in(q) safe: slot q%3 was read out
// in out(q-3), one iteration earlier, and every peer finished reducing it before that (flagB).
// Flags: laneIn[lane][k] (local, copy CTA k -> switch CTA), pipeA[lane][src] ("src staged round q"),
// pipeB[lane][src] ("src reduced + broadcast its chunk of round q", also raised on the own arena).
// ---------------------------------------------------------------------------------------------
constexpr int kLaneSlots = 3;

template <typename TI, typename TW>
__global__ void __launch_bounds__(kThreads, 2) k_allreduce_nvls_lanes(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world, t = threadIdx.x;
  if (!coll_prologue(a)) return;
  check_signature(a);
  constexpr int V = 16 / sizeof(TW);
  const int per = 1 + a.lane_copy, Kc = a.lane_copy;
  const int lane = blockIdx.x / per, role = blockIdx.x % per, L = gridDim.x / per;
  const size_t T = a.tile;
  const size_t ngran = (a.chunk + T - 1) / T;
  const int R = (size_t)lane < ngran ? (int)((ngran - lane + L - 1) / L) : 0;
  const size_t half_off = c.off_staging + (size_t)(a.seq & 1) * c.staging_bytes;
  auto ring_elem = [&](int slot, int j) { return (((size_t)lane * kLaneSlots + slot) * W + j) * T; };
  uint32_t* laneIn = flag_at(c, r, kOffLaneIn, lane, 0);
  if (role == 0) {
    // ------------------------------------------------------------------ switch CTA
    const uint32_t* fA = flag_at(c, r, kOffPipeA, lane, 0);
    for (int q = 0; q < R; q++) {
      const uint32_t v = a.pipe_base + q + 1;
      int ok = 1;
      if (t < Kc) ok = wait_flag(laneIn + t, v, c, r, kWaitFlagA);
      if (!__syncthreads_and(ok)) return;
      if (t < W && t != r) st_release_sys(flag_at(c, t, kOffPipeA, lane, r), v);
      ok = 1;
      if (t < W && t != r) ok = wait_flag(fA + t, v, c, t, kWaitFlagA);
      if (!__syncthreads_and(ok)) return;
      const size_t g0 = ((size_t)q * L + lane) * T;   // clipped by hand, as in k_allreduce_nvls_rounds
      const size_t lo = (size_t)r * a.chunk + g0;
      const size_t hi = (size_t)r * a.chunk + (g0 + T < a.chunk ? g0 + T : a.chunk);
      const size_t cnt = clip_count(lo, hi, a.n);
      if (cnt) nvls_reduce_bcast<TW>(c.mc_arena + half_off + ring_elem(q % kLaneSlots, r) * sizeof(TW), (cnt + V - 1) / V, a);
      __syncthreads();
      if (t < W) st_release_sys(flag_at(c, t, kOffPipeB, lane, r), v);
    }
    return;
  }
  // -------------------------------------------------------------------- copy CTA
  const int k = role - 1;
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  TW* ring = reinterpret_cast<TW*>(c.arena[r] + half_off);
  const size_t Tk = ((T + Kc - 1) / Kc + V - 1) / V * V;   // this CTA's share of a granule (whole vectors)
  const uint32_t* fB = flag_at(c, r, kOffPipeB, lane, 0);
  for (int q = 0; q < R + 2; q++) {
    if (q < R) {
      const size_t g0 = ((size_t)q * L + lane) * T;
      const size_t s0 = (size_t)k * Tk, s1 = s0 + Tk < T ? s0 + Tk : T;
      for (int j = 0; j < W && s0 < s1; j++) {
        const size_t base = (size_t)j * a.chunk;
        const size_t cend = base + a.chunk;   // the granule may reach past the chunk on its last round
        size_t lo = base + g0 + s0, hi = base + g0 + s1;
        if (hi > cend) hi = cend;
        size_t cnt = lo < hi ? clip_count(lo, hi, a.n) : 0;
        TW* dst = ring + ring_elem(q % kLaneSlots, j) + s0;
        if (cnt) move_tile<TI, TW, false>(dst, in + lo, cnt);
        size_t padded = (cnt + V - 1) / V * V;
        if (cnt && padded > cnt && padded <= s1 - s0) {   // zero-pad the message's last vector for the switch
          TW z = Traits<TW>::from_acc((typename Traits<TW>::A)0);
          for (size_t e = cnt + t; e < padded; e += kThreads) dst[e] = z;
        }
      }
      __syncthreads();
      if (t == 0) st_release_sys(laneIn + k, a.pipe_base + q + 1);
    }
    if (q >= 2) {
      const int qq = q - 2;
      int ok = 1;
      if (t < W) ok = wait_flag(fB + t, a.pipe_base + qq + 1, c, t, kWaitFlagB);
      if (!__syncthreads_and(ok)) return;
      const size_t g0 = ((size_t)qq * L + lane) * T;
      const size_t s0 = (size_t)k * Tk, s1 = s0 + Tk < T ? s0 + Tk : T;
      for (int j = 0; j < W && s0 < s1; j++) {
        const size_t base = (size_t)j * a.chunk;
        const size_t cend = base + a.chunk;
        size_t lo = base + g0 + s0, hi = base + g0 + s1;
        if (hi > cend) hi = cend;
        size_t cnt = lo < hi ? clip_count(lo, hi, a.n) : 0;
        if (cnt) move_tile<TW, TI, true>(out + lo, ring + ring_elem(qq % kLaneSlots, j) + s0, cnt);
      }
    }
  }
}

// Plain local staging copy (user tensor <-> arena region), one CTA per tile, grid-stride.  Used by the
// multi-stream NVLS pipeline, where copies and switch traffic are separate kernels on separate streams.
// BYPASS: the source was written by remote multimem stores (read past L1).
constexpr size_t kStageTileBytes = 32768;
template <typename TS, typename TD, bool BYPASS>
__global__ void __launch_bounds__(kThreads) k_stage_copy(const TS* __restrict__ src, TD* __restrict__ dst, size_t n) {
  constexpr size_t T = kStageTileBytes / (sizeof(TS) > sizeof(TD) ? sizeof(TS) : sizeof(TD));
  for (size_t t0 = (size_t)blockIdx.x * T; t0 < n; t0 += (size_t)gridDim.x * T)
    move_tile<TS, TD, BYPASS>(dst + t0, src + t0, n - t0 < T ? n - t0 : T);
}

// world == 1: no peers, only the wire rounding and the scale remain (the DDP hook at N = 1).
// Grid-stride over 16-byte vectors, four loads in flight per thread; the host sizes the grid to the
// resident capacity (no second, partial wave); HBM-bound (read n, write n).
template <typename TI, typename TW>
__device__ __forceinline__ TI local_scale_one(TI x, const CollArgs& a) {
  using A = typename Traits<TW>::A;
  A v = Traits<TW>::to_acc(Traits<TW>::from_acc((A)Traits<TI>::to_acc(x)));
  if (a.has_scale) v = apply_scale<A>(v, a.scale, 1);
  return Traits<TI>::from_acc((typename Traits<TI>::A)Traits<TW>::to_acc(Traits<TW>::from_acc(v)));
}

template <typename TI, typename TW>
__global__ void __launch_bounds__(kThreads) k_local_scale(const __grid_constant__ CollArgs a) {
  constexpr int VI = 16 / sizeof(TI);
  const TI* in = static_cast<const TI*>(a.in);
  TI* out = static_cast<TI*>(a.out);
  const size_t n = a.n;
  const size_t stride = (size_t)gridDim.x * kThreads;
  const size_t gtid = (size_t)blockIdx.x * kThreads + threadIdx.x;
  if (aligned16(in) && aligned16(out)) {
    const size_t nv = n / VI;
    const uint4* s = reinterpret_cast<const uint4*>(in);
    uint4* d = reinterpret_cast<uint4*>(out);
    size_t i = gtid;
    for (; i + (kUnroll - 1) * stride < nv; i += kUnroll * stride) {
      Pack16<TI> p[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) p[u].u = s[i + u * stride];
#pragma unroll
      for (int u = 0; u < kUnroll; u++) {
#pragma unroll
        for (int e = 0; e < VI; e++) p[u].e[e] = local_scale_one<TI, TW>(p[u].e[e], a);
        d[i + u * stride] = p[u].u;
      }
    }
    for (; i < nv; i += stride) {
      Pack16<TI> p;
      p.u = s[i];
#pragma unroll
      for (int e = 0; e < VI; e++) p.e[e] = local_scale_one<TI, TW>(p.e[e], a);
      d[i] = p.u;
    }
    for (size_t k = nv * VI + gtid; k < n; k += stride) out[k] = local_scale_one<TI, TW>(in[k], a);
  } else {
    for (size_t k = gtid; k < n; k += stride) out[k] = local_scale_one<TI, TW>(in[k], a);
  }
}


// ---------------------------------------------------------------------------------------------
// TMA-staged variant of k_local_scale: the streaming is done by the copy engine, not by LSU
// instructions.  One elected thread issues bulk asynchronous copies (cp.async.bulk, SASS UBLKCP)
// global -> shared, completion is signalled on an mbarrier (complete_tx::bytes); the CTA converts the
// tile in shared memory; the same thread sends it back with a bulk shared -> global copy
// (bulk_group).  kTmaStages tiles are in flight per CTA, so the loads of tiles i+1..i+3 and the store
// of tile i-1 overlap the arithmetic on tile i without costing registers (the LSU version keeps four
// 16-byte vectors per thread in registers and gets 2 CTAs/SM; this one keeps none).
// Requires 16-byte aligned in/out; handles n / tile whole tiles, the caller's plain kernel the rest.
// ---------------------------------------------------------------------------------------------
constexpr int kTmaThreads = 256;
constexpr int kTmaStages = 4;
constexpr int kTmaTileBytes = 16384;
constexpr int kTmaSmemBytes = kTmaStages * kTmaTileBytes + kTmaStages * 8;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

template <typename TI, typename TW>
__global__ void __launch_bounds__(kTmaThreads) k_local_scale_tma(const __grid_constant__ CollArgs a) {
  extern __shared__ __align__(128) unsigned char tma_smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(tma_smem + kTmaStages * kTmaTileBytes);
  constexpr int VI = 16 / sizeof(TI);
  const char* in = static_cast<const char*>(a.in);
  char* out = static_cast<char*>(a.out);
  const size_t ntiles = a.n * sizeof(TI) / kTmaTileBytes;
  const int tid = threadIdx.x;
  const size_t mine = blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  if (tid == 0) {
    for (int s = 0; s < kTmaStages; s++) mbar_init(&bars[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    for (int s = 0; s < kTmaStages && (size_t)s < mine; s++) {
      mbar_expect_tx(&bars[s], kTmaTileBytes);
      bulk_g2s(tma_smem + s * kTmaTileBytes, in + (blockIdx.x + (size_t)s * gridDim.x) * kTmaTileBytes, kTmaTileBytes, &bars[s]);
    }
  }
  for (size_t i = 0; i < mine; i++) {
    const int stage = (int)(i % kTmaStages);
    mbar_wait(&bars[stage], (uint32_t)((i / kTmaStages) & 1));
    uint4* tile = reinterpret_cast<uint4*>(tma_smem + stage * kTmaTileBytes);
#pragma unroll
    for (int j = 0; j < kTmaTileBytes / 16 / kTmaThreads; j++) {
      Pack16<TI> p;
      p.u = tile[tid + j * kTmaThreads];
#pragma unroll
      for (int e = 0; e < VI; e++) p.e[e] = local_scale_one<TI, TW>(p.e[e], a);
      tile[tid + j * kTmaThreads] = p.u;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the copy engine
    __syncthreads();
    if (tid == 0) {
      bulk_s2g(out + (blockIdx.x + i * gridDim.x) * kTmaTileBytes, tile, kTmaTileBytes);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      // the stage converted one iteration ago is free once ITS store has finished reading shared memory
      // (at most the store just issued may still be pending): refill it with the tile kTmaStages ahead
      if (i >= 1 && i - 1 + kTmaStages < mine) {
        asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        const int ps = (int)((i - 1) % kTmaStages);
        mbar_expect_tx(&bars[ps], kTmaTileBytes);
        bulk_g2s(tma_smem + ps * kTmaTileBytes, in + (blockIdx.x + (i - 1 + kTmaStages) * gridDim.x) * kTmaTileBytes, kTmaTileBytes, &bars[ps]);
      }
    }
  }
  if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores must have landed before the CTA retires
}

}  // namespace b200c
