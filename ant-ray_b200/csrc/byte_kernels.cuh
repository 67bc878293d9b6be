// Untyped (byte-moving) kernels: allgather, broadcast, barrier, p2p send/recv.
// Included by exactly one translation unit (b200coll.cu).
#pragma once
#include "coll_kernels.cuh"

namespace b200c {

// ---------------------------------------------------------------------------------------------
// allgather: push own tensor to slot [r] of every peer, then copy the W slots into the caller's
// W output tensors (out_ptrs[j]).  Pure byte movement -> instantiated once (uint8_t).
// broadcast: root pushes into slot 0 of every peer; peers copy out.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads) k_allgather(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world;
  if (!coll_prologue(a)) return;
  const size_t slot_bytes = a.chunk;                       // n = bytes per rank
  const uint8_t* in = static_cast<const uint8_t*>(a.in);
  uint8_t* own_out = static_cast<uint8_t*>(a.out_ptrs[r]);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    for (int k = 1; k < W; k++)
      copy_tile<uint8_t, false>(staging_ptr<uint8_t>(c, peer_at(r, k, W), a.seq, (size_t)r * slot_bytes) + t0, in + t0, t1 - t0);
    if (own_out != in) copy_tile<uint8_t, false>(own_out + t0, in + t0, t1 - t0);
  }
  block_signal_all(kOffFlagA, a.seq, c);
  if (!block_wait_all(kOffFlagA, a.seq, c, kWaitFlagA)) return;
  check_signature(a);
  B200C_FOR_GRANULES(t0, t1, a, a.n) {
    for (int k = 1; k < W; k++) {
      const int j = peer_at(r, k, W);
      copy_tile<uint8_t, true>(static_cast<uint8_t*>(a.out_ptrs[j]) + t0, staging_ptr<uint8_t>(c, r, a.seq, (size_t)j * slot_bytes) + t0, t1 - t0);
    }
  }
}

// nv 16-byte vectors: src (plain or staging) -> multicast address
template <bool SRC_BYPASS>
__device__ __forceinline__ void multicast_tile(char* mc, const uint4* s, size_t nv) {
  size_t i = threadIdx.x;
  for (; i + (size_t)(kUnroll - 1) * kThreads < nv; i += (size_t)kUnroll * kThreads) {
    uint4 v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) v[u] = SRC_BYPASS ? ld_bypass16(s + i + (size_t)u * kThreads) : s[i + (size_t)u * kThreads];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) multimem_st16(mc + (i + (size_t)u * kThreads) * 16, v[u]);
  }
  for (; i < nv; i += kThreads) multimem_st16(mc + i * 16, SRC_BYPASS ? ld_bypass16(s + i) : s[i]);
}

// a.symmetric selects the variant:
//   0  unicast: the root pushes every granule into slot 0 of every peer (egress (W-1)*S);
//   1  root multicast: the root stores each 16-byte vector ONCE to the multicast address of staging
//      slot 0 and the NVSwitch replicates it (egress S); the sub-vector tail and unaligned sources go
//      by unicast stores.
__global__ void __launch_bounds__(kThreads) k_broadcast(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world, root = a.root;
  if (!coll_prologue(a)) return;
  if (r == root) {
    B200C_FOR_GRANULES(t0, t1, a, a.n) {
      const size_t cnt = t1 - t0;
      const uint8_t* src = static_cast<const uint8_t*>(a.in) + t0;
      size_t done = 0;
      if (a.symmetric && c.mc_arena && aligned16(src)) {
        const size_t nv = cnt / 16;
        multicast_tile<false>(c.mc_arena + c.off_staging + (size_t)(a.seq & 1) * c.staging_bytes + t0, reinterpret_cast<const uint4*>(src), nv);
        done = nv * 16;
      }
      if (done < cnt) {
        for (int k = 1; k < W; k++)
          copy_tile<uint8_t, false>(staging_ptr<uint8_t>(c, peer_at(r, k, W), a.seq, 0) + t0 + done, src + done, cnt - done);
      }
    }
    block_signal_all(kOffFlagA, a.seq, c);
  } else {
    if (!block_wait_one(flag_at(c, r, kOffFlagA, blockIdx.x, root), a.seq, c, root, kWaitFlagA)) return;
    check_signature(a);
    B200C_FOR_GRANULES(t0, t1, a, a.n) {
      copy_tile<uint8_t, true>(static_cast<uint8_t*>(a.out) + t0, staging_ptr<uint8_t>(c, r, a.seq, 0) + t0, t1 - t0);
    }
  }
}

// Scatter + multicast-allgather broadcast for large messages (W > 2, multicast bound, 16-byte aligned,
// n a multiple of 16): the message is cut into W rank chunks (a.chunk bytes).  Per round (one granule of
// every chunk per block):
//   root    : unicast-pushes the granule of chunk j into rank j's staging (its natural offset) and
//             multicasts the granule of its own chunk straight from user memory; raises pipeA on every
//             peer ("your granule has landed") and pipeB ("chunk[root] granule is everywhere");
//   rank j  : waits pipeA(root), re-multicasts its granule from its staging to everybody, raises pipeB;
//             then waits pipeB of every other rank for the previous round and copies that round's W
//             granules out of its staging into the user buffer.
// Root egress is ~S (unicast (W-1)/W*S + multicast S/W) instead of (W-1)*S, and — unlike the root-only
// multicast — the W-1 receivers share the multicast work, so no single multimem.st stream is the bottleneck.
__global__ void __launch_bounds__(kThreads, 2) k_broadcast_rounds(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world, root = a.root;
  if (!coll_prologue(a)) return;
  check_signature(a);
  const size_t half_off = c.off_staging + (size_t)(a.seq & 1) * c.staging_bytes;
  uint8_t* mine = reinterpret_cast<uint8_t*>(c.arena[r] + half_off);
  const BlockRounds rd(a);
  if (rd.empty()) return;
  const int R = rd.count();
  const int t = threadIdx.x;
  if (a.symmetric == 3) {
    // Unicast rounds (world of two, or no multicast object): chunk == the whole message.  The root pushes
    // granule q to every peer and raises pipeA; a peer copies granule q out as soon as it has landed, so
    // the root's NVLink stores and the peers' local copies overlap instead of running back to back.
    if (r == root) {
      const uint8_t* src = static_cast<const uint8_t*>(a.in);
      for (int q = 0; q < R; q++) {
        const auto [g0, cnt] = chunk_span(a, 0, rd.lo(q), rd.hi(q));
        for (int k = 1; k < W && cnt; k++)
          copy_tile<uint8_t, false>(reinterpret_cast<uint8_t*>(c.arena[peer_at(r, k, W)] + half_off) + g0, src + g0, cnt);
        block_signal_all(kOffPipeA, a.pipe_base + q + 1, c);
      }
      return;
    }
    uint8_t* out = static_cast<uint8_t*>(a.out);
    const uint32_t* fA = flag_at(c, r, kOffPipeA, blockIdx.x, root);
    for (int q = 0; q < R; q++) {
      if (!block_wait_one(fA, a.pipe_base + q + 1, c, root, kWaitFlagA)) return;
      const auto [g0, cnt] = chunk_span(a, 0, rd.lo(q), rd.hi(q));
      if (cnt) copy_tile<uint8_t, true>(out + g0, mine + g0, cnt);
    }
    return;
  }
  // the multicast rounds clip by hand: chunk_span() here changes this kernel's register allocation
  char* mc = c.mc_arena + half_off;
  if (r == root) {
    const uint8_t* src = static_cast<const uint8_t*>(a.in);
    for (int q = 0; q < R; q++) {
      const size_t g0 = rd.lo(q), g1 = rd.hi(q);
      for (int k = 1; k < W; k++) {
        const int j = peer_at(r, k, W);
        size_t lo = (size_t)j * a.chunk + g0;
        size_t cnt = clip_count(lo, (size_t)j * a.chunk + g1, a.n);
        if (cnt) copy_tile<uint8_t, false>(reinterpret_cast<uint8_t*>(c.arena[j] + half_off) + lo, src + lo, cnt);
      }
      {
        size_t lo = (size_t)r * a.chunk + g0;
        size_t cnt = clip_count(lo, (size_t)r * a.chunk + g1, a.n);
        if (cnt) multicast_tile<false>(mc + lo, reinterpret_cast<const uint4*>(src + lo), cnt / 16);
      }
      __syncthreads();
      if (t < W && t != r) {
        // one fence covers both flags of this peer
        asm volatile("fence.acq_rel.sys;" ::: "memory");
        st_relaxed_sys(flag_at(c, t, kOffPipeA, blockIdx.x, r), a.pipe_base + q + 1);
        st_relaxed_sys(flag_at(c, t, kOffPipeB, blockIdx.x, r), a.pipe_base + q + 1);
      }
    }
    return;
  }
  uint8_t* out = static_cast<uint8_t*>(a.out);
  const uint32_t* fA = flag_at(c, r, kOffPipeA, blockIdx.x, root);
  for (int q = 0; q <= R; q++) {
    if (q < R) {
      if (!block_wait_one(fA, a.pipe_base + q + 1, c, root, kWaitFlagA)) return;
      size_t lo = (size_t)r * a.chunk + rd.lo(q);
      size_t cnt = clip_count(lo, (size_t)r * a.chunk + rd.hi(q), a.n);
      if (cnt) multicast_tile<true>(mc + lo, reinterpret_cast<const uint4*>(mine + lo), cnt / 16);
      block_signal_all(kOffPipeB, a.pipe_base + q + 1, c);
    }
    if (q >= 1) {
      if (!block_wait_all(kOffPipeB, a.pipe_base + q, c, kWaitFlagB)) return;
      for (int j = 0; j < W; j++) {
        size_t lo = (size_t)j * a.chunk + rd.lo(q - 1);
        size_t cnt = clip_count(lo, (size_t)j * a.chunk + rd.hi(q - 1), a.n);
        if (cnt) copy_tile<uint8_t, true>(out + lo, mine + lo, cnt);
      }
    }
  }
}

// barrier: arrive[] exchange only (the prologue publishes arrive = seq; wait for everyone at seq).
__global__ void __launch_bounds__(32) k_barrier(const __grid_constant__ CollArgs a) {
  const DevComm& c = a.c;
  int t = threadIdx.x;
  if (t < c.world && t != c.rank) {
    st_release_sys(flag_at(c, t, kOffArrive, 0, c.rank), a.seq);
    wait_flag(flag_at(c, c.rank, kOffArrive, 0, t), a.seq, c, t, kWaitArrive);
  }
}

// ---------------------------------------------------------------------------------------------
// p2p: ring of cells in the receiver's arena, one ready flag and one ack flag per cell.
// Cell k of the pair's lifetime lives at ring position k % cells and carries flag value k+1.
// The same two kernels serve the pairwise rings (one per ordered pair) and the multi-reader rings
// (one per source rank, identical offset in every arena): only the offsets in P2PArgs differ.
// ---------------------------------------------------------------------------------------------
struct P2PArgs {
  DevComm c;
  void* buf;          // user buffer (send: source, recv: destination)
  size_t bytes;
  int peer;           // recv: source rank; pairwise send: destination rank
  uint32_t first_cell;  // cumulative cell index of this message's first cell
  uint32_t ncells;
  size_t off_ring;    // arena offset of ring [8 src][cells][cell_bytes]
  size_t off_ready;   // pad offset of ready[8 src][kMaxCells]   (lives on the receiver)
  size_t off_ack;     // pad offset of ack[8 dst][kMaxCells]     (lives on the sender)
  int cells;
  uint32_t reader_mask;  // multi-reader send: bit j = rank j receives this message
  int batch;          // pairwise send: cells published per release fence (1..kSendBatch)
};

// A system-scope release fence costs far more while the SM's other warps stream stores to the peer than
// on a quiet SM, so a sender block publishes kSendBatch
// cells per fence: copy cells i, i+grid, ... , then one __syncthreads + fence and one flag per cell.
constexpr int kSendBatch = 4;

__global__ void __launch_bounds__(kThreads) k_send(const __grid_constant__ P2PArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, d = a.peer, t = threadIdx.x;
  const size_t cb = c.p2p_cell_bytes;
  const uint8_t* src = static_cast<const uint8_t*>(a.buf);
  const int B = a.batch;
  for (uint32_t i0 = blockIdx.x; i0 < a.ncells; i0 += gridDim.x * B) {
    // the previous occupants of these ring positions (cell k - cells) must have been consumed
    int ok = 1;
    if (t < B) {
      uint32_t i = i0 + (uint32_t)t * gridDim.x, k = a.first_cell + i;
      if (i < a.ncells && k >= (uint32_t)a.cells) {
        uint32_t pos = k % (uint32_t)a.cells;
        ok = wait_flag(reinterpret_cast<const uint32_t*>(c.arena[r] + a.off_ack) + (size_t)d * kMaxCells + pos, k + 1 - (uint32_t)a.cells, c, d, kWaitP2PAck);
      }
    }
    if (!__syncthreads_and(ok)) return;
#pragma unroll 1
    for (int b = 0; b < B; b++) {
      uint32_t i = i0 + (uint32_t)b * gridDim.x;
      if (i >= a.ncells) break;
      uint32_t pos = (a.first_cell + i) % (uint32_t)a.cells;
      size_t off = (size_t)i * cb;
      size_t cnt = a.bytes - off < cb ? a.bytes - off : cb;
      copy_tile<uint8_t, false>(reinterpret_cast<uint8_t*>(c.arena[d] + a.off_ring + ((size_t)r * a.cells + pos) * cb), src + off, cnt);
    }
    __syncthreads();
    if (t == 0) {
      asm volatile("fence.acq_rel.sys;" ::: "memory");
      for (int b = 0; b < B; b++) {
        uint32_t i = i0 + (uint32_t)b * gridDim.x;
        if (i >= a.ncells) break;
        uint32_t k = a.first_cell + i;
        st_relaxed_sys(reinterpret_cast<uint32_t*>(c.arena[d] + a.off_ready) + (size_t)r * kMaxCells + k % (uint32_t)a.cells, k + 1);
      }
    }
  }
}

// Multi-reader send (the reference sends once per reader: torch_tensor_accelerator_channel.py:586-590,
// "TODO: If there are multiple readers, can replace with a broadcast").  Every cell is written ONCE to
// the multicast address of this rank's ring — the NVSwitch replicates it into every arena — when a
// multicast object is bound and the source is 16-byte aligned; otherwise once per reader by unicast.
// Flow control is per reader: a ring position is reused only after every reader of the (fixed) reader
// set has acknowledged its previous occupant.
__global__ void __launch_bounds__(kThreads) k_send_multi(const __grid_constant__ P2PArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, W = c.world, t = threadIdx.x;
  const size_t cb = c.p2p_cell_bytes;
  const uint8_t* src = static_cast<const uint8_t*>(a.buf);
  const bool reader = t < W && ((a.reader_mask >> t) & 1u);
  for (uint32_t i = blockIdx.x; i < a.ncells; i += gridDim.x) {
    uint32_t k = a.first_cell + i;
    uint32_t pos = k % (uint32_t)a.cells;
    if (k >= (uint32_t)a.cells) {
      int ok = 1;
      if (reader) ok = wait_flag(reinterpret_cast<const uint32_t*>(c.arena[r] + a.off_ack) + (size_t)t * kMaxCells + pos, k + 1 - (uint32_t)a.cells, c, t, kWaitP2PAck);
      if (!__syncthreads_and(ok)) return;
    }
    size_t off = (size_t)i * cb;
    size_t cnt = a.bytes - off < cb ? a.bytes - off : cb;
    const size_t cell_off = a.off_ring + ((size_t)r * a.cells + pos) * cb;
    size_t done = 0;
    if (c.mc_arena && aligned16(src + off)) {
      multicast_tile<false>(c.mc_arena + cell_off, reinterpret_cast<const uint4*>(src + off), cnt / 16);
      done = cnt / 16 * 16;
    }
    if (done < cnt) {
      for (int j = 0; j < W; j++)
        if ((a.reader_mask >> j) & 1u) copy_tile<uint8_t, false>(reinterpret_cast<uint8_t*>(c.arena[j] + cell_off) + done, src + off + done, cnt - done);
    }
    __syncthreads();
    if (reader) st_release_sys(reinterpret_cast<uint32_t*>(c.arena[t] + a.off_ready) + (size_t)r * kMaxCells + pos, k + 1);
  }
}

__global__ void __launch_bounds__(kThreads) k_recv(const __grid_constant__ P2PArgs a) {
  const DevComm& c = a.c;
  const int r = c.rank, s = a.peer;
  const size_t cb = c.p2p_cell_bytes;
  uint8_t* dstbuf = static_cast<uint8_t*>(a.buf);
  for (uint32_t i = blockIdx.x; i < a.ncells; i += gridDim.x) {
    uint32_t k = a.first_cell + i;
    uint32_t pos = k % (uint32_t)a.cells;
    const uint32_t* ready = reinterpret_cast<const uint32_t*>(c.arena[r] + a.off_ready) + (size_t)s * kMaxCells + pos;
    if (!block_wait_one(ready, k + 1, c, s, kWaitP2PReady)) return;
    size_t off = (size_t)i * cb;
    size_t cnt = a.bytes - off < cb ? a.bytes - off : cb;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(c.arena[r] + a.off_ring + ((size_t)s * a.cells + pos) * cb);
    copy_tile<uint8_t, true>(dstbuf + off, src, cnt);
    __syncthreads();
    if (threadIdx.x == 0)
      st_release_sys(reinterpret_cast<uint32_t*>(c.arena[s] + a.off_ack) + (size_t)r * kMaxCells + pos, k + 1);
  }
}

}  // namespace b200c
