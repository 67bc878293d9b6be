"""Seeded mixed schedules of collectives on loopback worlds of every size from 2 to 8 (one GPU).

The other loopback tests run one kind of operation at a time, with every rank on the same layout.  Here each world
runs about 120 operations drawn from a fixed seed: every allreduce algorithm, dtype and op, the fused gradient means,
reduce, reducescatter, allgather, broadcast (the pipelined unicast rounds included), barrier, send/recv, send_multi,
empty calls, and calls the library must refuse.  The layout is drawn per rank and per pointer: data offsets that put
some ranks on the vector path and others on the scalar path, in place or out of place, and `recv = NULL` on the
non-roots of reduce.  Every buffer of an operation is cut out of one allocation, between 4 KiB of guard bytes.
After every operation:
  * reducing results match the oracle (bit-exact up to NaN payloads) and are the same values on every rank; data
    movement is bit-identical to its source;
  * every byte that is not an output still holds what it held before: the guards, the inputs of out-of-place calls,
    the buffers of reduce's non-roots and of the ranks outside a p2p step;
  * `b200c_comm_seq` is the same on every rank and equals `expected_pieces`, a restatement of the piece arithmetic
    of b200coll.cu, and the launch counter moved by the ranks' pieces plus one per p2p call;
  * a refused call changed neither counter and left `check()` clean, and the next operation still lines up.
A failure names the world, configuration, seed and step and prints the operation, which `run_ops` replays alone.
The schedules themselves are plain Python: the tests without the gpu mark check what they cover on any machine.
"""
import dataclasses
import itertools
import random
from dataclasses import dataclass
from typing import Optional, Tuple

import pytest
import torch

from gpu_common import NATIVE, assert_equal_bits, assert_same_values, bits_of, make_edge_inputs, make_input

from ant_ray_b200 import _native as N
from oracle import oracle as O

KiB, MiB = 1 << 10, 1 << 20
GUARD, GUARD_BYTE = 4 * KiB, 0xA5
ALL_DTYPES = [torch.int8, torch.uint8, torch.int32, torch.uint32, torch.int64, torch.uint64,
              torch.float16, torch.bfloat16, torch.float32, torch.float64]
OPS = {"sum": (N.SUM, O.SUM), "prod": (N.PROD, O.PROD), "max": (N.MAX, O.MAX), "min": (N.MIN, O.MIN), "avg": (N.AVG, O.AVG)}
ALGOS = {"ll": N.ALGO_LL, "oneshot": N.ALGO_ONESHOT, "twoshot": N.ALGO_TWOSHOT, "auto": N.ALGO_AUTO}
# the (bucket, wire) pairs of the fused gradient means
SCALED_PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.float32, torch.float16),
                (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16)]

# Both configurations make pieces frequent (a 256 KiB staging half) and send broadcasts of 64 KiB and more through
# the pipelined unicast rounds (there is no multicast object on one GPU).  One-shot stops at 192 KiB, so that AUTO
# switches from two-shot to one-shot inside one message, and the p2p rings have 64 cells, so that they wrap during a
# schedule.  The second configuration adds max_blocks = 3: block-cyclic walks with many granules per block.
BASE_CONFIG = dict(staging_bytes=256 * KiB, bcast_rounds_min_bytes=64 * KiB, granule_bytes=16 * KiB,
                   oneshot_max_bytes=192 * KiB, p2p_slots=64, timeout_ms=20000)
CONFIGS = {"pieces": BASE_CONFIG, "blockcyclic": dict(BASE_CONFIG, max_blocks=3)}
WORLDS = list(range(2, 9))
SEED = 7101
STEPS = 120
REFUSAL_P = 0.05
P2P = ("sendrecv", "send_multi")


# ---- the piece arithmetic of b200coll.cu, restated ------------------------------------------------------------
def ll_capacity(cfg):
    """Bytes the LL region holds per source: ll_max_bytes rounded up to whole 16-byte vectors (ll_words)."""
    return -(-((cfg.ll_max_bytes + 3) // 4) // 4) * 4 * 4


def oneshot_max(cfg, W):
    return cfg.oneshot_max_bytes or (8 * MiB if W <= 2 else 1 * MiB)


def expected_pieces(kind, W, count, dtype, wire, algo, cfg):
    """The pieces one rank launches for a call, as (what, extent): the caps of b200c_allreduce's planners (LL one
    piece, one-shot staging/W/wsz rounded down to the vector, two-shot W times that, AUTO choosing per piece from
    the bytes left, LL decided on the total), reduce / reducescatter (staging/W/esz, the scaled one in wire
    elements), allgather (staging/W/16*16 bytes), broadcast (staging/16*16 bytes; a piece of at least
    bcast_rounds_min_bytes takes the pipelined rounds) and barrier (one).  Empty calls and p2p take no sequence
    number: an empty list."""
    if kind == "barrier":
        return [("barrier", 0)]
    if count == 0 or kind in P2P:
        return []
    esz = dtype.itemsize
    wsz = (wire or dtype).itemsize
    staging = cfg.staging_bytes
    if kind in ("allreduce", "allreduce_scaled"):
        vec = 16 // wsz
        ll_ok = (wire or dtype) == dtype and count * esz <= ll_capacity(cfg)
        if algo == "ll" or (algo == "auto" and ll_ok and count * esz <= cfg.ll_max_bytes):
            return [("ll", count)]
        slot = staging // W // wsz // vec * vec
        pieces, left = [], count
        while left:
            al = algo if algo != "auto" else ("oneshot" if left * wsz <= oneshot_max(cfg, W) else "twoshot")
            n = min(left, slot if al == "oneshot" else slot * W)
            pieces.append((al, n))
            left -= n
        return pieces
    if kind in ("reduce", "reducescatter", "reducescatter_scaled"):
        unit = wsz if kind == "reducescatter_scaled" else esz
        vec = 16 // unit
        cap = staging // W // unit // vec * vec
        return [(kind, min(cap, count - d)) for d in range(0, count, cap)]
    nbytes = count * esz
    if kind == "allgather":
        cap = staging // W // 16 * 16
        return [(kind, min(cap, nbytes - d)) for d in range(0, nbytes, cap)]
    assert kind == "broadcast", kind
    cap = staging // 16 * 16
    rounds_min = cfg.bcast_rounds_min_bytes
    return [("rounds" if rounds_min and min(cap, nbytes - d) >= rounds_min else "push", min(cap, nbytes - d))
            for d in range(0, nbytes, cap)]


def expected_launches(op, W, cfg):
    """Kernel launches of one operation over all ranks: every rank launches each piece; a p2p call launches one
    kernel per participant unless it moves no bytes."""
    if op.kind == "sendrecv":
        return 2 if op.count else 0
    if op.kind == "send_multi":
        return W if op.count else 0
    return W * len(expected_pieces(op.kind, W, op.count, op.dtype, op.wire, op.algo, cfg))


# ---- operations and their schedules ---------------------------------------------------------------------------
@dataclass
class Op:
    kind: str
    dtype: torch.dtype = torch.float32
    count: int = 0
    algo: str = "-"
    op: str = "sum"
    wire: Optional[torch.dtype] = None
    scale: float = 1.0
    root: int = -1
    peers: Tuple[int, ...] = ()        # sendrecv: (src, dst); send_multi: (writer,)
    edge: bool = False                 # inputs from make_edge_inputs instead of make_input
    seed: int = 0
    offsets: Tuple[Tuple[int, ...], ...] = ()   # [rank][pointer] byte offset of the data, see pointer_names()
    inplace: Tuple[bool, ...] = ()
    recv_null: Tuple[bool, ...] = ()   # reduce: non-roots that pass recv = NULL
    size_class: str = ""
    refusal: str = ""                  # kind == "refused": which refusal, on which rank
    variant: int = 0
    rank: int = -1


def pointer_names(kind, W):
    """The pointers each rank passes, in the order of Op.offsets[rank]."""
    if kind in ("allreduce", "allreduce_scaled", "reduce"):
        return ["send", "recv"]
    if kind in ("reducescatter", "reducescatter_scaled"):
        return [f"send_ptrs[{j}]" for j in range(W)] + ["recv"]
    if kind == "allgather":
        return ["send"] + [f"recv_ptrs[{j}]" for j in range(W)]
    return [] if kind == "barrier" else ["buf"]


def size_classes(kind, W, dtype, wire, algo, cfg):
    """Each operation's boundary sizes in elements, {class: count}, and the largest uniform draw."""
    if kind == "barrier":
        return {"none": 0}, 0
    esz, wsz = dtype.itemsize, (wire or dtype).itemsize
    vec = 16 // wsz
    sizes = {"zero": 0, "one": 1, "vec-1": vec - 1, "vec+1": vec + 1}
    staging = cfg.staging_bytes
    if kind in ("allreduce", "allreduce_scaled"):
        ll = ll_capacity(cfg) // esz
        if algo == "ll":
            sizes.update({"llcap-1": ll - 1, "llcap": ll})
            return sizes, ll
        sizes.update({"llcap-1": ll - 1, "llcap+1": ll + 1})
        cap = staging // W // wsz // vec * vec * (1 if algo == "oneshot" else W)
        if algo == "auto":
            om = oneshot_max(cfg, W) // wsz
            sizes.update({"oneshotmax-1": om - 1, "oneshotmax+1": om + 1})
    elif kind in ("reduce", "reducescatter", "reducescatter_scaled"):
        cap = staging // W // wsz // vec * vec
    elif kind == "allgather":
        cap = staging // W // 16 * 16 // esz
    elif kind == "broadcast":
        cap = staging // 16 * 16 // esz
        sizes.update({"rounds-1": cfg.bcast_rounds_min_bytes // esz - 1, "rounds+1": cfg.bcast_rounds_min_bytes // esz + 1})
    else:
        cap = cfg.p2p_slot_bytes // esz
    sizes.update({"cap-1": cap - 1, "cap": cap, "cap+1": cap + 1, "2cap+vec+3": 2 * cap + vec + 3})
    return sizes, int(3.5 * cap)


def op_kinds(W):
    kinds = [("allreduce", a) for a in ALGOS] + [("allreduce_scaled", a) for a in ALGOS]
    kinds += [(k, "-") for k in ("reduce", "reducescatter", "reducescatter_scaled", "allgather", "broadcast", "barrier", "sendrecv")]
    if W > 2:   # with one reader, send_multi is the pairwise send
        kinds.append(("send_multi", "-"))
    return kinds


KIND_WEIGHT = {"allreduce": 7, "allreduce_scaled": 2, "reduce": 2, "reducescatter": 2, "reducescatter_scaled": 1.5,
               "allgather": 2, "broadcast": 2.5, "barrier": 0.5, "sendrecv": 1, "send_multi": 1}
REFUSALS = ["bad-root", "bad-op", "bad-algo", "bad-dtype", "null-buffer", "scaled-wire", "nvls-without-multicast",
            "ll-over-capacity"]


def _offset(rng, dtype):
    """A data offset in bytes: 0, one element or 8 bytes; 1-byte types also 1..15."""
    if dtype.itemsize == 1:
        return rng.choice([0, 8] + list(range(1, 16)))
    return rng.choice([0, dtype.itemsize, 8])


def _classes(kind, algo):
    return set(size_classes(kind, 4, torch.float32, None, algo, _CLASS_CFG)[0])


class _ClassCfg:   # class names do not depend on the numbers
    staging_bytes, ll_max_bytes, oneshot_max_bytes, bcast_rounds_min_bytes, p2p_slot_bytes = 256 * KiB, 64 * KiB, 0, 64 * KiB, 32 * KiB


_CLASS_CFG = _ClassCfg()


def draw_op(rng, W, cfg, kind, algo, size_class, index, deck):
    op = Op(kind=kind, algo=algo, seed=index)
    if kind == "allreduce":
        op.dtype, op.op = next(deck)
    elif kind in ("allreduce_scaled", "reducescatter_scaled"):
        pairs = [p for p in SCALED_PAIRS if algo != "ll" or p[0] == p[1]]
        op.dtype, op.wire = rng.choice(pairs)
        op.scale = rng.choice([1.0 / W, 0.5, 0.3])
    elif kind in ("reduce", "reducescatter"):
        op.dtype, op.op = rng.choice(ALL_DTYPES), rng.choice(list(OPS))
    elif kind != "barrier":
        op.dtype = rng.choice(ALL_DTYPES)
    sizes, most = size_classes(kind, W, op.dtype, op.wire, algo, cfg)
    op.size_class = size_class or rng.choice(list(sizes) + ["uniform"] * 2 if kind != "barrier" else list(sizes))
    op.count = sizes[op.size_class] if op.size_class != "uniform" else rng.randint(2, most)
    op.edge = kind != "barrier" and rng.random() < 0.25
    mixed = rng.random() < 0.6
    op.offsets = tuple(tuple(_offset(rng, op.dtype) if mixed else 0 for _ in pointer_names(kind, W)) for _ in range(W))
    op.inplace = tuple(rng.random() < 0.5 for _ in range(W))
    if kind in ("reduce", "broadcast"):
        op.root = rng.randrange(W)
    if kind == "reduce":
        op.recv_null = tuple(r != op.root and rng.random() < 0.4 for r in range(W))
    if kind == "sendrecv":
        op.peers = tuple(rng.sample(range(W), 2))
    if kind == "send_multi":
        op.peers = (W - 1,)   # one fixed writer: the native layer binds a writer to one reader set
    return op


def _cycle(rng, items):
    items = list(items)
    rng.shuffle(items)
    return itertools.cycle(items)


def make_schedule(W, cfg_name, seed=SEED, steps=STEPS, cfg=None):
    """About `steps` operations for a world of W ranks: every (operation, algorithm) pair and every size class at
    least once, the rest drawn by weight; the allreduces walk a shuffled deck of every (dtype, op); a refused call
    is slipped in before a step with probability REFUSAL_P."""
    from ant_ray_b200.b200_group import make_config

    cfg = cfg or make_config(**CONFIGS[cfg_name])
    rng = random.Random(f"{seed}/{W}/{cfg_name}")
    kinds = op_kinds(W)
    plan = [(k, a, None) for k, a in kinds]
    for cls in sorted(set().union(*(_classes(k, a) for k, a in kinds))):
        k, a = rng.choice([ka for ka in kinds if cls in _classes(*ka)])
        plan.append((k, a, cls))
    weights = [KIND_WEIGHT[k] / (len(ALGOS) if k.startswith("allreduce") else 1) for k, _ in kinds]
    while len(plan) < steps:
        plan.append((*rng.choices(kinds, weights)[0], None))
    rng.shuffle(plan)
    deck = _cycle(rng, itertools.product(ALL_DTYPES, OPS))
    refusals = _cycle(rng, REFUSALS)
    ops = []
    for kind, algo, cls in plan:
        if rng.random() < REFUSAL_P:
            ops.append(Op(kind="refused", refusal=next(refusals), variant=rng.randrange(8), rank=rng.randrange(W), seed=len(ops)))
        ops.append(draw_op(rng, W, cfg, kind, algo, cls, len(ops), deck))
    return ops


def assert_coverage(ops, W):
    got_pairs = {(o.kind, o.algo) for o in ops}
    missing = set(op_kinds(W)) - got_pairs
    assert not missing, f"W={W}: the schedule lacks {sorted(missing)}"
    want_classes = set().union(*(_classes(k, a) for k, a in op_kinds(W)))
    missing = want_classes - {o.size_class for o in ops}
    assert not missing, f"W={W}: the schedule lacks the size classes {sorted(missing)}"


def _mixed_alignment(op):
    return len({off % 16 == 0 for row in op.offsets for off in row}) > 1


def schedule_stats(ops, W, cfg):
    """What one schedule reaches: operations by kind and algorithm, pipelined broadcasts (ragged ones: a rounds piece
    that is not a whole number of 16-byte vectors), mixed-alignment operations, refusals by kind, AUTO allreduces
    that change algorithm between pieces, and the most pieces of one operation."""
    st = {"ops": {}, "rounds_broadcasts": 0, "ragged_rounds": 0, "mixed_alignment": 0, "refused": {}, "auto_switch": 0,
          "max_pieces": 0}
    for o in ops:
        if o.kind == "refused":
            st["refused"][o.refusal] = st["refused"].get(o.refusal, 0) + 1
            continue
        key = o.kind if o.algo == "-" else f"{o.kind}/{o.algo}"
        st["ops"][key] = st["ops"].get(key, 0) + 1
        pieces = expected_pieces(o.kind, W, o.count, o.dtype, o.wire, o.algo, cfg)
        st["max_pieces"] = max(st["max_pieces"], len(pieces))
        rounds = [n for what, n in pieces if what == "rounds"]
        st["rounds_broadcasts"] += bool(rounds)
        st["ragged_rounds"] += any(n % 16 for n in rounds)
        st["mixed_alignment"] += _mixed_alignment(o)
        st["auto_switch"] += o.algo == "auto" and len({what for what, _ in pieces}) > 1
    return st


# ---- guarded buffers -------------------------------------------------------------------------------------------
@dataclass
class Region:
    name: str
    start: int
    numel: int
    dtype: torch.dtype

    @property
    def end(self):
        return self.start + self.numel * self.dtype.itemsize


class Arena:
    """Every buffer of one operation, cut out of one allocation with GUARD bytes of GUARD_BYTE before and after
    each.  The allocation is 16-byte aligned, so a buffer's alignment is its offset."""

    def __init__(self):
        self.size, self.regions = 0, []

    def carve(self, name, dtype, numel, offset):
        reg = Region(name, self.size + GUARD + offset, numel, dtype)
        self.regions.append(reg)
        self.size = (reg.end + 15) // 16 * 16
        return reg

    def build(self, contents):
        self.host = torch.full((self.size + GUARD,), GUARD_BYTE, dtype=torch.uint8)
        for reg, t in contents:
            if reg.numel:
                self.host[reg.start:reg.end] = bits_of(t).view(torch.uint8)
        self.dev = self.host.cuda()

    def ptr(self, reg):
        return 0 if reg is None else self.dev.data_ptr() + reg.start

    def where(self, i):
        """Which buffer, or which guard, byte i belongs to."""
        for k, reg in enumerate(self.regions):
            if reg.start <= i < reg.end:
                return f"inside {reg.name} (element {(i - reg.start) // reg.dtype.itemsize})"
            if i < reg.start:
                before = f"{i - self.regions[k - 1].end} bytes after {self.regions[k - 1].name}, " if k else ""
                return f"the guard ({before}{reg.start - i} bytes before {reg.name})"
        return f"the guard {i - self.regions[-1].end} bytes after {self.regions[-1].name}"


class Prepared:
    """One operation ready to issue: its buffers, the per-rank call and what every output must hold."""

    def __init__(self, op, W, cfg):
        op = dataclasses.replace(op, offsets=op.offsets or ((0,) * len(pointer_names(op.kind, W)),) * W,
                                 inplace=op.inplace or (False,) * W, recv_null=op.recv_null or (False,) * W)
        self.op, self.W = op, W
        self.pieces = expected_pieces(op.kind, W, op.count, op.dtype, op.wire, op.algo, cfg)
        self.launches = expected_launches(op, W, cfg)
        self.outputs = []   # (region, expected tensor, bit-exact, label)
        self.same = []      # regions that must hold the same bits on every rank
        self.arena = Arena()
        getattr(self, "_" + op.kind)(op, W)

    def _inputs(self, n, salt=0):
        op = self.op
        if op.edge:
            return make_edge_inputs(op.dtype, n, self.W, 1000 * op.seed + salt)
        return [make_input(op.dtype, n, 1000 * op.seed + 16 * salt + r, op.op) for r in range(self.W)]

    def _fold(self, ins):
        op = self.op
        if not op.count:
            return torch.empty(0, dtype=op.dtype)
        if op.wire is not None:
            return O.allreduce_scaled(ins, op.wire, op.scale)
        return O.allreduce(ins, OPS[op.op][1])

    def _out(self, reg, want, exact, what):
        self.outputs.append((reg, want, exact, what))

    def _allreduce(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        send = [A.carve(f"rank {r} send", op.dtype, n, op.offsets[r][0]) for r in range(W)]
        recv = [send[r] if op.inplace[r] else A.carve(f"rank {r} recv", op.dtype, n, op.offsets[r][1]) for r in range(W)]
        A.build(zip(send, ins))
        want = self._fold(ins)
        for r in range(W):
            self._out(recv[r], want, False, f"rank {r} result")
        self.same.append(recv)
        scaled = op.wire is not None

        def call(r, c):
            if scaled:
                c.allreduce_scaled(A.ptr(send[r]), A.ptr(recv[r]), n, NATIVE[op.dtype], NATIVE[op.wire], op.scale, ALGOS[op.algo])
            else:
                c.allreduce(A.ptr(send[r]), A.ptr(recv[r]), n, NATIVE[op.dtype], OPS[op.op][0], ALGOS[op.algo])
        self.call = call

    _allreduce_scaled = _allreduce

    def _reduce(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        send = [A.carve(f"rank {r} send", op.dtype, n, op.offsets[r][0]) for r in range(W)]
        recv = [None if op.recv_null[r] else send[r] if op.inplace[r] else
                A.carve(f"rank {r} recv" + ("" if r == op.root else " (not the root)"), op.dtype, n, op.offsets[r][1])
                for r in range(W)]
        A.build(zip(send, ins))
        self._out(recv[op.root], self._fold(ins), False, f"root {op.root} result")
        self.call = lambda r, c: c.reduce(A.ptr(send[r]), A.ptr(recv[r]), n, NATIVE[op.dtype], OPS[op.op][0], op.root)

    def _reducescatter(self, op, W):
        A, n = self.arena, op.count
        cols = [self._inputs(n, salt=j) for j in range(W)]   # cols[j][s]: rank s's contribution to rank j
        send = [[A.carve(f"rank {r} send_ptrs[{j}]", op.dtype, n, op.offsets[r][j]) for j in range(W)] for r in range(W)]
        recv = [send[r][r] if op.inplace[r] else A.carve(f"rank {r} recv", op.dtype, n, op.offsets[r][W]) for r in range(W)]
        A.build((send[r][j], cols[j][r]) for r in range(W) for j in range(W))
        for r in range(W):
            self._out(recv[r], self._fold(cols[r]), False, f"rank {r} result")
        scaled = op.wire is not None

        def call(r, c):
            ptrs = [A.ptr(s) for s in send[r]]
            if scaled:
                c.reducescatter_scaled(ptrs, A.ptr(recv[r]), n, NATIVE[op.dtype], NATIVE[op.wire], op.scale)
            else:
                c.reducescatter(ptrs, A.ptr(recv[r]), n, NATIVE[op.dtype], OPS[op.op][0])
        self.call = call

    _reducescatter_scaled = _reducescatter

    def _allgather(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        recv = [[A.carve(f"rank {r} recv_ptrs[{j}]", op.dtype, n, op.offsets[r][1 + j]) for j in range(W)] for r in range(W)]
        send = [recv[r][r] if op.inplace[r] else A.carve(f"rank {r} send", op.dtype, n, op.offsets[r][0]) for r in range(W)]
        A.build(zip(send, ins))
        for r in range(W):
            for j in range(W):
                self._out(recv[r][j], ins[j], True, f"rank {r} recv_ptrs[{j}]")
        self.call = lambda r, c: c.allgather(A.ptr(send[r]), [A.ptr(x) for x in recv[r]], n, NATIVE[op.dtype])

    def _broadcast(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        buf = [A.carve(f"rank {r} buf", op.dtype, n, op.offsets[r][0]) for r in range(W)]
        A.build(zip(buf, ins))
        for r in range(W):
            self._out(buf[r], ins[op.root], True, f"rank {r} (root {op.root})")
        self.call = lambda r, c: c.broadcast(A.ptr(buf[r]), n, NATIVE[op.dtype], op.root)

    def _barrier(self, op, W):
        self.arena = None
        self.call = lambda r, c: c.barrier()

    def _sendrecv(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        src, dst = op.peers
        buf = [A.carve(f"rank {r} buf" + ("" if r in op.peers else " (not in this step)"), op.dtype, n, op.offsets[r][0])
               for r in range(W)]
        A.build(zip(buf, ins))
        self._out(buf[dst], ins[src], True, f"rank {dst} received from {src}")
        nbytes = n * op.dtype.itemsize

        def call(r, c):
            if r == src:
                c.send(A.ptr(buf[r]), nbytes, dst)
            elif r == dst:
                c.recv(A.ptr(buf[r]), nbytes, src)
        self.call = call

    def _send_multi(self, op, W):
        A, n, ins = self.arena, op.count, self._inputs(op.count)
        writer = op.peers[0]
        readers = [r for r in range(W) if r != writer]
        buf = [A.carve(f"rank {r} buf", op.dtype, n, op.offsets[r][0]) for r in range(W)]
        A.build(zip(buf, ins))
        for r in readers:
            self._out(buf[r], ins[writer], True, f"rank {r} received from {writer}")
        nbytes = n * op.dtype.itemsize

        def call(r, c):
            if r == writer:
                c.send_multi(A.ptr(buf[r]), nbytes, readers)
            else:
                c.recv_multi(A.ptr(buf[r]), nbytes, writer)
        self.call = call

    def verify(self):
        A = self.arena
        if A is None:
            return
        got = A.dev.cpu()
        rest = A.host.clone()
        for reg, want, exact, what in self.outputs:
            g = got[reg.start:reg.end].clone().view(reg.dtype)
            (assert_equal_bits if exact else assert_same_values)(g, want, what)
            rest[reg.start:reg.end] = got[reg.start:reg.end]
        # Every rank holds the same bits, up to NaN payloads: one-shot and LL fold every rank's copy on that rank, and
        # a rank on the scalar path may hand the same two operands to the multiply or add in the other register
        # order, so where two NaNs of different payloads meet it keeps the other payload (f64 PROD over the edge
        # values at W = 6, mixed layouts).  Every other bit, and where the NaNs are, must agree.
        for group in self.same:
            first = got[group[0].start:group[0].end].clone().view(group[0].dtype)
            for reg in group[1:]:
                assert_same_values(got[reg.start:reg.end].clone().view(reg.dtype), first, f"{reg.name} vs {group[0].name}")
        bad = (got != rest).nonzero().flatten()
        if bad.numel():
            i = int(bad[0])
            raise AssertionError(f"{bad.numel()} bytes outside the outputs changed; the first, byte {i}, lies in "
                                 f"{A.where(i)}: {int(got[i]):#04x}, was {int(rest[i]):#04x}")


def seq_of(c):
    return int(N.load().b200c_comm_seq(c.handle))


def run_ops(world, ops, cfg):
    """Issue `ops` back to back on every rank (one join at the end), then check values, untouched bytes, the
    sequence numbers and the launch count."""
    W = world.world_size
    preps = [Prepared(op, W, cfg) for op in ops]
    seq0, launches0 = [seq_of(c) for c in world.comms], N.launch_count()

    def issue(r, c):
        for p in preps:
            p.call(r, c)
    world.run(issue)
    torch.cuda.synchronize()
    world.check()
    for p in preps:
        p.verify()
    seqs = [seq_of(c) for c in world.comms]
    want = seq0[0] + sum(len(p.pieces) for p in preps)
    assert len(set(seq0)) == 1 and seqs == [want] * W, \
        f"b200c_comm_seq went from {seq0} to {seqs}; the pieces {[p.pieces for p in preps]} give {want}"
    launched = N.launch_count() - launches0
    assert launched == sum(p.launches for p in preps), f"{launched} launches, expected {sum(p.launches for p in preps)}"


def refusal_call(op, W, cfg, p):
    """(status, call) of refusal op.refusal, variant op.variant (modulo the variants): a call every rank refuses
    before it launches anything.  `p` is a valid device pointer of at least 1 MiB."""
    q = op.rank
    ll_over = ll_capacity(cfg) // 4 + 1
    E, U = N.EINVAL, N.EUNSUPPORTED
    table = {
        "bad-root": [(E, lambda c: c.reduce(p, p, 8, N.FLOAT32, N.SUM, W)),
                     (E, lambda c: c.broadcast(p, 8, N.INT32, -1))],
        "bad-op": [(E, lambda c: c.allreduce(p, p, 8, N.FLOAT32, 5, N.ALGO_AUTO)),
                   (E, lambda c: c.reducescatter([p] * W, p, 8, N.INT32, -1)),
                   (E, lambda c: c.reduce(p, p, 8, N.INT64, 9, 0))],
        "bad-algo": [(E, lambda c: c.allreduce(p, p, 8, N.FLOAT32, N.SUM, 8)),
                     (E, lambda c: c.allreduce_scaled(p, p, 8, N.FLOAT32, N.BFLOAT16, 0.5, -1))],
        "bad-dtype": [(E, lambda c: c.allreduce(p, p, 8, 10, N.SUM, N.ALGO_AUTO)),
                      (E, lambda c: c.allgather(p, [p] * W, 8, 11)),
                      (E, lambda c: c.broadcast(p, 8, 10, 0)),
                      (E, lambda c: c.reduce(p, p, 8, -1, N.SUM, 0)),
                      (U, lambda c: c.reducescatter_scaled([p] * W, p, 8, N.INT32, N.INT32, 0.5)),
                      (U, lambda c: c.allreduce_scaled(p, p, 8, N.FLOAT64, N.FLOAT64, 0.5, N.ALGO_AUTO))],
        "null-buffer": [(E, lambda c: c.allreduce(0, p, 8, N.FLOAT32, N.SUM, N.ALGO_AUTO)),
                        (E, lambda c: c.reducescatter([p] * (W - 1) + [0], p, 8, N.INT32, N.SUM)),
                        (E, lambda c: c.allgather(p, [0] + [p] * (W - 1), 8, N.UINT8)),
                        (E, lambda c: c.broadcast(0, 8, N.FLOAT32, 0)),
                        (E, lambda c: c.reduce(p, 0, 8, N.FLOAT32, N.SUM, q))],   # recv may be NULL off the root only
        "scaled-wire": [(U, lambda c: c.allreduce_scaled(p, p, 8, N.FLOAT32, N.FLOAT64, 0.5, N.ALGO_AUTO)),
                        (U, lambda c: c.allreduce_scaled(p, p, 8, N.BFLOAT16, N.FLOAT16, 0.5, N.ALGO_TWOSHOT)),
                        (U, lambda c: c.reducescatter_scaled([p] * W, p, 8, N.FLOAT16, N.BFLOAT16, 0.5))],
        "nvls-without-multicast": [(U, lambda c, a=a: c.allreduce(p, p, 4096, N.FLOAT32, N.SUM, a))
                                   for a in (N.ALGO_NVLS, N.ALGO_NVLS_PIPE, N.ALGO_NVLS_LANES, N.ALGO_NVLS_STREAMS)],
        "ll-over-capacity": [(U, lambda c: c.allreduce(p, p, ll_over, N.FLOAT32, N.SUM, N.ALGO_LL)),
                             (U, lambda c: c.allreduce_scaled(p, p, 100, N.FLOAT32, N.BFLOAT16, 0.5, N.ALGO_LL))],
    }
    variants = table[op.refusal]
    return variants[op.variant % len(variants)]


def refuse(world, op, cfg, scratch_ptr):
    """Issue a refused call on rank op.rank alone: the status, unchanged counters and a clean check()."""
    status, call = refusal_call(op, world.world_size, cfg, scratch_ptr)
    seq0, launches0 = [seq_of(c) for c in world.comms], N.launch_count()
    with pytest.raises(N.B200CollError) as ei:
        call(world.comms[op.rank])
    assert ei.value.status == status, f"status {ei.value.status} ({ei.value}), expected {status}"
    assert [seq_of(c) for c in world.comms] == seq0, "a refused call moved b200c_comm_seq"
    assert N.launch_count() == launches0, "a refused call launched a kernel"
    world.check()


def make_world(W, cfg_name):
    from ant_ray_b200.loopback import LoopbackWorld

    return LoopbackWorld(W, device=0, key=f"sched-{W}-{cfg_name}", **CONFIGS[cfg_name])


# ---- tests that need no GPU: the schedules and the model -------------------------------------------------------
def test_expected_pieces_restates_the_planners():
    """Hand-computed caps at W = 3 with the 256 KiB staging half: the one-shot slot is 87,381 bytes of fp32 rounded
    down to the vector, 21,844 elements; two-shot takes three slots."""
    from ant_ray_b200.b200_group import make_config

    cfg = make_config(**CONFIGS["pieces"])
    f32 = torch.float32
    assert expected_pieces("allreduce", 3, 21_845, f32, None, "oneshot", cfg) == [("oneshot", 21_844), ("oneshot", 1)]
    assert expected_pieces("allreduce", 3, 65_533, f32, None, "twoshot", cfg) == [("twoshot", 65_532), ("twoshot", 1)]
    # AUTO: 150,000 fp32 = 600,000 bytes; two-shot while more than 192 KiB is left, then one-shot slots
    assert expected_pieces("allreduce", 3, 150_000, f32, None, "auto", cfg) == [
        ("twoshot", 65_532), ("twoshot", 65_532), ("oneshot", 18_936)]
    assert expected_pieces("allreduce", 3, 16_384, f32, None, "auto", cfg) == [("ll", 16_384)]
    assert expected_pieces("allreduce_scaled", 3, 16_384, f32, torch.bfloat16, "auto", cfg) == [("oneshot", 16_384)]
    # the scaled reducescatter's pieces are counted in wire elements: bf16 slots hold twice the fp32 ones
    assert len(expected_pieces("reducescatter", 3, 43_689, f32, None, "-", cfg)) == 3
    assert len(expected_pieces("reducescatter_scaled", 3, 43_689, f32, torch.bfloat16, "-", cfg)) == 2
    assert expected_pieces("allgather", 3, 87_377, torch.uint8, None, "-", cfg) == [("allgather", 87_376), ("allgather", 1)]
    assert expected_pieces("broadcast", 3, 65_536 + 256 * KiB, torch.uint8, None, "-", cfg) == [
        ("rounds", 256 * KiB), ("rounds", 65_536)]
    assert expected_pieces("broadcast", 3, 256 * KiB + 100, torch.uint8, None, "-", cfg) == [("rounds", 256 * KiB), ("push", 100)]
    assert expected_pieces("barrier", 3, 0, f32, None, "-", cfg) == [("barrier", 0)]
    assert expected_pieces("reduce", 3, 0, f32, None, "-", cfg) == [] == expected_pieces("sendrecv", 3, 9, f32, None, "-", cfg)


def test_schedules_cover_every_case():
    """Every schedule holds every (operation, algorithm) pair and every size class; over all worlds the schedules hold
    every refusal, every (dtype, op) of allreduce, every (bucket, wire) pair of both fused means, ragged pipelined
    broadcasts, AUTO allreduces that change algorithm between pieces and mixed-alignment operations of every kind."""
    from ant_ray_b200.b200_group import make_config

    refused, dtype_ops, pairs, mixed = set(), set(), set(), set()
    ragged = switches = 0
    for cfg_name in CONFIGS:
        cfg = make_config(**CONFIGS[cfg_name])
        for W in WORLDS:
            ops = make_schedule(W, cfg_name, cfg=cfg)
            assert ops == make_schedule(W, cfg_name, cfg=cfg), "a schedule must be a function of its seed"
            assert_coverage(ops, W)
            st = schedule_stats(ops, W, cfg)
            ragged += st["ragged_rounds"]
            switches += st["auto_switch"]
            refused |= set(st["refused"])
            for o in ops:
                if o.kind == "allreduce":
                    dtype_ops.add((o.dtype, o.op))
                if o.kind in ("allreduce_scaled", "reducescatter_scaled"):
                    pairs.add((o.kind, o.dtype, o.wire))
                if o.kind != "refused" and _mixed_alignment(o) and o.count:
                    mixed.add(o.kind)
    assert refused == set(REFUSALS)
    assert dtype_ops == set(itertools.product(ALL_DTYPES, OPS))
    assert pairs == {(k, d, w) for k in ("allreduce_scaled", "reducescatter_scaled") for d, w in SCALED_PAIRS}
    assert ragged and switches
    assert mixed == {k for k, _ in op_kinds(8)} - {"barrier"}


# ---- the schedules on the GPU ----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", list(CONFIGS))
@pytest.mark.parametrize("W", WORLDS)
def test_seeded_schedule(W, cfg_name):
    ops = make_schedule(W, cfg_name)
    assert_coverage(ops, W)
    world = make_world(W, cfg_name)
    try:
        cfg = world.comms[0].config
        scratch = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
        for i, op in enumerate(ops):
            try:
                if op.kind == "refused":
                    refuse(world, op, cfg, scratch.data_ptr())
                else:
                    run_ops(world, [op], cfg)
            except Exception as e:  # noqa: BLE001
                raise AssertionError(
                    f"W={W} config={cfg_name} {CONFIGS[cfg_name]} seed={SEED}, step {i} of {len(ops)}: {op}\n"
                    f"  (replay: run_ops(world, [make_schedule({W}, {cfg_name!r})[{i}]], cfg))\n"
                    f"  {type(e).__name__}: {e}") from e
    finally:
        world.destroy()


# ---- deterministic cases ---------------------------------------------------------------------------------------
def _uniform(W, P, off=0):
    return tuple(tuple(off for _ in range(P)) for _ in range(W))


@pytest.mark.gpu
@pytest.mark.parametrize("cfg_name", list(CONFIGS))
@pytest.mark.parametrize("W", WORLDS)
def test_pipelined_unicast_broadcast(W, cfg_name):
    """k_broadcast_rounds with symmetric == 3 (no multicast object): a ragged last granule, unaligned roots and
    receivers, a message whose last piece falls below the rounds threshold and one whose last piece stays above it,
    and three rounds broadcasts back to back, whose different sizes give different grids on one pipe_base epoch."""
    world = make_world(W, cfg_name)
    try:
        cfg = world.comms[0].config
        staging = cfg.staging_bytes
        cases = [
            # 100 KiB + 5 bytes: one rounds piece, n % 16 != 0; the root 3 bytes off, receivers at 16 offsets
            Op("broadcast", torch.uint8, 100 * KiB + 5, root=W - 1, seed=1,
               offsets=tuple((3 if r == W - 1 else 5 * r % 16,) for r in range(W))),
            # one full rounds piece, then 1000 bytes by the plain push; root one element off, receivers alternate
            Op("broadcast", torch.float32, (staging + 1000) // 4, root=0, seed=2,
               offsets=tuple(((4, 0, 8)[r % 3],) for r in range(W))),
            # the last piece (100 KiB + 6 bytes) is above the threshold and ragged
            Op("broadcast", torch.bfloat16, (staging + 100 * KiB) // 2 + 3, root=W // 2, seed=3, edge=True,
               offsets=tuple(((0, 2, 8)[r % 3],) for r in range(W))),
        ]
        want = [["rounds"], ["rounds", "push"], ["rounds", "rounds"]]
        for op, kinds in zip(cases, want):
            assert [k for k, _ in expected_pieces("broadcast", W, op.count, op.dtype, None, "-", cfg)] == kinds
            run_ops(world, [op], cfg)
        back_to_back = [Op("broadcast", torch.uint8, n, root=root % W, seed=10 + i, offsets=_uniform(W, 1, off))
                        for i, (n, root, off) in enumerate(((64 * KiB, 1, 0), (150 * KiB + 7, 0, 1), (staging - 16, 2, 0)))]
        for op in back_to_back:
            assert [k for k, _ in expected_pieces("broadcast", W, op.count, op.dtype, None, "-", cfg)] == ["rounds"]
        run_ops(world, back_to_back, cfg)
    finally:
        world.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("W", WORLDS)
def test_per_pointer_alignment(W):
    """Allgather whose recv_ptrs[j] each sit at another offset, reducescatter whose send_ptrs[j] each do, and LL where
    rank 0 is aligned and its peers sit one element off (every other rank), in place and out of place."""
    world = make_world(W, "pieces")
    try:
        cfg = world.comms[0].config
        ag_cap = cfg.staging_bytes // W // 16 * 16
        for dtype, offs in ((torch.uint8, lambda r, j: (3 * j + r) % 16), (torch.bfloat16, lambda r, j: (0, 2, 8)[(j + r) % 3])):
            n = (ag_cap + 37) // dtype.itemsize
            offsets = tuple((offs(r, W),) + tuple(offs(r, j) for j in range(W)) for r in range(W))
            run_ops(world, [Op("allgather", dtype, n, seed=20, offsets=offsets, inplace=tuple(r % 2 == 1 for r in range(W)))], cfg)
        rs_cap = cfg.staging_bytes // W
        for dtype, opname, offs in ((torch.int8, "sum", lambda r, j: (5 * j + r) % 16),
                                    (torch.float32, "max", lambda r, j: (0, 4, 8)[(j + r) % 3])):
            n = rs_cap // dtype.itemsize + 17
            offsets = tuple(tuple(offs(r, j) for j in range(W)) + (8,) for r in range(W))
            run_ops(world, [Op("reducescatter", dtype, n, op=opname, seed=21, edge=dtype.is_floating_point, offsets=offsets,
                               inplace=tuple(r % 2 == 0 for r in range(W)))], cfg)
        for dtype in (torch.float16, torch.int32, torch.float64, torch.uint8):
            e = dtype.itemsize
            for n in (1003, ll_capacity(cfg) // e):
                offsets = tuple(((0, 0) if r % 2 == 0 else (e, 8 if e < 8 else 0)) for r in range(W))
                run_ops(world, [Op("allreduce", dtype, n, algo="ll", seed=22, offsets=offsets,
                                   inplace=tuple(r % 3 != 1 for r in range(W)))], cfg)
    finally:
        world.destroy()
