"""The reducing kernels at value edges, compared bit for bit with the CPU oracle on ONE GPU.

Inputs come from gpu_common.make_edge_inputs: every element is a value where reductions go wrong
(NaN with and without payload, +-Inf, +-0, subnormals, max / overflowing sums, f16 / bf16 rounding
ties, integer min / max / wrap-around / high words), and fixed blocks put every ordered pair of them
at the first and at the last two ranks.  Checks: every rank matches the oracle (bit-exact except
that NaN matches NaN whatever its bits; x86 and the GPU make different NaNs), every rank holds the
same bits as rank 0, and no kernel recorded an error.

Loopback worlds of 2 and 8 ranks run the kernels compiled for that world size, 3 ranks the kernels
that take the world size at run time.  A 1 MiB staging half makes the multi-piece sizes cheap.
"""
import pytest
import torch

from gpu_common import FLOAT_DTYPES, INT_DTYPES, NATIVE, assert_equal_bits, assert_same_values, bits_of, make_edge_inputs

from ant_ray_b200 import _native as N
from oracle import oracle as O

pytestmark = pytest.mark.gpu

DTYPES = INT_DTYPES + FLOAT_DTYPES
OPS = {"sum": (N.SUM, O.SUM), "prod": (N.PROD, O.PROD), "max": (N.MAX, O.MAX), "min": (N.MIN, O.MIN), "avg": (N.AVG, O.AVG)}
STAGING = 1 << 20


def _esz(dtype):
    return torch.empty((), dtype=dtype).element_size()


def _sizes(dtype, W=1):
    """A tail (one 16-byte vector + 3 elements), a mid size that holds the fixed blocks of every pattern,
    and 1.5 times the largest piece: a staging half (two-shot allreduce), or one rank's slot of it
    (reduce and reducescatter, W > 1)."""
    return [16 // _esz(dtype) + 3, 4099, (3 * STAGING) // (2 * W * _esz(dtype)) + 3]


@pytest.fixture(scope="module", params=[2, 3, 8])
def world(request):
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(request.param, device=0, key=f"edges{request.param}", staging_bytes=STAGING, timeout_ms=20000)
    yield w
    w.destroy()


def _check(outs, want, what):
    """Rank 0 matches the oracle; every other rank holds rank 0's bits."""
    first = outs[0].cpu()
    assert_same_values(first, want, f"{what} rank=0")
    for r, o in enumerate(outs[1:], 1):
        assert torch.equal(bits_of(o.cpu()), bits_of(first)), f"{what}: rank {r} and rank 0 disagree"


def _allreduce(world, dtype, n, opname, algo, seed, inplace=True, offset=0):
    W = world.world_size
    nat, orc = OPS[opname]
    ins = make_edge_inputs(dtype, n + offset, W, seed)
    dev = [t.cuda() for t in ins]
    out = dev if inplace else [torch.empty_like(t) for t in dev]
    world.run(lambda r, c: c.allreduce(dev[r][offset:].data_ptr(), out[r][offset:].data_ptr(), n, NATIVE[dtype], nat, algo))
    torch.cuda.synchronize()
    world.check()
    what = f"allreduce {dtype} {opname} n={n} algo={algo} inplace={inplace} offset={offset}"
    _check([o[offset:] for o in out], O.allreduce([t[offset:] for t in ins], orc), what)
    for r in range(W):
        if offset:
            assert_equal_bits(out[r][:offset], ins[r][:offset], f"{what}: element before the view")
        if not inplace:
            assert_equal_bits(dev[r], ins[r], f"{what}: input must be untouched")


@pytest.mark.parametrize("opname", list(OPS))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_allreduce_edges(world, dtype, opname):
    ll_cap = 64 << 10   # default ll_max_bytes
    for seed, n in enumerate(_sizes(dtype)):
        for algo in (N.ALGO_LL, N.ALGO_ONESHOT, N.ALGO_TWOSHOT):
            if algo == N.ALGO_LL and n * _esz(dtype) > ll_cap:
                continue
            _allreduce(world, dtype, n, opname, algo, seed)
    _allreduce(world, dtype, 4099, opname, N.ALGO_TWOSHOT, 7, inplace=False)
    for algo in (N.ALGO_ONESHOT, N.ALGO_TWOSHOT):   # a view one element into its allocation: the scalar path
        _allreduce(world, dtype, 4099, opname, algo, 8, offset=1)


@pytest.mark.parametrize("opname", list(OPS))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_reduce_edges(world, dtype, opname):
    W = world.world_size
    nat, orc = OPS[opname]
    for root in (0, W - 1):
        for seed, n in enumerate(_sizes(dtype, W)):
            ins = make_edge_inputs(dtype, n, W, 10 * root + seed)
            dev = [t.cuda() for t in ins]
            world.run(lambda r, c: c.reduce(dev[r].data_ptr(), dev[r].data_ptr(), n, NATIVE[dtype], nat, root))
            torch.cuda.synchronize()
            world.check()
            what = f"reduce {dtype} {opname} n={n} root={root}"
            assert_same_values(dev[root], O.reduce(ins, orc), what)
            for r in range(W):
                if r != root:
                    assert_equal_bits(dev[r], ins[r], f"{what}: non-root rank {r} must be untouched")


@pytest.mark.parametrize("opname", list(OPS))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_reducescatter_edges(world, dtype, opname):
    W = world.world_size
    nat, orc = OPS[opname]
    for seed, n in enumerate(_sizes(dtype, W)):
        per_dst = [make_edge_inputs(dtype, n, W, 100 * seed + j) for j in range(W)]   # per_dst[j][r]: rank r's part for rank j
        lists = [[per_dst[j][r] for j in range(W)] for r in range(W)]
        dev = [[t.cuda() for t in row] for row in lists]
        outs = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(W)]
        world.run(lambda r, c: c.reducescatter([t.data_ptr() for t in dev[r]], outs[r].data_ptr(), n, NATIVE[dtype], nat))
        torch.cuda.synchronize()
        world.check()
        want = O.reducescatter(lists, orc)
        for r in range(W):
            assert_same_values(outs[r], want[r], f"reducescatter {dtype} {opname} n={n} rank={r}")


@pytest.mark.parametrize("bucket,wire,algo", [
    (torch.float32, torch.float32, N.ALGO_ONESHOT), (torch.float32, torch.float32, N.ALGO_TWOSHOT),
    (torch.float32, torch.float32, N.ALGO_LL),
    (torch.float32, torch.bfloat16, N.ALGO_ONESHOT), (torch.float32, torch.bfloat16, N.ALGO_TWOSHOT),
    (torch.float32, torch.float16, N.ALGO_ONESHOT), (torch.float32, torch.float16, N.ALGO_TWOSHOT),
    (torch.bfloat16, torch.bfloat16, N.ALGO_ONESHOT), (torch.bfloat16, torch.bfloat16, N.ALGO_TWOSHOT),
    (torch.float16, torch.float16, N.ALGO_ONESHOT), (torch.float16, torch.float16, N.ALGO_TWOSHOT),
], ids=str)
def test_fused_mean_edges(world, bucket, wire, algo):
    """The fused gradient mean rounds every contribution to the wire, sums in fp32 and rounds ONCE after
    the 1/W scale: a contribution that overflows the f16 wire is Inf, a sum that would overflow before
    the scale is not."""
    W = world.world_size
    for seed, n in enumerate(_sizes(bucket)):
        if algo == N.ALGO_LL and n * _esz(bucket) > (64 << 10):
            continue
        ins = make_edge_inputs(bucket, n, W, 50 + seed)
        dev = [t.cuda() for t in ins]
        world.run(lambda r, c: c.allreduce_scaled(dev[r].data_ptr(), dev[r].data_ptr(), n, NATIVE[bucket], NATIVE[wire], 1.0 / W, algo))
        torch.cuda.synchronize()
        world.check()
        want = O.allreduce_scaled(ins, None if wire == bucket else wire, 1.0 / W)
        _check(dev, want, f"fused mean {bucket} wire={wire} algo={algo} n={n}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_nan_bits(world, dtype):
    """The reducing kernels round to f16 / bf16 with __float2half_rn / __float2bfloat16_rn, whose NaN is
    0x7fff, the NaN the oracle produces: half-precision outputs match the oracle bit for bit, NaNs included."""
    W = world.world_size
    for opname in ("sum", "max"):
        ins = make_edge_inputs(dtype, 4099, W, 9)
        dev = [t.cuda() for t in ins]
        world.run(lambda r, c: c.allreduce(dev[r].data_ptr(), dev[r].data_ptr(), 4099, NATIVE[dtype], OPS[opname][0], N.ALGO_ONESHOT))
        torch.cuda.synchronize()
        world.check()
        want = O.allreduce(ins, OPS[opname][1])
        assert bool(want.isnan().any())
        for r in range(W):
            assert_equal_bits(bits_of(dev[r].cpu()), bits_of(want), f"{dtype} {opname} rank={r}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32, torch.float64])
def test_data_movement_keeps_nan_payloads(world, dtype):
    """allgather, broadcast and send/recv are byte copies: NaN payloads and signs come back bit-identical."""
    W = world.world_size
    for seed, n in enumerate((16 // _esz(dtype) + 3, 50_001)):
        ins = make_edge_inputs(dtype, n, W, 300 + seed)
        dev = [t.cuda() for t in ins]
        outs = [[torch.zeros(n, dtype=dtype, device="cuda") for _ in range(W)] for _ in range(W)]
        world.run(lambda r, c: c.allgather(dev[r].data_ptr(), [t.data_ptr() for t in outs[r]], n, NATIVE[dtype]))
        torch.cuda.synchronize()
        world.check()
        for r in range(W):
            for j in range(W):
                assert_equal_bits(bits_of(outs[r][j].cpu()), bits_of(ins[j]), f"allgather {dtype} n={n} rank={r} slot={j}")
        for root in (0, W - 1):
            dev = [t.cuda() for t in ins]
            world.run(lambda r, c: c.broadcast(dev[r].data_ptr(), n, NATIVE[dtype], root))
            torch.cuda.synchronize()
            world.check()
            for r in range(W):
                assert_equal_bits(bits_of(dev[r].cpu()), bits_of(ins[root]), f"broadcast {dtype} n={n} root={root} rank={r}")
        src, dst = ins[0].cuda(), torch.zeros(n, dtype=dtype, device="cuda")
        nbytes = n * _esz(dtype)

        def step(r, c):
            if r == 0:
                c.send(src.data_ptr(), nbytes, W - 1)
            elif r == W - 1:
                c.recv(dst.data_ptr(), nbytes, 0)

        world.run(step)
        torch.cuda.synchronize()
        world.check()
        assert_equal_bits(bits_of(dst.cpu()), bits_of(ins[0]), f"send/recv {dtype} n={n}")


# ---- one rank: only the wire rounding and the scale remain (k_local_scale, k_local_scale_tma) -------
# The bulk-copy kernel moves kTmaTileBytes = 16 KiB tiles with kTmaStages = 4 in flight per CTA, on a grid
# of as many CTAs as are resident: 132 SMs x 3 CTAs (each holds 4 x 16 KiB of shared memory, 228 KiB per SM).
# A CTA runs the refill branch from its 5th tile on and waits on both mbarrier parities from its 9th, so
# every CTA needs at least 2 * kTmaStages + 1 = 9 tiles: 396 x 9 x 16 KiB = 55.7 MiB.  80 MiB gives every
# CTA 12 or 13 tiles, and still 9 at four CTAs per SM (528 x 9 x 16 KiB = 74.25 MiB).
TMA_BYTES = 80 << 20
LOCAL_PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.float32, torch.float16),
               (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16)]


@pytest.fixture(scope="module")
def solo():
    from ant_ray_b200.b200_group import PeerMemoryComm, make_config
    from ant_ray_b200.loopback import _MemStore

    comm = PeerMemoryComm(1, 0, "solo-edges", 0, _MemStore(), make_config(staging_bytes=STAGING))
    yield comm
    comm.destroy()


def _scaled_one_rank(comm, bucket, wire, n, scale, offset, inplace, seed):
    (x,) = make_edge_inputs(bucket, n + offset, 1, seed)
    d = x.cuda()
    out = d if inplace else torch.empty(n + offset, dtype=bucket, device="cuda")
    comm.allreduce_scaled(d[offset:].data_ptr(), out[offset:].data_ptr(), n, NATIVE[bucket], NATIVE[wire], scale)
    torch.cuda.synchronize()
    comm.check()
    want = O.allreduce_scaled([x[offset:]], None if wire == bucket else wire, scale)
    assert_same_values(out[offset:], want, f"W=1 {bucket} wire={wire} n={n} offset={offset} inplace={inplace}")


@pytest.mark.parametrize("bucket,wire", LOCAL_PAIRS, ids=str)
def test_one_rank_scaled_edges(solo, bucket, wire):
    for n in (16 // _esz(bucket) + 3, 4099, 100_003):   # all below the 1 MiB bulk-copy threshold
        for offset in (0, 1):
            for inplace in (True, False):
                _scaled_one_rank(solo, bucket, wire, n, 1.0 / 3, offset, inplace, n + offset)


@pytest.mark.parametrize("bucket,wire", LOCAL_PAIRS, ids=str)
def test_one_rank_bulk_copy_edges(solo, bucket, wire):
    """The pipelined bulk-copy (TMA) path in its steady state, with a ragged tail of 20 bytes past the last
    whole 16 KiB tile that the plain kernel finishes."""
    n = (TMA_BYTES + 20) // _esz(bucket)
    for inplace in (True, False):
        _scaled_one_rank(solo, bucket, wire, n, 1.0 / 3, 0, inplace, 11 + inplace)


@pytest.mark.parametrize("opname", list(OPS))
@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_one_rank_ops_edges(solo, dtype, opname):
    """Every op over one rank: AVG of a float type runs k_local_scale (f64 divides by 1), the rest copy."""
    nat, orc = OPS[opname]
    for n in (16 // _esz(dtype) + 3, 4099):
        for offset in (0, 1):
            (x,) = make_edge_inputs(dtype, n + offset, 1, n)
            d = x.cuda()
            out = torch.empty_like(d)
            solo.allreduce(d[offset:].data_ptr(), out[offset:].data_ptr(), n, NATIVE[dtype], nat)
            torch.cuda.synchronize()
            solo.check()
            assert_same_values(out[offset:], O.allreduce([x[offset:]], orc), f"W=1 {dtype} {opname} n={n} offset={offset}")
