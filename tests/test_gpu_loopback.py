"""GPU parity tests that need ONE GPU: W communicators in one process (ant_ray_b200.loopback).

Every op goes through the C-ABI (ctypes -> libb200coll.so) and is compared with the CPU oracle on
the same seeded inputs: bit-exact for every dtype, floats included, because the peer-memory kernels
fold ranks in the oracle's order (0..W-1, fp32 accumulate for f16/bf16).
Sizes cover empty, tiny, ragged (not a multiple of the 16-byte vector or of W), multi-block and
multi-piece (larger than the staging half) messages.
"""
import pytest
import torch

from gpu_common import FLOAT_DTYPES, INT_DTYPES, NATIVE, assert_equal_bits, make_input

from ant_ray_b200 import _native as N
from oracle import oracle as O

pytestmark = pytest.mark.gpu

OPS = {"sum": (N.SUM, O.SUM), "prod": (N.PROD, O.PROD), "max": (N.MAX, O.MAX), "min": (N.MIN, O.MIN), "avg": (N.AVG, O.AVG)}
SIZES = [1, 3, 10, 257, 4096 + 5, 100_003]


@pytest.fixture(scope="module", params=[2, 4, 8])
def world(request):
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(request.param, device=0, key=f"lb{request.param}", staging_bytes=1 << 20, timeout_ms=20000)
    yield w
    w.destroy()


def _run_allreduce(world, dtype, n, opname, algo, inplace=True):
    W = world.world_size
    nat, orc = OPS[opname]
    ins = [make_input(dtype, n, r, opname) for r in range(W)]
    dev_in = [t.cuda() for t in ins]
    dev_out = dev_in if inplace else [torch.empty_like(t) for t in dev_in]
    world.run(lambda r, c: c.allreduce(dev_in[r].data_ptr(), dev_out[r].data_ptr(), n, NATIVE[dtype], nat, algo))
    torch.cuda.synchronize()
    world.check()
    want = O.allreduce(ins, orc)
    for r in range(W):
        assert_equal_bits(dev_out[r], want, f"allreduce {dtype} n={n} op={opname} algo={algo} rank={r}")
        if not inplace:
            assert_equal_bits(dev_in[r], ins[r], "input must be untouched")


@pytest.mark.parametrize("algo", [N.ALGO_ONESHOT, N.ALGO_TWOSHOT])
@pytest.mark.parametrize("dtype", INT_DTYPES + FLOAT_DTYPES)
def test_allreduce_sum_all_dtypes(world, dtype, algo):
    for n in SIZES:
        _run_allreduce(world, dtype, n, "sum", algo)


@pytest.mark.parametrize("algo", [N.ALGO_ONESHOT, N.ALGO_TWOSHOT])
@pytest.mark.parametrize("opname", ["prod", "max", "min", "avg"])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64, torch.uint8, torch.float32, torch.bfloat16, torch.float16, torch.float64,
                                   torch.uint32, torch.uint64])
def test_allreduce_ops(world, dtype, opname, algo):
    for n in (7, 5000):
        _run_allreduce(world, dtype, n, opname, algo)


LL_SIZES = [1, 3, 10, 257, 4000, 8190]   # 8190 x 8-byte elements = 65,520 bytes: just under the 64 KiB LL capacity


@pytest.mark.parametrize("dtype", INT_DTYPES + FLOAT_DTYPES)
def test_allreduce_ll_all_dtypes(world, dtype):
    """LL path (packed data+flag stores, no flag round): same rank-order fold, so bit-exact too."""
    for n in LL_SIZES:
        _run_allreduce(world, dtype, n, "sum", N.ALGO_LL)
    _run_allreduce(world, dtype, 100, "sum", N.ALGO_LL, inplace=False)


@pytest.mark.parametrize("opname", ["prod", "max", "min", "avg"])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64, torch.uint8, torch.float32, torch.bfloat16, torch.float64,
                                   torch.uint32, torch.uint64])
def test_allreduce_ll_ops(world, dtype, opname):
    for n in (7, 3001):
        _run_allreduce(world, dtype, n, opname, N.ALGO_LL)


def test_allreduce_ll_limits_and_auto(world):
    """AUTO picks LL up to ll_max_bytes; asking for LL beyond the region's capacity is refused, not truncated."""
    cap = int(world.comms[0].config.ll_max_bytes) // 4                    # fp32 elements the LL region holds (64 KiB)
    _run_allreduce(world, torch.float32, cap, "sum", N.ALGO_AUTO)        # exactly ll_max_bytes -> LL
    _run_allreduce(world, torch.float32, cap + 1, "sum", N.ALGO_AUTO)    # one element more -> one-shot
    x = torch.ones(cap + 1, device="cuda")
    with pytest.raises(N.B200CollError) as ei:
        world.comms[0].allreduce(x.data_ptr(), x.data_ptr(), cap + 1, N.FLOAT32, N.SUM, N.ALGO_LL)
    assert ei.value.status == N.EUNSUPPORTED
    # the refused call must not have consumed a sequence number: the next op still lines up with the peers
    _run_allreduce(world, torch.int32, 100, "sum", N.ALGO_LL)
    with pytest.raises(N.B200CollError):
        world.comms[0].allreduce_scaled(x.data_ptr(), x.data_ptr(), 100, N.FLOAT32, N.BFLOAT16, 0.5, N.ALGO_LL)
    _run_allreduce(world, torch.int32, 100, "sum", N.ALGO_TWOSHOT)


def test_allreduce_ll_unaligned_and_scaled(world):
    W, n = world.world_size, 1001
    ins = [make_input(torch.float32, n + 1, r) for r in range(W)]
    cur = [t.cuda() for t in ins]
    world.run(lambda r, c: c.allreduce(cur[r][1:].data_ptr(), cur[r][1:].data_ptr(), n, N.FLOAT32, N.SUM, N.ALGO_LL))
    torch.cuda.synchronize()
    world.check()
    want = O.allreduce([t[1:] for t in ins])
    for r in range(W):
        assert_equal_bits(cur[r][1:], want, "LL unaligned")
        assert cur[r][0].item() == ins[r][0].item()
    # fused mean with an fp32 wire takes LL under AUTO for small buckets (the RLlib-sized case)
    dev = [t[:n].contiguous().cuda() for t in ins]
    world.run(lambda r, c: c.allreduce_scaled(dev[r].data_ptr(), dev[r].data_ptr(), n, N.FLOAT32, N.FLOAT32, 1.0 / W, N.ALGO_AUTO))
    torch.cuda.synchronize()
    world.check()
    want = O.allreduce_scaled([t[:n] for t in ins], None, 1.0 / W)
    for r in range(W):
        assert_equal_bits(dev[r], want, "LL fused mean fp32 wire")


def test_allreduce_out_of_place_and_auto(world):
    for n in (5, 70_000):
        _run_allreduce(world, torch.float32, n, "sum", N.ALGO_AUTO, inplace=False)


def test_allreduce_multi_piece(world):
    # staging half is 1 MiB here: 3 MiB of fp32 needs several pieces under every algorithm
    for algo in (N.ALGO_ONESHOT, N.ALGO_TWOSHOT, N.ALGO_AUTO):
        _run_allreduce(world, torch.float32, 3 * (1 << 18) + 11, "sum", algo)


def test_allreduce_unaligned_views(world):
    """Tensor views that start 4 bytes into an allocation take the scalar path."""
    W, n = world.world_size, 1001
    ins = [make_input(torch.float32, n + 1, r) for r in range(W)]
    dev = [t.cuda() for t in ins]
    for algo in (N.ALGO_ONESHOT, N.ALGO_TWOSHOT):
        cur = [d.clone() for d in dev]
        world.run(lambda r, c: c.allreduce(cur[r][1:].data_ptr(), cur[r][1:].data_ptr(), n, N.FLOAT32, N.SUM, algo))
        torch.cuda.synchronize()
        want = O.allreduce([t[1:] for t in ins])
        for r in range(W):
            assert_equal_bits(cur[r][1:], want, f"unaligned algo={algo}")
            assert cur[r][0].item() == ins[r][0].item()


def test_allreduce_empty(world):
    x = [torch.empty(0, device="cuda") for _ in range(world.world_size)]
    world.run(lambda r, c: c.allreduce(x[r].data_ptr(), x[r].data_ptr(), 0, N.FLOAT32, N.SUM))
    torch.cuda.synchronize()
    world.check()


@pytest.mark.parametrize("wire", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("algo", [N.ALGO_ONESHOT, N.ALGO_TWOSHOT])
def test_fused_gradient_mean(world, wire, algo):
    """K13: fp32 bucket, 16-bit wire, fp32 accumulate, x 1/W, all in one launch."""
    W = world.world_size
    for n in (9, 33_333):
        ins = [make_input(torch.float32, n, r) for r in range(W)]
        dev = [t.cuda() for t in ins]
        world.run(lambda r, c: c.allreduce_scaled(dev[r].data_ptr(), dev[r].data_ptr(), n, N.FLOAT32, NATIVE[wire], 1.0 / W, algo))
        torch.cuda.synchronize()
        world.check()
        want = O.allreduce_scaled(ins, None if wire == torch.float32 else wire, 1.0 / W)
        for r in range(W):
            assert_equal_bits(dev[r], want, f"fused mean wire={wire} n={n} rank={r}")
        # sanity against plain fp32 math: the mean, to the wire's precision
        ref = torch.stack(ins).mean(0)
        tol = {torch.float32: 1e-5, torch.bfloat16: 2e-2, torch.float16: 2e-3}[wire]
        assert torch.allclose(dev[0].cpu(), ref, rtol=tol, atol=tol)


@pytest.mark.parametrize("dtype", [torch.int32, torch.float32, torch.bfloat16, torch.uint8, torch.int8, torch.int64, torch.uint32,
                                   torch.uint64, torch.float16, torch.float64])
def test_reducescatter(world, dtype):
    W = world.world_size
    for opname, (nat, orc) in OPS.items():
        for n in (6, 20_001):
            lists = [[make_input(dtype, n, r * 16 + j, opname) for j in range(W)] for r in range(W)]
            dev = [[t.cuda() for t in row] for row in lists]
            outs = [torch.empty(n, dtype=dtype, device="cuda") for _ in range(W)]
            world.run(lambda r, c: c.reducescatter([t.data_ptr() for t in dev[r]], outs[r].data_ptr(), n, NATIVE[dtype], nat))
            torch.cuda.synchronize()
            world.check()
            want = O.reducescatter(lists, orc)
            for r in range(W):
                assert_equal_bits(outs[r], want[r], f"reducescatter {dtype} {opname} n={n} rank={r}")
                for j in range(W):
                    assert_equal_bits(dev[r][j], lists[r][j], "inputs must be untouched")


@pytest.mark.parametrize("dtype", [torch.int64, torch.float16, torch.uint8])
def test_allgather(world, dtype):
    W = world.world_size
    for n in (1, 13, 50_001):
        ins = [make_input(dtype, n, r) for r in range(W)]
        dev = [t.cuda() for t in ins]
        outs = [[torch.zeros(n, dtype=dtype, device="cuda") for _ in range(W)] for _ in range(W)]
        world.run(lambda r, c: c.allgather(dev[r].data_ptr(), [t.data_ptr() for t in outs[r]], n, NATIVE[dtype]))
        torch.cuda.synchronize()
        world.check()
        for r in range(W):
            for j in range(W):
                assert_equal_bits(outs[r][j], ins[j], f"allgather {dtype} n={n} rank={r} slot={j}")


def test_broadcast_and_reduce(world):
    W = world.world_size
    for root in (0, W - 1):
        for n in (3, 40_000):
            ins = [make_input(torch.float32, n, r) for r in range(W)]
            dev = [t.cuda() for t in ins]
            world.run(lambda r, c: c.broadcast(dev[r].data_ptr(), n, N.FLOAT32, root))
            torch.cuda.synchronize()
            for r in range(W):
                assert_equal_bits(dev[r], ins[root], f"broadcast root={root} rank={r}")
            for dtype in INT_DTYPES + FLOAT_DTYPES:
                for opname, (nat, orc) in OPS.items():
                    ins = [make_input(dtype, n, r, opname) for r in range(W)]
                    dev = [t.cuda() for t in ins]
                    world.run(lambda r, c: c.reduce(dev[r].data_ptr(), dev[r].data_ptr(), n, NATIVE[dtype], nat, root))
                    torch.cuda.synchronize()
                    world.check()
                    want = O.reduce(ins, orc)
                    for r in range(W):
                        assert_equal_bits(dev[r], want if r == root else ins[r], f"reduce {dtype} {opname} n={n} root={root} rank={r}")


def test_send_recv(world):
    W = world.world_size
    for nbytes in (1, 100_000, (32 << 10) * 1100 + 17):  # the last one wraps the 1024-cell ring
        src = torch.randint(0, 255, (nbytes,), dtype=torch.uint8, generator=torch.Generator().manual_seed(7))
        d_src = src.cuda()
        d_dst = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")

        def step(r, c):
            if r == 0:
                c.send(d_src.data_ptr(), nbytes, 1)
            elif r == 1:
                c.recv(d_dst.data_ptr(), nbytes, 0)

        world.run(step)
        torch.cuda.synchronize()
        world.check()
        assert_equal_bits(d_dst, src, f"send/recv {nbytes} bytes")


def test_barrier_and_back_to_back(world):
    """200 small collectives in a row exercise the double-buffered staging, the LL region halves and the
    flag epochs (LL skips the prologue wait, so it is interleaved with the staged algorithms on purpose)."""
    W, n = world.world_size, 300
    ins = [make_input(torch.int32, n, r) for r in range(W)]
    dev = [t.cuda() for t in ins]
    acc = [t.clone() for t in ins]
    cycle = [N.ALGO_TWOSHOT, N.ALGO_LL, N.ALGO_LL, N.ALGO_ONESHOT, N.ALGO_LL]
    for it in range(200):
        world.run(lambda r, c: c.allreduce(dev[r].data_ptr(), dev[r].data_ptr(), n, N.INT32, N.SUM, cycle[it % len(cycle)]))
        s = O.allreduce(acc)
        acc = [s.clone() for _ in range(W)]
        if it % 50 == 0:
            world.run(lambda r, c: c.barrier())
    torch.cuda.synchronize()
    world.check()
    for r in range(W):
        assert_equal_bits(dev[r], acc[r], "after 200 allreduces")


@pytest.mark.parametrize("W", [2, 4])
def test_block_cyclic_granules(W):
    """Few blocks + the smallest granule: every block loops over several granules of every chunk (the
    large-message layout), with ragged tails, for every kernel that uses it."""
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(W, device=0, key=f"lb-gran{W}", staging_bytes=4 << 20, max_blocks=3, granule_bytes=16384,
                      bcast_rounds_min_bytes=4 << 20, timeout_ms=20000)
    try:
        n = 300_007
        for dtype, algo in ((torch.float32, N.ALGO_TWOSHOT), (torch.int32, N.ALGO_ONESHOT), (torch.bfloat16, N.ALGO_TWOSHOT)):
            _run_allreduce(w, dtype, n, "sum", algo)
        ins = [make_input(torch.float32, n, r) for r in range(W)]
        dev = [t.cuda() for t in ins]
        w.run(lambda r, c: c.allreduce_scaled(dev[r].data_ptr(), dev[r].data_ptr(), n, N.FLOAT32, N.BFLOAT16, 1.0 / W, N.ALGO_TWOSHOT))
        torch.cuda.synchronize()
        w.check()
        want = O.allreduce_scaled(ins, torch.bfloat16, 1.0 / W)
        for r in range(W):
            assert_equal_bits(dev[r], want, "granules: fused mean")
        m = 120_001
        lists = [[make_input(torch.int32, m, r * 16 + j) for j in range(W)] for r in range(W)]
        devl = [[t.cuda() for t in row] for row in lists]
        outs = [torch.empty(m, dtype=torch.int32, device="cuda") for _ in range(W)]
        w.run(lambda r, c: c.reducescatter([t.data_ptr() for t in devl[r]], outs[r].data_ptr(), m, N.INT32, N.SUM))
        gouts = [[torch.zeros(m, dtype=torch.int32, device="cuda") for _ in range(W)] for _ in range(W)]
        w.run(lambda r, c: c.allgather(devl[r][0].data_ptr(), [t.data_ptr() for t in gouts[r]], m, N.INT32))
        torch.cuda.synchronize()
        w.check()
        want = O.reducescatter(lists)
        for r in range(W):
            assert_equal_bits(outs[r], want[r], "granules: reducescatter")
            for j in range(W):
                assert_equal_bits(gouts[r][j], lists[j][0], "granules: allgather")
        # past one staging half: the first 4 MiB piece takes the pipelined unicast push (bcast_rounds_min_bytes),
        # the ragged rest the plain kernel
        big = [make_input(torch.float32, 1_300_007, r) for r in range(W)]
        for root in (0, W - 1):
            for src, what in ((ins, "granules: broadcast"), (big, "granules: pipelined broadcast")):
                dev = [t.cuda() for t in src]
                w.run(lambda r, c: c.broadcast(dev[r].data_ptr(), dev[r].numel(), N.FLOAT32, root))
                torch.cuda.synchronize()
                w.check()
                for r in range(W):
                    assert_equal_bits(dev[r], src[root], what)
            dev = [t.cuda() for t in ins]
            w.run(lambda r, c: c.reduce(dev[r].data_ptr(), dev[r].data_ptr(), n, N.FLOAT32, N.SUM, root))
            torch.cuda.synchronize()
            w.check()
            for r in range(W):
                assert_equal_bits(dev[r], O.reduce(ins) if r == root else ins[r], "granules: reduce")
    finally:
        w.destroy()


def test_ll_mismatch_is_detected_not_hung():
    """LL has no flag round to compare arguments on: a peer that entered the op with a different count is
    diagnosed from the poll loop (signature slot), not by waiting out the timeout."""
    import time

    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(2, device=0, key="lb-ll-mismatch", staging_bytes=1 << 20, timeout_ms=30000)
    try:
        x = [torch.ones(64, device="cuda"), torch.ones(128, device="cuda")]
        t0 = time.time()
        w.run(lambda r, c: c.allreduce(x[r].data_ptr(), x[r].data_ptr(), x[r].numel(), N.FLOAT32, N.SUM, N.ALGO_LL))
        torch.cuda.synchronize()
        assert time.time() - t0 < 10, "mismatch must not wait for the 30 s device timeout"
        with pytest.raises(N.B200CollError) as ei:
            w.check()
        assert ei.value.status in (N.EMISMATCH, N.EABORTED)
    finally:
        w.destroy()


def test_mismatch_is_detected_not_hung():
    """Ranks that disagree on the element count must surface an error instead of hanging or reading
    out of bounds (reference expectation: test_torch_tensor_dag.py:1544-1588)."""
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(2, device=0, key="lb-mismatch", staging_bytes=1 << 20, timeout_ms=3000)
    try:
        x = [torch.ones(64, device="cuda"), torch.ones(128, device="cuda")]
        w.run(lambda r, c: c.allreduce(x[r].data_ptr(), x[r].data_ptr(), x[r].numel(), N.FLOAT32, N.SUM, N.ALGO_ONESHOT))
        torch.cuda.synchronize()
        with pytest.raises(N.B200CollError) as ei:
            w.check()
        assert ei.value.status in (N.EMISMATCH, N.ETIMEOUT, N.EABORTED)
        with pytest.raises(RuntimeError):  # the communicator stays poisoned
            w.comms[0].allreduce(x[0].data_ptr(), x[0].data_ptr(), 64, N.FLOAT32, N.SUM)
    finally:
        w.destroy()


def test_abort_unblocks_a_waiting_kernel():
    """destroy()/abort must release a kernel that waits for a peer that never comes
    (reference: _NcclGroup.destroy -> comm.abort(), nccl_group.py:347-365)."""
    import time

    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(2, device=0, key="lb-abort", staging_bytes=1 << 20, timeout_ms=60000)
    try:
        x = torch.ones(64, device="cuda")
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            w.comms[0].allreduce(x.data_ptr(), x.data_ptr(), 64, N.FLOAT32, N.SUM)  # rank 1 never joins
        time.sleep(0.2)
        assert not s.query()
        t0 = time.time()
        w.comms[0].abort()
        s.synchronize()
        assert time.time() - t0 < 5
        with pytest.raises(N.B200CollError) as ei:
            w.comms[0].check()
        assert ei.value.status == N.EABORTED
    finally:
        w.destroy()


def test_world_size_one_scale_and_wire_rounding():
    """W = 1 (the N=1 bench / single-worker TorchTrainer): no peers, only the wire rounding and the
    scale remain (k_local_scale).  Bit-exact against the oracle, aligned and unaligned, in and out of place."""
    from ant_ray_b200.b200_group import PeerMemoryComm, make_config
    from ant_ray_b200.loopback import _MemStore

    comm = PeerMemoryComm(1, 0, "solo", 0, _MemStore(), make_config(staging_bytes=1 << 20))
    try:
        for n in (1, 7, 4099, 1_000_003):
            x = make_input(torch.float32, n + 1, 0)
            for wire, owire in ((N.BFLOAT16, torch.bfloat16), (N.FLOAT16, torch.float16), (N.FLOAT32, None)):
                for off in (0, 1):  # off = 1: a view 4 bytes into the allocation -> scalar path
                    src = x[off:off + n].clone() if off == 0 else x[off:off + n]
                    d = x.cuda()[off:off + n]
                    out = torch.empty(n + 1, device="cuda")[off:off + n]
                    comm.allreduce_scaled(d.data_ptr(), out.data_ptr(), n, N.FLOAT32, wire, 0.25)
                    torch.cuda.synchronize()
                    want = O.allreduce_scaled([src], owire, 0.25)
                    assert_equal_bits(out, want, f"W=1 scaled n={n} wire={wire} off={off}")
                    comm.allreduce_scaled(d.data_ptr(), d.data_ptr(), n, N.FLOAT32, wire, 0.25)  # in place
                    torch.cuda.synchronize()
                    assert_equal_bits(d, want, "in place")
        h = make_input(torch.bfloat16, 5001, 3)
        d = h.cuda()
        comm.allreduce_scaled(d.data_ptr(), d.data_ptr(), 5001, N.BFLOAT16, N.BFLOAT16, 0.5)
        torch.cuda.synchronize()
        assert_equal_bits(d, O.allreduce_scaled([h], None, 0.5), "bf16 bucket")
        # plain ops over one rank: identity / copy
        a = make_input(torch.int32, 1000, 1).cuda()
        b = torch.zeros_like(a)
        comm.allreduce(a.data_ptr(), b.data_ptr(), 1000, N.INT32, N.SUM)
        comm.allreduce(a.data_ptr(), a.data_ptr(), 1000, N.INT32, N.AVG)
        comm.broadcast(a.data_ptr(), 1000, N.INT32, 0)
        comm.barrier()
        torch.cuda.synchronize()
        assert_equal_bits(b, a, "W=1 allreduce is a copy")
        comm.check()
    finally:
        comm.destroy()


def test_full_size_properties_loopback():
    """256 MiB per rank (many staging pieces) checked through size-independent properties, as in
    test_gpu_multiproc.py::test_full_size_properties, but runnable on a single GPU."""
    from ant_ray_b200.loopback import LoopbackWorld

    W, n = 2, 1 << 26
    w = LoopbackWorld(W, device=0, key="lb-big", staging_bytes=32 << 20, timeout_ms=30000)
    try:
        xs = [torch.randint(-2**31, 2**31 - 1, (n,), dtype=torch.int32, device="cuda",
                            generator=torch.Generator(device="cuda").manual_seed(99 + r)) for r in range(W)]
        locals_ = [int(x.sum(dtype=torch.int64).item()) for x in xs]
        w.run(lambda r, c: c.allreduce(xs[r].data_ptr(), xs[r].data_ptr(), n, N.INT32, N.SUM))
        torch.cuda.synchronize()
        w.check()
        total = int(xs[0].sum(dtype=torch.int64).item())
        assert (sum(locals_) - total) % (1 << 32) == 0, "checksum of checksums mismatch"
        assert torch.equal(xs[0], xs[1]), "ranks must hold identical bits"
        ys = [x.clone() for x in xs]
        w.run(lambda r, c: c.allreduce(ys[r].data_ptr(), ys[r].data_ptr(), n, N.INT32, N.MAX))
        torch.cuda.synchronize()
        assert torch.equal(ys[0], xs[0]) and torch.equal(ys[1], xs[0]), "MAX over identical buffers must be idempotent"
        del ys
        fs = [torch.ones(n, device="cuda") for _ in range(W)]
        w.run(lambda r, c: c.allreduce(fs[r].data_ptr(), fs[r].data_ptr(), n, N.FLOAT32, N.SUM))
        torch.cuda.synchronize()
        w.check()
        assert all(bool((f == float(W)).all().item()) for f in fs)
    finally:
        w.destroy()


def test_symmetric_pool_allocator_mechanics():
    """torch.cuda.MemPool over a communicator's symmetric region (the zero-copy path itself needs the
    multicast object, i.e. >= 2 GPUs: tests/test_gpu_multiproc.py): segments come from the region, freed
    segments are reused first-fit, exhaustion is an ordinary CUDA OOM, and collectives on pool tensors work."""
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(2, device=0, key="lb-pool", staging_bytes=4 << 20, symmetric_bytes=64 << 20, timeout_ms=20000)
    try:
        c0 = w.comms[0]
        base = int(c0.lib.b200c_comm_symmetric_base(c0.handle))
        size = int(c0.lib.b200c_comm_symmetric_bytes(c0.handle))
        pool = c0.symmetric_pool()
        with torch.cuda.use_mem_pool(pool):
            a = torch.full((1 << 20,), 2.0, device="cuda")          # 4 MiB
            b = torch.full((3 << 20,), 3.0, device="cuda")          # 12 MiB
        for t in (a, b):
            assert base <= t.data_ptr() and t.data_ptr() + t.numel() * 4 <= base + size
        assert a.data_ptr() != b.data_ptr()
        off_a = a.data_ptr() - base
        # a plain tensor on the other rank, the pool tensor on this one: the staged path handles the mix
        other = torch.full((1 << 20,), 5.0, device="cuda")
        w.run(lambda r, c: c.allreduce((a if r == 0 else other).data_ptr(), (a if r == 0 else other).data_ptr(), 1 << 20, N.FLOAT32, N.SUM))
        torch.cuda.synchronize()
        w.check()
        assert bool((a == 7).all()) and bool((other == 7).all())
        with pytest.raises(torch.OutOfMemoryError):
            with torch.cuda.use_mem_pool(pool):
                torch.empty(size // 4 + 1024, device="cuda")
        del a
        torch.cuda.synchronize()
        # the raw entry points: first fit reuses the lowest free offset
        p1 = c0.lib.b200c_pool_malloc(1 << 20, 0, None)
        assert p1 is not None and base <= p1 < base + size
        c0.lib.b200c_pool_free(p1, 1 << 20, 0, None)
        p2 = c0.lib.b200c_pool_malloc(1 << 20, 0, None)
        assert p2 == p1
        c0.lib.b200c_pool_free(p2, 1 << 20, 0, None)
        assert off_a % (2 << 20) == 0
    finally:
        w.destroy()
