"""The FSDP collectives on ONE GPU: `reducescatter_scaled` and the FSDP2 / FSDP1 adapters of ant_ray_b200.fsdp,
compared with the CPU oracle.

Rank r's output of the scaled reducescatter is defined as
    oracle.allreduce_scaled([x_s[r*n:(r+1)*n] for every rank s], wire, scale)
(every contribution rounded to the wire type, fp32 fold in rank order, one scale, rounded to the wire type, stored
as the buffer type) and must match it bit for bit, NaN matching NaN.  Loopback worlds of 2, 4 and 8 ranks run the
kernels compiled for that world size, 3 ranks the kernel that takes the world size at run time.  A 1 MiB staging
half makes the multi-piece sizes cheap.
"""
import pytest
import torch
import torch.distributed as dist

from gpu_common import NATIVE, assert_same_values, make_edge_inputs

from ant_ray_b200 import _native as N
from ant_ray_b200 import ddp_hook, fsdp
from oracle import oracle as O

pytestmark = pytest.mark.gpu

STAGING = 1 << 20
PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.float32, torch.float16),
         (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float16)]
WIRE_NAME = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}


def _esz(dtype):
    return torch.empty((), dtype=dtype).element_size()


@pytest.fixture(scope="module", params=[2, 3, 4, 8])
def world(request):
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(request.param, device=0, key=f"fsdp{request.param}", staging_bytes=STAGING, timeout_ms=20000)
    yield w
    w.destroy()


def _want(ins, r, n, wire, bucket, scale, offset=0):
    return O.allreduce_scaled([x[offset + r * n:offset + (r + 1) * n] for x in ins], None if wire == bucket else wire, scale)


def _run_scaled(world, bucket, wire, n, seed, offset=0, inplace=False, edges=True, scale=None):
    W = world.world_size
    scale = 1.0 / W if scale is None else scale
    esz = _esz(bucket)
    if edges:
        ins = make_edge_inputs(bucket, offset + W * n, W, seed)
    else:
        g = torch.Generator().manual_seed(seed)
        ins = [torch.randn(offset + W * n, generator=g).to(bucket) for _ in range(W)]
    dev = [t.cuda() for t in ins]
    if inplace:
        outs = [dev[r][offset + r * n:offset + (r + 1) * n] for r in range(W)]
    else:
        outs = [torch.empty(offset + n, dtype=bucket, device="cuda")[offset:] for _ in range(W)]

    def op(r, c):
        base = dev[r].data_ptr() + offset * esz
        c.reducescatter_scaled([base + j * n * esz for j in range(W)], outs[r].data_ptr(), n, NATIVE[bucket], NATIVE[wire], scale)

    world.run(op)
    torch.cuda.synchronize()
    world.check()
    for r in range(W):
        assert_same_values(outs[r].cpu(), _want(ins, r, n, wire, bucket, scale, offset),
                           f"W={W} {bucket} wire={wire} n={n} offset={offset} inplace={inplace} rank={r}")


@pytest.mark.parametrize("bucket,wire", PAIRS, ids=str)
def test_reducescatter_scaled_matches_the_oracle(world, bucket, wire):
    W = world.world_size
    cap = STAGING // W // _esz(wire)   # one rank's slot of the staging half, in wire elements
    for k, n in enumerate((16 // _esz(bucket) + 3, 4099, cap + cap // 2 + 3)):   # a tail, odd, several pieces
        for inplace in (False, True):
            _run_scaled(world, bucket, wire, n, seed=100 * W + 10 * k + inplace, inplace=inplace)
    # unaligned: every pointer one element past a 16-byte boundary (the scalar path of every tile)
    _run_scaled(world, bucket, wire, 4099, seed=7, offset=1)
    _run_scaled(world, bucket, wire, 4099, seed=8, offset=1, inplace=True)


def test_reducescatter_scaled_with_another_scale(world):
    _run_scaled(world, torch.float32, torch.bfloat16, 10_007, seed=3, edges=False, scale=0.37)


def test_unsupported_dtypes_are_refused(world):
    c = world.comms[0]
    ptrs = [1] * world.world_size
    with pytest.raises(N.B200CollError) as ei:
        c.reducescatter_scaled(ptrs, 1, 16, N.INT32, N.INT32, 1.0)
    assert ei.value.status == N.EUNSUPPORTED
    with pytest.raises(N.B200CollError) as ei:
        c.reducescatter_scaled(ptrs, 1, 16, N.BFLOAT16, N.FLOAT16, 1.0)
    assert ei.value.status == N.EUNSUPPORTED
    world.check()


class _StubGroup:
    """What FSDP hands the collectives: only size() and rank() are used."""

    def __init__(self, W, r):
        self.W, self.r = W, r

    def size(self):
        return self.W

    def rank(self):
        return self.r


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.uint8])
def test_fsdp2_all_gather_in_place(world, dtype):
    """FSDP2's layout: the input is the rank's own slice of the output, already filled by the copy-in."""
    W = world.world_size
    n = 12_345
    g = torch.Generator().manual_seed(W)
    shards = [torch.randint(0, 255, (n,), generator=g).to(dtype) for _ in range(W)]
    ags = [fsdp.B200AllGather(c) for c in world.comms]
    outs = []
    for r in range(W):
        out = ags[r].allocate((W * n,), dtype=dtype, device=torch.device("cuda", 0))
        out.fill_(0)
        out[r * n:(r + 1) * n].copy_(shards[r])
        outs.append(out)
    res = []
    world.run(lambda r, c: res.append(ags[r](outs[r], outs[r][r * n:(r + 1) * n], _StubGroup(W, r))))
    torch.cuda.synchronize()
    world.check()
    assert res == [None] * W
    want = torch.cat(shards)
    for r in range(W):
        assert torch.equal(outs[r].cpu(), want), (dtype, r)


@pytest.mark.parametrize("dtype,wire,op", [(torch.float32, "fp32", "avg"), (torch.float32, "bf16", "avg"),
                                           (torch.bfloat16, "fp32", "avg"), (torch.float16, "fp32", "sum")], ids=str)
def test_fsdp2_reduce_scatter(world, dtype, wire, op):
    """FSDP2's layout: a padded W*n input, a separate n-element output; AVG for fp32 / bf16, SUM for fp16."""
    W = world.world_size
    n = 5_003
    ins = make_edge_inputs(dtype, W * n, W, 31 + W)
    dev = [t.cuda() for t in ins]
    rss = [fsdp.B200ReduceScatter(ddp_hook.B200GradState(c, wire=wire)) for c in world.comms]
    outs = [rs.allocate((n,), dtype=dtype, device=torch.device("cuda", 0)) for rs in rss]
    rop = dist.ReduceOp.AVG if op == "avg" else dist.ReduceOp.SUM
    world.run(lambda r, c: rss[r](outs[r], dev[r], _StubGroup(W, r), rop))
    torch.cuda.synchronize()
    world.check()
    wdt = torch.bfloat16 if (wire == "bf16" and dtype == torch.float32) else dtype
    scale = 1.0 / W if op == "avg" else 1.0
    for r in range(W):
        assert_same_values(outs[r].cpu(), _want(ins, r, n, wdt, dtype, scale), f"W={W} {dtype} wire={wire} {op} rank={r}")
    assert all(rs.state.launches == 1 for rs in rss)


def test_fsdp2_refuses_other_ops_and_groups(world):
    W = world.world_size
    rs = fsdp.B200ReduceScatter(ddp_hook.B200GradState(world.comms[0]))
    x = torch.zeros(W * 16, device="cuda")
    with pytest.raises(ValueError, match="set_gradient_divide_factor"):
        rs(x[:16], x, _StubGroup(W, 0), dist._make_nccl_premul_sum(0.5))
    with pytest.raises(ValueError):
        rs(x[:16], x, _StubGroup(W, 1), dist.ReduceOp.AVG)
    with pytest.raises(ValueError):
        fsdp.B200AllGather(world.comms[0])(x, x[:16], _StubGroup(W + 1, 0))
    world.check()


@pytest.mark.parametrize("wire", ["fp32", "bf16"])
def test_fsdp1_hooks(world, wire):
    """FSDP1: the sharded hook gets the padded flat gradient and a pre-sized shard, NO_SHARD the flat gradient."""
    W = world.world_size
    n = 7_001
    ins = make_edge_inputs(torch.float32, W * n, W, 57 + W)
    wdt = torch.bfloat16 if wire == "bf16" else torch.float32
    states = [ddp_hook.B200GradState(c, wire=wire) for c in world.comms]
    dev = [t.cuda() for t in ins]
    outs = [torch.empty(n, device="cuda") for _ in range(W)]
    world.run(lambda r, c: fsdp.b200_reduce_scatter_hook(states[r], dev[r], outs[r]))
    torch.cuda.synchronize()
    world.check()
    for r in range(W):
        assert_same_values(outs[r].cpu(), _want(ins, r, n, wdt, torch.float32, 1.0 / W), f"sharded hook W={W} wire={wire} rank={r}")
    world.run(lambda r, c: fsdp.b200_allreduce_hook_no_shard(states[r], dev[r]))
    torch.cuda.synchronize()
    world.check()
    want = O.allreduce_scaled(ins, None if wdt == torch.float32 else wdt, 1.0 / W)
    for r in range(W):
        assert_same_values(dev[r].cpu(), want, f"NO_SHARD hook W={W} wire={wire} rank={r}")


def test_scaled_and_plain_reducescatter_are_a_mismatch():
    """The wire is part of the op signature: a plain reducescatter on one rank and a scaled one on the other is
    reported, not folded into wrong data silently."""
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(2, device=0, key="fsdp-mismatch", staging_bytes=1 << 20, timeout_ms=3000)
    try:
        n = 256
        x = [torch.ones(2 * n, device="cuda") for _ in range(2)]
        out = [torch.empty(n, device="cuda") for _ in range(2)]

        def op(r, c):
            ptrs = [x[r].data_ptr(), x[r].data_ptr() + 4 * n]
            if r == 0:
                c.reducescatter(ptrs, out[r].data_ptr(), n, N.FLOAT32, N.SUM)
            else:
                c.reducescatter_scaled(ptrs, out[r].data_ptr(), n, N.FLOAT32, N.FLOAT32, 1.0)

        w.run(op)
        torch.cuda.synchronize()
        with pytest.raises(N.B200CollError) as ei:
            w.check()
        assert ei.value.status in (N.EMISMATCH, N.EABORTED)
    finally:
        w.destroy()


def test_one_rank_is_the_wire_rounding_and_the_scale():
    from ant_ray_b200.b200_group import PeerMemoryComm, make_config
    from ant_ray_b200.loopback import _MemStore

    comm = PeerMemoryComm(1, 0, "fsdp-solo", 0, _MemStore(), make_config(staging_bytes=1 << 20))
    try:
        for bucket, wire in PAIRS:
            (x,) = make_edge_inputs(bucket, 4099, 1, 5)
            d = x.cuda()
            out = torch.empty_like(d)
            comm.reducescatter_scaled([d.data_ptr()], out.data_ptr(), 4099, NATIVE[bucket], NATIVE[wire], 0.25)
            torch.cuda.synchronize()
            comm.check()
            assert_same_values(out.cpu(), O.allreduce_scaled([x], None if wire == bucket else wire, 0.25), f"W=1 {bucket} {wire}")
    finally:
        comm.destroy()
