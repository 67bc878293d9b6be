"""Sync batch-norm sites (fused_norm.FusedSyncBatchNorm, b200c_bn_sync_*) in loopback worlds, bit for bit.

W ranks on one GPU, one stream each, each with its own replica of the batch norm.  The reference is torch's own
SyncBatchNorm arithmetic per rank: batch_norm_stats, the ranks' rows stacked in rank order with empty ranks dropped,
batch_norm_gather_stats_with_counts, batch_norm_elemt and bf16 ReLU / add forward; threshold_backward,
batch_norm_backward_reduce, an fp32 left fold of the ranks' [sum_dy; sum_dy_xmu] in rank order and
batch_norm_backward_elemt backward.  Every rank's output, input / identity gradients, dweight, dbias, running
statistics and num_batches_tracked must have the reference's bits.

Sites: ReLU (stem / conv1 / conv2 positions), tails with one and with two output gradients, and plain sites (the
module's own forward, e.g. a downsample branch).  Shapes: every batch-norm shape of ResNet-50 with a global batch
split unevenly over the ranks, including an empty and a single-row rank; one shape per launch regime of the reducing
kernels on rank 0 with one image on every other rank (gpu_common.BN_REGIME_SHAPES); C = 100 (scalar kernels, no
mask); an operand off the 16-byte grid, on every rank or on one rank only; ranks whose row walks through the
statistics' and backward reduce's rings have different lengths (test_bn_ring_cpu.sync_splits); the value edges of
test_gpu_fused_norm; through the C-ABI, a ReLU site that reads y instead of a mask at C % 8 == 0, with one output
gradient or two, and the sync scratch's guard bytes."""
import copy

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_MAX_CHANNELS, BN_REGIME_SHAPES, assert_same_values
from test_bn_ring_cpu import SYNC_RING_C, sync_splits
from test_gpu_fused_norm import RESNET50_BN_SHAPES, edge_bn_setup, edge_site_inputs, misaligned

pytestmark = pytest.mark.gpu

CL = torch.channels_last
KINDS = ["relu", "tail", "tail2", "plain"]
# Sites where the batch norm runs alone (its module forward) and torch's ops follow in place on its output: a
# SyncBatchNorm followed by an inplace ReLU, and the fused blocks' fallbacks when the batch norm has a forward hook
# (`relu(bn(x))` and `out = bn(x); out += identity; relu(out)` with the block's inplace ReLU) or the ReLU has one
# (`relu(bn(x))`, the hook called on every rank).  Each is checked against the reference of the site it computes.
INPLACE_KINDS = {"seq_inplace_relu": "relu", "hooked_relu": "relu", "hooked_tail": "tail", "hooked_relu_module": "relu"}
GUARD = 64 << 10


@pytest.fixture(scope="module", params=[2, 3, 4, 8])
def world(request):
    from ant_ray_b200.loopback import LoopbackWorld

    w = LoopbackWorld(request.param, device=0, key=f"syncbn{request.param}", staging_bytes=1 << 20, max_blocks=8,
                      timeout_ms=20000)
    load_torch_kernels()
    yield w
    w.destroy()


def load_torch_kernels():
    """Launch the torch kernels a sync site uses between its collectives once, outside the world: with lazy module
    loading, a kernel's first launch can wait for the kernels running in the context, and in a loopback world those
    include a peer's collective that waits for this rank (one process per GPU has no such wait)."""
    t = torch.zeros(8, 8, 2, 2, dtype=torch.bfloat16, device="cuda")
    torch.zeros(16, dtype=torch.uint8, device="cuda")
    torch.zeros_like(t, memory_format=CL)
    torch.cuda.synchronize()


def split_rows(n, W, seed):
    """Uneven per-rank batch sizes summing to n: one row on rank 1 and, for W > 2, an empty rank 0."""
    if W == 2:
        return [n - 1, 1]
    g = torch.Generator().manual_seed(seed)
    sizes = [0, 1] + [1] * (W - 2)
    for _ in range(n - W + 1):
        sizes[2 + int(torch.randint(0, W - 2, (1,), generator=g))] += 1
    return sizes


def make_sync_bn(c, seed, momentum=0.1, eps=1e-5):
    g = torch.Generator().manual_seed(seed)
    bn = nn.SyncBatchNorm(c, eps=eps, momentum=momentum)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
        bn.bias.copy_(0.2 * torch.randn(c, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
        bn.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
        bn.num_batches_tracked.fill_(5)
    return bn.cuda()


def cl(t):
    n, c, h, w = t.shape
    return torch.empty(n, h, w, c, dtype=t.dtype, device=t.device).permute(0, 3, 1, 2).copy_(t)


def reference(bn, xs, ids, dys, dy2s, kind):
    """torch's SyncBatchNorm arithmetic for every rank: a list of per-rank result dicts.  As in torch, a rank
    without rows has no gradient for the batch norm's input, weight or bias (None)."""
    kind = INPLACE_KINDS.get(kind, kind)
    W, c = len(xs), bn.num_features
    eps, momentum = bn.eps, bn.momentum
    w, b = bn.weight.detach(), bn.bias.detach()
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    rows = []
    for x in xs:
        if x.numel():
            mean, invstd = torch.batch_norm_stats(x, eps)
            rows.append(torch.cat([mean, invstd, torch.full((1,), x.numel() // c, dtype=torch.float32, device=x.device)]))
        else:
            rows.append(torch.zeros(2 * c + 1, dtype=torch.float32, device=x.device))
    gathered = torch.stack(rows)
    keep = gathered[:, 2 * c] >= 1
    mean_all, invstd_all, count_all = gathered[keep, :c], gathered[keep, c:2 * c], gathered[keep, 2 * c:]
    x0 = next(x for x in xs if x.numel())
    mean, invstd = torch.batch_norm_gather_stats_with_counts(x0, mean_all, invstd_all, rm, rv, momentum, eps, count_all.view(-1))
    counts = count_all.view(-1).to(torch.int32)
    out, grads, sums = [], [], []
    for r, x in enumerate(xs):
        res = {}
        if x.numel():
            t = torch.batch_norm_elemt(x, w, b, mean, invstd, eps)
            if kind in ("tail", "tail2"):
                t = t + ids[r]
            y = torch.relu(t) if kind != "plain" else t
            dy = dys[r] + dy2s[r] if kind == "tail2" else dys[r]
            g = torch.ops.aten.threshold_backward(dy, y, 0) if kind != "plain" else dy
            s_dy, s_dy_xmu, dw, db = torch.batch_norm_backward_reduce(g, x, mean, invstd, w, True, True, True)
        else:
            y, g = torch.empty_like(x), torch.empty_like(x)
            s_dy = s_dy_xmu = torch.zeros(c, dtype=torch.float32, device=x.device)
            dw = db = None
        res.update(y=y, dweight=dw, dbias=db)
        if kind in ("tail", "tail2"):
            res["d_identity"] = g
        out.append(res)
        grads.append(g)
        sums.append(torch.cat([s_dy, s_dy_xmu]))
    total = sums[0]
    for s in sums[1:]:
        total = total + s   # the rank-order fold
    for r, x in enumerate(xs):
        dx = torch.batch_norm_backward_elemt(grads[r], x, mean, invstd, w, total[:c], total[c:], counts) if x.numel() else None
        out[r].update(dx=dx, running_mean=rm, running_var=rv, num_batches_tracked=bn.num_batches_tracked + 1)
    return out


def run_native(world, bn, xs, ids, dys, dy2s, kind, misalign=(), misalign_ranks=None):
    """`misalign` names the operands moved off the 16-byte grid, on the ranks in `misalign_ranks` (every rank when
    None)."""
    W = world.world_size
    bns = [fused_norm.sync_batch_norm(copy.deepcopy(bn), world.comms[r]) for r in range(W)]
    relu = nn.ReLU(inplace=True)
    results = [None] * W
    hook_ranks = []
    # inputs that require grad are leaves made on the current stream before the ranks' streams start
    # (an empty input keeps its own strides: see test_empty_rank_input_from_a_convolution)
    off = lambda r: misalign_ranks is None or r in misalign_ranks  # noqa: E731
    xs = [(misaligned(x) if "x" in misalign and x.numel() and off(r) else x.clone() if x.numel() else x.detach()).requires_grad_()
          for r, x in enumerate(xs)]
    ids = [(i.clone() if i is not None else None) for i in ids]
    for i in ids:
        if i is not None:
            i.requires_grad_()

    def step(r, comm):
        bnr = bns[r]
        assert type(bnr) is fused_norm.FusedSyncBatchNorm and bnr.b200_comm is comm
        if kind == "relu":
            outs, gs = [fused_norm.bn_relu(bnr, relu, xs[r])], [dys[r]]
        elif kind == "tail":
            outs, gs = [fused_norm.bn_add_relu(bnr, relu, xs[r], ids[r])], [dys[r]]
        elif kind == "tail2":
            outs, gs = list(fused_norm.bn_add_relu(bnr, relu, xs[r], ids[r], pair=True)), [dys[r], dy2s[r]]
        elif kind == "seq_inplace_relu":
            outs, gs = [nn.Sequential(bnr, nn.ReLU(inplace=True))(xs[r])], [dys[r]]
        elif kind == "hooked_relu":
            bnr.register_forward_hook(lambda *a: None)
            outs, gs = [fused_norm.bn_relu(bnr, relu, xs[r])], [dys[r]]
        elif kind == "hooked_tail":
            bnr.register_forward_hook(lambda *a: None)
            outs, gs = [fused_norm.bn_add_relu(bnr, relu, xs[r], ids[r], pair=True)[0]], [dys[r]]
        elif kind == "hooked_relu_module":
            hooked = nn.ReLU(inplace=True)
            hooked.register_forward_hook(lambda *a: hook_ranks.append(r))
            outs, gs = [fused_norm.bn_relu(bnr, hooked, xs[r])], [dys[r]]
        else:
            outs, gs = [bnr(xs[r])], [dys[r]]
        torch.autograd.backward(outs, gs)
        results[r] = outs[0]

    before = N.launch_count()
    world.run(step)
    torch.cuda.synchronize()
    launched = N.launch_count() - before
    world.check()
    if kind == "hooked_relu_module":
        assert sorted(hook_ranks) == list(range(W)), hook_ranks
    got = []
    for r in range(W):
        res = {"y": results[r].detach(), "dx": xs[r].grad, "dweight": bns[r].weight.grad, "dbias": bns[r].bias.grad,
               "running_mean": bns[r].running_mean, "running_var": bns[r].running_var,
               "num_batches_tracked": bns[r].num_batches_tracked}
        if ids[r] is not None:
            res["d_identity"] = ids[r].grad
        got.append(res)
    return got, launched


def collective_launches(world, c):
    """The launches of one sync site's two collectives over all ranks: the allgather of 2C + 1 statistics floats and
    the all-reduce of 2C sums, each in as many pieces as the world's staging takes."""
    W = world.world_size
    rows = [torch.zeros(2 * c + 1, device="cuda") for _ in range(W)]
    gathered = [[torch.empty(2 * c + 1, device="cuda") for _ in range(W)] for _ in range(W)]
    sums = [torch.zeros(2 * c, device="cuda") for _ in range(W)]
    before = N.launch_count()

    def step(r, comm):
        comm.allgather(rows[r].data_ptr(), [t.data_ptr() for t in gathered[r]], 2 * c + 1, N.FLOAT32)
        comm.allreduce(sums[r].data_ptr(), sums[r].data_ptr(), 2 * c, N.FLOAT32, N.SUM)

    world.run(step)
    torch.cuda.synchronize()
    world.check()
    return N.launch_count() - before


def check_sites(world, n, c, h, w, kind, seed, inputs=None, bn_setup=None, misalign=(), sizes=None, collectives=None,
                misalign_ranks=None, **bn_args):
    W = world.world_size
    sizes = sizes or split_rows(n, W, seed)
    assert sum(sizes) == n
    g = torch.Generator(device="cuda").manual_seed(seed)
    if inputs is None:
        act = lambda s, t: cl((torch.randn(n, c, h, w, device="cuda", generator=g) * s + t).to(torch.bfloat16))
        x, dy, dy2, identity = act(2.0, 0.5), act(1.0, 0.0), act(1.0, 0.1), act(1.0, -0.2)
    else:
        x, dy, identity = inputs
        dy2 = cl(torch.randn(n, c, h, w, device="cuda", generator=g).to(torch.bfloat16))
    bounds = [sum(sizes[:r]) for r in range(W + 1)]
    part = lambda t: [cl(t[bounds[r]:bounds[r + 1]]) for r in range(W)]
    xs, dys, dy2s, ids = part(x), part(dy), part(dy2), part(identity)
    if INPLACE_KINDS.get(kind, kind) not in ("tail", "tail2"):
        ids = [None] * W
    bn = make_sync_bn(c, seed, **bn_args)
    if bn_setup is not None:
        bn_setup(bn)
    want = reference(bn, xs, ids, dys, dy2s, kind)
    got, launched = run_native(world, bn, xs, ids, dys, dy2s, kind, misalign, misalign_ranks)
    compare(got, want, sizes)
    # per rank: 2 collectives (one launch each, unless `collectives` counts their pieces), the merge, and 4 local
    # kernels when it has rows
    collectives = 2 * W if collectives is None else collectives
    assert launched == collectives + sum(1 + (4 if s else 0) for s in sizes), launched


def compare(got, want, sizes):
    bad = []
    for r in range(len(want)):
        for k in want[r]:
            try:
                if want[r][k] is None or got[r][k] is None:
                    assert want[r][k] is None and got[r][k] is None, f"rank {r} {k}: None on one side only"
                    continue
                assert_same_values(got[r][k], want[r][k], f"rank {r} ({sizes[r]} images) {k}")
            except AssertionError as e:
                print(e)
                bad.append((r, k))
    assert not bad, f"differs from torch's SyncBatchNorm arithmetic: {bad}"


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("c,h,w", RESNET50_BN_SHAPES)
def test_resnet50_sites_match_torch_sync_batch_norm(world, c, h, w, kind):
    n = 2 * world.world_size + 3
    check_sites(world, n, c, h, w, kind, seed=c * 7 + h + world.world_size)


@pytest.mark.parametrize("kind", ["relu", "tail2", "plain"])
@pytest.mark.parametrize("n,c,h,w", list(BN_REGIME_SHAPES))
def test_every_launch_regime_matches_torch_sync_batch_norm(world, n, c, h, w, kind):
    # rank 0 runs the regime's launch shape; every other rank holds one image, so the ranks' launch shapes differ
    W = world.world_size
    if W > 3:
        pytest.skip("the regime sweep runs at W = 2 and W = 3")
    sizes = [n] + [1] * (W - 1)
    collectives = None
    if c == BN_MAX_CHANNELS:
        # 2C + 1 floats are more than the world's 1 MiB staging takes in one piece
        collectives = collective_launches(world, c)
        assert collectives > 2 * W, collectives
    check_sites(world, sum(sizes), c, h, w, kind, seed=n + c + h + W, sizes=sizes, collectives=collectives)


@pytest.mark.parametrize("kind", KINDS)
def test_scalar_channels_and_one_row_ranks(world, kind):
    # C = 100: the scalar statistics / elementwise kernels and no mask; every rank holds 0 or 1 image of 3 x 3
    W = world.world_size
    sizes = [1 if r % 2 == 0 else 0 for r in range(W)]
    sizes[-1] = 1
    check_sites(world, sum(sizes), 100, 3, 3, kind, seed=11 + W, sizes=sizes)


@pytest.mark.parametrize("kind", KINDS)
def test_empty_rank_at_every_position(world, kind):
    W = world.world_size
    for empty in range(W):
        sizes = [3] * W
        sizes[empty] = 0
        check_sites(world, sum(sizes), 256, 5, 5, kind, seed=empty, sizes=sizes)


@pytest.mark.parametrize("kind", list(INPLACE_KINDS))
def test_inplace_ops_after_a_batch_norm_alone(world, kind):
    # the plain site saves only its input, so torch's inplace ReLU or `+= identity` on its output is allowed
    check_sites(world, 2 * world.world_size + 3, 64, 14, 14, kind, seed=21)
    check_sites(world, 2 * world.world_size + 3, 100, 7, 7, kind, seed=22)


@pytest.mark.parametrize("kind", ["relu", "plain"])
def test_empty_rank_input_from_a_convolution(world, kind):
    # A convolution over an empty batch returns default (NCHW) strides whatever its input's layout, so the empty
    # rank's activation is not channels-last; it must still take the sync site, or its peers would wait for it.
    W, c = world.world_size, 64
    sizes = [0] + [2 + r for r in range(1, W)]
    torch.manual_seed(4)
    conv = nn.Conv2d(16, c, 3, padding=1).cuda().to(torch.bfloat16).to(memory_format=CL)
    g = torch.Generator(device="cuda").manual_seed(4)
    with torch.no_grad():
        xs = [conv(torch.randn(m, 16, 9, 9, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL))
              for m in sizes]
    dys = [cl(torch.randn(x.shape, device="cuda", generator=g).to(torch.bfloat16)) for x in xs]
    bn = make_sync_bn(c, 4)
    want = reference(bn, xs, [None] * W, dys, [None] * W, kind)
    got, launched = run_native(world, bn, xs, [None] * W, dys, [None] * W, kind)
    compare(got, want, sizes)
    assert launched == sum(3 + (4 if s else 0) for s in sizes), launched


@pytest.mark.parametrize("kind", ["relu", "tail2", "plain"])
def test_misaligned_input_takes_the_scalar_kernels(world, kind):
    check_sites(world, 3 * world.world_size, 64, 7, 7, kind, seed=5, misalign=("x",))


@pytest.mark.parametrize("kind", ["relu", "tail2", "plain"])
def test_ranks_walk_the_rings_for_different_lengths(world, kind):
    # H = W = 1: each rank's rows are its images.  Every split runs once with every rank on its ring and once with one
    # rank's x off the 16-byte grid, so that rank takes the register walks while its peers take the rings.
    W = world.world_size
    for i, sizes in enumerate(sync_splits(W)):
        check_sites(world, sum(sizes), SYNC_RING_C, 1, 1, kind, seed=31 * i + W, sizes=sizes)
        rank = max(range(W), key=lambda r: (sizes[r], -r)) if i % 2 else (i // 2) % W
        if sizes[rank]:
            check_sites(world, sum(sizes), SYNC_RING_C, 1, 1, kind, seed=31 * i + W, sizes=sizes, misalign=("x",),
                        misalign_ranks=(rank,))


@pytest.mark.parametrize("kind", ["tail", "plain"])
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges(world, grad_edges, kind):
    n, c, h, w = 8, 64, 16, 16
    inputs = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    inputs = tuple(cl(t) for t in inputs)
    check_sites(world, n, c, h, w, kind, seed=3, inputs=inputs, bn_setup=edge_bn_setup(grad_edges))


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters(world, momentum, eps):
    check_sites(world, 2 * world.world_size + 1, 100, 14, 14, "tail2", seed=9, momentum=momentum, eps=eps)


def test_sync_scratch_guard_and_semaphores(world):
    # direct C-ABI calls on each rank's own scratch with guard bytes past b200c_bn_sync_scratch_bytes(c, W)
    W = world.world_size
    lib = N.load()
    c, rows = 2048, [64 * 49 if r % 2 else 0 for r in range(W)]
    rows[0] = 32768   # a 128-block grid merge in the statistics and backward-reduce kernels
    need = int(lib.b200c_bn_sync_scratch_bytes(c, W))
    assert need > int(lib.b200c_bn_scratch_bytes(c))
    bufs = []
    for _ in range(W):
        buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
        buf[:need].zero_()
        buf[need:].fill_(0xA5)
        bufs.append(buf)
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16) for m in rows]
    dys = [torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16) for m in rows]
    bn = make_sync_bn(c, 1)
    st = [dict(rm=bn.running_mean.clone(), rv=bn.running_var.clone(), y=torch.empty_like(x), dx=torch.empty_like(x),
               stats=torch.empty(2 * c + 1, device="cuda"), dw=torch.empty(c, device="cuda"), db=torch.empty(c, device="cuda"))
          for x in xs]
    w_, b_ = bn.weight.detach(), bn.bias.detach()

    def step(r, comm):
        s, m, p = st[r], rows[r], st[r]["stats"].data_ptr()
        stream = torch.cuda.current_stream().cuda_stream
        for _ in range(2):
            N.check(lib.b200c_bn_sync_forward(comm._h(), xs[r].data_ptr(), None, s["y"].data_ptr(), None, 0, w_.data_ptr(),
                                              b_.data_ptr(), s["rm"].data_ptr(), s["rv"].data_ptr(), None, p, p + 4 * c,
                                              p + 8 * c, m, c, 0.1, 1e-5, bufs[r].data_ptr(), stream))
            N.check(lib.b200c_bn_sync_backward(comm._h(), dys[r].data_ptr(), None, None, None, 0, xs[r].data_ptr(), None,
                                               s["dx"].data_ptr(), w_.data_ptr(), p, p + 4 * c, p + 8 * c, s["dw"].data_ptr(),
                                               s["db"].data_ptr(), m, c, bufs[r].data_ptr(), stream))

    world.run(step)
    torch.cuda.synchronize()
    world.check()
    for buf in bufs:
        assert (buf[need:] == 0xA5).all(), "a call wrote past b200c_bn_sync_scratch_bytes(c, W)"
        assert (buf[:16384] == 0).all(), "a call left a semaphore set"
    # every rank holds the same global statistics
    for s in st[1:]:
        assert_same_values(s["stats"], st[0]["stats"], "global statistics")


@pytest.mark.parametrize("c", [64, 2048])
def test_relu_site_reading_y_through_the_c_abi(world, c):
    check_relu_site_reading_y(world, c)


@pytest.mark.parametrize("c", [64, 2048])
def test_relu_site_reading_y_with_two_gradients_through_the_c_abi(world, c):
    # the backward reduce's ring of dy, x, y and dy2: 4 operands, 2 stages
    check_relu_site_reading_y(world, c, two_grads=True)


def check_relu_site_reading_y(world, c, two_grads=False):
    """b200c_bn_sync_forward with relu = 1 and no mask, then b200c_bn_sync_backward from y: the vector elementwise
    backward that reads y and the device's 1 / rows of all ranks (the fused module passes a mask at C % 8 == 0).  The
    ranks hold different batch sizes, so a rank's own 1 / rows would differ from the global one.  With `two_grads`
    the output has a second gradient dy2, summed to bf16(dy + dy2) as autograd sums it."""
    W, h, w = world.world_size, 5, 5
    sizes = [2 + r for r in range(W)]
    lib = N.load()
    g = torch.Generator(device="cuda").manual_seed(c + W)
    xs = [cl((torch.randn(m, c, h, w, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)) for m in sizes]
    dys = [cl(torch.randn(m, c, h, w, device="cuda", generator=g).to(torch.bfloat16)) for m in sizes]
    dy2s = [cl(torch.randn(m, c, h, w, device="cuda", generator=g).to(torch.bfloat16)) if two_grads else None for m in sizes]
    bn = make_sync_bn(c, c + W)
    want = reference(bn, xs, [None] * W, [d + d2 for d, d2 in zip(dys, dy2s)] if two_grads else dys, [None] * W, "relu")
    need = int(lib.b200c_bn_sync_scratch_bytes(c, W))
    w_, b_ = bn.weight.detach(), bn.bias.detach()
    st = [dict(rm=bn.running_mean.clone(), rv=bn.running_var.clone(), nbt=bn.num_batches_tracked.clone(), y=torch.empty_like(x),
               dx=torch.empty_like(x), stats=torch.empty(2 * c + 1, device="cuda"), dw=torch.empty(c, device="cuda"),
               db=torch.empty(c, device="cuda"), scratch=torch.zeros(need, dtype=torch.uint8, device="cuda")) for x in xs]

    def step(r, comm):
        s, m, p = st[r], sizes[r] * h * w, st[r]["stats"].data_ptr()
        stream = torch.cuda.current_stream().cuda_stream
        N.check(lib.b200c_bn_sync_forward(comm._h(), xs[r].data_ptr(), None, s["y"].data_ptr(), None, 1, w_.data_ptr(),
                                          b_.data_ptr(), s["rm"].data_ptr(), s["rv"].data_ptr(), s["nbt"].data_ptr(), p, p + 4 * c,
                                          p + 8 * c, m, c, 0.1, 1e-5, s["scratch"].data_ptr(), stream))
        N.check(lib.b200c_bn_sync_backward(comm._h(), dys[r].data_ptr(), dy2s[r].data_ptr() if two_grads else None, s["y"].data_ptr(),
                                           None, 1, xs[r].data_ptr(), None, s["dx"].data_ptr(), w_.data_ptr(), p, p + 4 * c, p + 8 * c,
                                           s["dw"].data_ptr(), s["db"].data_ptr(), m, c, s["scratch"].data_ptr(), stream))

    world.run(step)
    torch.cuda.synchronize()
    world.check()
    got = [{"y": s["y"], "dx": s["dx"], "dweight": s["dw"], "dbias": s["db"], "running_mean": s["rm"], "running_var": s["rv"],
            "num_batches_tracked": s["nbt"]} for s in st]
    compare(got, want, sizes)
