"""The vector paths' row rings (norm_kernels.cuh) against eager torch, bit for bit.

k_bn_stats<4>, k_bn_stats_dual<4> and the vector path of k_bn_bwd_reduce (kBwdVec channels per hardware thread)
read their rows through per-thread cp.async rings of kStatsStages or bwd_ring_stages(dual) iterations.  Each case
runs a row walk of 1, D - 1, D, D + 1 and 2D + 1 iterations for every ring depth D, with the last iteration partly
past M, through every ring kernel: the statistics, the dual statistics, and the reduce from the ReLU bits, from y,
from dy (no ReLU), for a tail with dy2 that writes g, and for a downsample tail (dual, from the bits and from y).
tests/test_bn_ring_cpu.py checks that these shapes walk those lengths.

Through the C-ABI, every ring is also held to the register walk: each site runs once with every operand on the
16-byte grid (the ring) and once with an operand moved off it, which bwd_reduce_launch and launch_stats answer with
the register walk.  Both claim torch's per-channel order, so every output must keep its bits: y, the mask, the
saved and running statistics, num_batches_tracked, dx, dx of the downsample branch, g, dweight and dbias.  The sweep
covers every operand set of the backward ring (2 to 5 operands: BWD_VARIANTS), C = 8 to 131072 and the walk lengths
above on one row of blocks and on merged grids (ABI_RING_WALKS); the local variants are compared with torch's functional
chain as well.  A second test moves each operand the launcher checks off the grid on its own, 2 and 8 bytes past a
16-byte boundary."""
import copy

import pytest
import torch
import torch.nn as nn

import test_gpu_fused_dual as D
import test_gpu_fused_norm as L
import test_gpu_fused_res as R
from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import assert_same_values, bn_launch_config, same_bits
from test_bn_ring_cpu import ABI_RING_WALKS, BWD_RINGS, BWD_VARIANTS, RING_WALKS, launcher_operands

pytestmark = pytest.mark.gpu

# M = 2 .. 513 keep one row of blocks, the others merge a grid of 128 rows of blocks.  C = 24 has a 16-wide tile
# with 8 channels past C, C = 4104 8 valid channels in its last tile.
SHAPES = [(m, c, 1, 1) for c, m in RING_WALKS]


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
@pytest.mark.parametrize("residual", [False, True], ids=["relu_bits", "tail_g"])
def test_stats_and_reduce_from_the_mask(n, c, h, w, residual):
    L.check_site(n, c, h, w, residual)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_reduce_from_y(n, c, h, w):
    L.check_native_site(n * h * w, c, c + n)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_reduce_from_dy(n, c, h, w):
    R.check_gauss_site("plain", n, c, h, w)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_tail_with_two_gradients_writes_g(n, c, h, w):
    g = torch.Generator(device="cuda").manual_seed(n + c)
    t = lambda s, o: nhwc((torch.randn(n, c, h, w, device="cuda", generator=g) * s + o).to(torch.bfloat16))  # noqa: E731
    x, identity, dy, dy2 = t(2.0, 0.5), t(1.0, -0.2), t(1.0, 0.0), t(1.0, 0.0)
    bn = L.make_bn(c, 4)

    def run(fused):
        b = copy.deepcopy(bn)
        xg, ig = x.clone().requires_grad_(), identity.clone().requires_grad_()
        relu = nn.ReLU(inplace=True)
        if fused:
            ys = fused_norm.bn_add_relu(b, relu, xg, ig, pair=True)
        else:
            out = b(xg)
            out += ig
            y = relu(out)
            ys = (y, y)
        torch.autograd.backward([ys[0], ys[1]], [dy, dy2])
        return [ys[0].detach(), xg.grad, ig.grad, b.weight.grad, b.bias.grad, b.running_mean, b.running_var]

    want, got = run(False), run(True)
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if not same_bits(a, b)]
    assert not bad, bad


@pytest.mark.parametrize("n,c,h,w", SHAPES)
@pytest.mark.parametrize("mode", ["one", "pair"])
def test_dual_stats_and_reduce(n, c, h, w, mode):
    x3, x_ds, dy1, dy2 = D.inputs(n, c, h, w, c + n)
    D.check_dual(x3, x_ds, dy1, dy2, mode, L.make_bn(c, 1), L.make_bn(c, 2))


@pytest.mark.parametrize("n,c,h,w", [s for s in SHAPES if s[1] <= 2048])
def test_dual_reduce_from_y(n, c, h, w):
    D.check_dual_through_the_c_abi(n, c, h, w)


# ---- ring against register walk, through the C-ABI ------------------------------------------------------------
DUAL_MAX_C = 65536
# forward call of each backward variant's site: the ReLU site writes y and its bits, a plain site (no ReLU) y alone
FORWARD_OF = {"mask": "relu", "y": "relu", "dy": "plain"}


def placed(t, offset):
    """A copy of `t` whose data pointer is `offset` bytes past a 16-byte boundary; `t` itself for 0."""
    if not offset:
        return t
    flat = torch.empty(t.numel() + 16 // t.element_size(), dtype=t.dtype, device=t.device)
    v = flat[offset // t.element_size():][:t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == offset
    return v


def nan_filled(shape, offset=0, dtype=torch.bfloat16):
    """An output buffer filled with all-ones bits (a NaN), so an element the kernel never writes shows."""
    t = placed(torch.empty(shape, dtype=dtype, device="cuda"), offset)
    t.view(torch.uint8 if dtype == torch.uint8 else torch.int16 if t.element_size() == 2 else torch.int32).fill_(-1 if dtype != torch.uint8 else 255)
    return t


class Site:
    """Seeded inputs of one (M, C) site and its two batch norms' parameters (the second is a downsample branch's)."""

    def __init__(self, m, c):
        g = torch.Generator(device="cuda").manual_seed(m * 7 + c)
        t = lambda s, o: (torch.randn(m, c, device="cuda", generator=g) * s + o).to(torch.bfloat16)  # noqa: E731
        self.m, self.c = m, c
        self.x, self.x_ds, self.dy, self.dy2 = t(2.0, 0.5), t(1.5, -0.3), t(1.0, 0.0), t(1.0, 0.1)
        self.bns = [L.make_bn(c, m + c), L.make_bn(c, m + c + 1)]
        self.scratch = {}

    def buf(self, dual):
        """One guarded scratch per kind for the whole site: every call must leave its semaphores at zero."""
        if dual not in self.scratch:
            lib = N.load()
            need = int(lib.b200c_bn_dual_scratch_bytes(self.c) if dual else lib.b200c_bn_scratch_bytes(self.c))
            b = torch.empty(need + L.GUARD, dtype=torch.uint8, device="cuda")
            b[:need].zero_()
            b[need:].fill_(0xA5)
            self.scratch[dual] = (b, need)
        return self.scratch[dual]


def p(t):
    return t.data_ptr() if t is not None else None


def forward(site, kind, place=None):
    """b200c_bn_forward_mask ("relu"), b200c_bn_forward_res without identity ("plain") or b200c_bn_forward_dual,
    with the operands named in `place` (name -> byte offset) moved off the 16-byte grid."""
    place = place or {}
    lib, m, c = N.load(), site.m, site.c
    s = torch.cuda.current_stream().cuda_stream
    x, x_ds = placed(site.x, place.get("x", 0)), placed(site.x_ds, place.get("x_ds", 0))
    y = nan_filled((m, c))
    mask = nan_filled((m * c // 8,), dtype=torch.uint8) if kind != "plain" else None
    out = {"y": y, "mask": mask}
    stats = []
    for i, bn in enumerate(site.bns[:2 if kind == "dual" else 1]):
        st = {"running_mean": bn.running_mean.clone(), "running_var": bn.running_var.clone(),
              "num_batches_tracked": bn.num_batches_tracked.clone(), "mean": nan_filled(c, dtype=torch.float32),
              "invstd": nan_filled(c, dtype=torch.float32)}
        stats.append([p(bn.weight), p(bn.bias), p(st["running_mean"]), p(st["running_var"]), p(st["num_batches_tracked"]),
                      p(st["mean"]), p(st["invstd"])])
        out.update({f"{k}{'_ds' * i}": v for k, v in st.items()})
    buf, need = site.buf(kind == "dual")
    if kind == "relu":
        N.check(lib.b200c_bn_forward_mask(p(x), None, p(y), p(mask), *stats[0], m, c, 0.1, 1e-5, p(buf), s))
    elif kind == "plain":
        N.check(lib.b200c_bn_forward_res(p(x), None, None, 0, p(y), *stats[0], m, c, 0.1, 1e-5, p(buf), s))
    else:
        N.check(lib.b200c_bn_forward_dual(p(x), p(x_ds), p(y), p(mask), *stats[0], 0.1, 1e-5, *stats[1], 0.1, 1e-5, m, c, p(buf), s))
    torch.cuda.synchronize()
    L.check_scratch(buf, need)
    return out


def backward(site, name, fwd, place=None):
    """One backward variant (BWD_VARIANTS) from the forward's y, bits and statistics, with the operands named in
    `place` moved off the 16-byte grid."""
    place = place or {}
    v = BWD_VARIANTS[name]
    lib, m, c = N.load(), site.m, site.c
    s = torch.cuda.current_stream().cuda_stream
    on = lambda k, t: placed(t, place.get(k, 0)) if t is not None else None  # noqa: E731
    x, dy, dy2 = on("x", site.x), on("dy", site.dy), on("dy2", site.dy2 if v["dy2"] else None)
    y = on("y", fwd["y"] if v["src"] == "y" else None)
    mask = fwd["mask"] if v["src"] == "mask" else None
    g = nan_filled((m, c), place.get("g", 0)) if v["g"] else None
    out = {"dx": nan_filled((m, c)), "g": g}
    sums = [nan_filled(c, dtype=torch.float32) for _ in range(4)]
    out.update(dweight=sums[0], dbias=sums[1])
    w, mean, invstd = p(site.bns[0].weight), p(fwd["mean"]), p(fwd["invstd"])
    buf, need = site.buf(v["dual"])
    if v["dual"]:
        out.update(dx_ds=nan_filled((m, c)), dweight_ds=sums[2], dbias_ds=sums[3])
        N.check(lib.b200c_bn_backward_dual(p(dy), p(dy2), p(y), p(mask), p(x), p(on("x_ds", site.x_ds)), p(out["dx"]),
                                           p(out["dx_ds"]), w, mean, invstd, p(sums[0]), p(sums[1]), p(site.bns[1].weight),
                                           p(fwd["mean_ds"]), p(fwd["invstd_ds"]), p(sums[2]), p(sums[3]), m, c, p(buf), s))
    elif v["src"] == "mask":
        N.check(lib.b200c_bn_backward_mask(p(dy), p(dy2), p(mask), p(x), p(g), p(out["dx"]), w, mean, invstd, p(sums[0]),
                                           p(sums[1]), m, c, p(buf), s))
    elif v["src"] == "y":
        N.check(lib.b200c_bn_backward(p(dy), p(y), p(x), p(g), p(out["dx"]), w, mean, invstd, p(sums[0]), p(sums[1]), m, c,
                                      p(buf), s))
    else:
        N.check(lib.b200c_bn_backward_res(p(dy), None, 0, p(x), p(g), p(out["dx"]), w, mean, invstd, p(sums[0]), p(sums[1]), m,
                                          c, p(buf), s))
    torch.cuda.synchronize()
    L.check_scratch(buf, need)
    return out


def assert_same(got, want, where):
    """Every output of `want` with the same bits in `got` (compared on the device; the report names the first
    differing element)."""
    for k, w in want.items():
        if w is None:
            assert got[k] is None, (where, k)
        elif not same_bits(got[k], w):
            assert_same_values(got[k], w, f"{where}: {k}")


def variants_of(c):
    return [n for n, v in BWD_VARIANTS.items() if c <= DUAL_MAX_C or not v["dual"]]


def against_torch(site, name, fwd, bwd):
    """The local variants against torch's functional chain (tests/test_gpu_fused_norm.torch_site)."""
    v = BWD_VARIANTS[name]
    bn = site.bns[0]
    want = L.torch_site(site.x, site.dy, bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var,
                        dy2=site.dy2 if v["dy2"] else None, relu=v["src"] != "dy")
    got = {"y": fwd["y"], "mean": fwd["mean"], "invstd": fwd["invstd"], "running_mean": fwd["running_mean"],
           "running_var": fwd["running_var"], "dx": bwd["dx"], "dweight": bwd["dweight"], "dbias": bwd["dbias"]}
    if v["g"]:
        got["g"] = bwd["g"]
    assert_same(got, {k: want[k] for k in got}, f"{name} against torch")


@pytest.mark.parametrize("c,m", list(ABI_RING_WALKS), ids=[f"c{c}-m{m}-walk{n}" for (c, m), n in ABI_RING_WALKS.items()])
def test_ring_and_register_walk_give_the_same_bits(c, m):
    """Every variant once with all operands on the 16-byte grid (the rings) and once with x 2 bytes past it (the
    statistics' and the backward reduce's register walks)."""
    site = Site(m, c)
    names = variants_of(c)
    for kind in ("relu", "plain", "dual"):
        if kind == "dual" and c > DUAL_MAX_C:
            continue
        ring, walk = forward(site, kind), forward(site, kind, {"x": 2})
        assert_same(walk, ring, f"{kind} forward")
        assert int(ring["num_batches_tracked"]) == int(site.bns[0].num_batches_tracked) + 1
        for name in names:
            v = BWD_VARIANTS[name]
            if (kind == "dual") != v["dual"] or (kind != "dual" and FORWARD_OF[v["src"]] != kind):
                continue
            want = backward(site, name, ring)
            assert_same(backward(site, name, ring, {"x": 2}), want, f"{name} ({BWD_RINGS[name][0]} operands, "
                                                                     f"{BWD_RINGS[name][1]} stages)")
            if v["dual"]:
                assert same_bits(want["dbias"], want["dbias_ds"])   # Σg is both dbias values
            else:
                against_torch(site, name, ring, want)


# one row of blocks at C = 4104 (a partial tile), a merged grid at C = 64 and C = 2048
ALONE_SHAPES = [(4104, 97), (64, 32769), (2048, 1793)]


@pytest.mark.parametrize("offset", [2, 8])
@pytest.mark.parametrize("c,m", ALONE_SHAPES)
def test_each_launcher_operand_off_the_grid_alone(c, m, offset):
    """Each operand bwd_reduce_launch checks, alone 2 or 8 bytes past a 16-byte boundary (8 is on cp.async's 8-byte
    grid but off vec_ok's 16-byte one), gives the bits of the all-aligned call."""
    assert m in {mm for cc, mm in ABI_RING_WALKS if cc == c} and bn_launch_config(m, c).block_x % 8 == 0
    site = Site(m, c)
    fwds = {kind: forward(site, kind) for kind in ("relu", "plain", "dual")}
    for name in variants_of(c):
        v = BWD_VARIANTS[name]
        fwd = fwds["dual" if v["dual"] else FORWARD_OF[v["src"]]]
        want = backward(site, name, fwd)
        for op in launcher_operands(v):
            assert_same(backward(site, name, fwd, {op: offset}), want, f"{name} with {op} at {offset} mod 16")
    # the statistics check x (and x_ds at a dual site) alone
    for kind, ops in (("relu", ("x",)), ("dual", ("x", "x_ds"))):
        for op in ops:
            assert_same(forward(site, kind, {op: offset}), fwds[kind], f"{kind} forward with {op} at {offset} mod 16")
