"""The squeeze-and-excitation kernels (se_kernels.cuh) and the concatenation batch-norm site (norm_cat.cuh) through the
C-ABI, against torch's own ops, bit for bit.

Squeeze-and-excitation: b200c_se_pool, b200c_se_scale, b200c_se_backward_reduce and b200c_se_backward_elemt against
DESIGN.md §12's references (x.mean((-1, -2)), s * x, (dy * x).sum_to_size(n, c, 1, 1), dy * s + gp / HW), at every
shape of test_fused_se_cpu.SE_REGIME_SHAPES with x at its address and at one row per sample:
- every output is filled with all-ones bits (a NaN) before its call, so an element no thread writes shows;
- one scratch of exactly b200c_se_scratch_bytes(n, c, hw) is followed by guard bytes: after every call the guard is
  intact and the semaphores are zero;
- pooled and ds sit 0, 2, 4 and 6 bytes past an 8-byte boundary (the reducing kernels store each output alone);
- x, dy, s, gp, y and dx are each moved 2 and 8 bytes past a 16-byte boundary alone: every output keeps the aligned
  call's bits (pooled wherever x's address leaves torch's vector width as it was) and torch's;
- pooled is held to a float64 mean within a bound derived from the launch's add-chain depth;
- one scratch serves sites of every launch kind in turn on one stream, and two streams run sites on their own scratch.
The launches follow from the device's own multiProcessorCount and maxThreadsPerMultiProcessor, and the shapes must
reach, for each vector width, a launch without a row split, one split across warps and one split across blocks.

Concatenation: b200c_bn_forward_cat, b200c_bn_backward_cat and b200c_bn_infer_cat at 64 segments (the most the C-ABI
takes) of 8 channels, with a 2048-channel segment first, and with it last (the segment search ends at the table's
last entry).  The segments are 16-byte-aligned views into one NaN-filled buffer, laid out in reverse table order with
gaps between them, so table order and memory order differ.  y, dx, the saved statistics, dweight and dbias are filled
with NaN and the mask with 0xA5 before the calls; against `relu(bn(torch.cat(segs, 1)))`, bit for bit: y, the mask,
the running statistics, num_batches_tracked, every segment's gradient, dweight and dbias, the saved statistics against
torch.native_batch_norm's and a float64 bound, the guard and semaphores after each call; eval with fp32 and bf16
parameters; and two streams, each with its own scratch."""
import ctypes
import math

import pytest
import torch

from ant_ray_b200 import _native as N
from gpu_common import same_bits
from test_fused_se_cpu import SE_REGIME_SHAPES, se_reduce_config
from test_gpu_bn_limits import check_mask, same
from test_gpu_bn_ring import assert_same, nan_filled, p, placed
from test_gpu_fused_cat import run as eager_cat
from test_gpu_fused_norm import GUARD, check_scratch, check_stats_against_float64, make_bn, scratch_with_guard

pytestmark = pytest.mark.gpu

U = 2.0 ** -24   # fp32 unit roundoff


# ---- squeeze-and-excitation ---------------------------------------------------------------------------------------
# (n, c, h, w, x's address mod 16): every regime shape, then one row per sample
SE_SHAPES = [(*shape, addr) for shape, addr in SE_REGIME_SHAPES] + [(8, 64, 1, 1, 0), (5, 3, 1, 1, 0), (4, 6, 1, 1, 0)]
SE_OPERANDS = ("x", "dy", "s", "gp", "y", "dx")


def device_launch(n, c, hw, addr=0):
    """se_reduce_config on the current device's multiProcessorCount and maxThreadsPerMultiProcessor."""
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    return se_reduce_config(n, c, hw, addr, props.multi_processor_count, props.max_threads_per_multi_processor)


class SeSite:
    """Seeded bf16 operands of one site: x and dy as [n * hw, c] rows, s and gp as [n, c]."""

    def __init__(self, n, c, h, w, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.n, self.c, self.h, self.w, self.hw = n, c, h, w, h * w
        gauss = lambda rows, scale, shift: (torch.randn(rows, c, device="cuda", generator=g) * scale + shift).to(torch.bfloat16)  # noqa: E731
        self.x, self.dy = gauss(n * h * w, 2.0, 0.5), gauss(n * h * w, 1.0, 0.0)
        self.s = torch.rand(n, c, device="cuda", generator=g).to(torch.bfloat16)
        self.gp = gauss(n, 0.5, 0.0)

    def nchw(self, rows):
        """[n * hw, c] rows as the channels-last [n, c, h, w] tensor they are."""
        return rows.view(self.n, self.h, self.w, self.c).permute(0, 3, 1, 2)


def torch_se(site, x):
    """torch's ops on x (at its own address: the mean's order follows it) and the site's other operands."""
    n, c, h, w = site.n, site.c, site.h, site.w
    x4, dy4 = site.nchw(x), site.nchw(site.dy)
    s4, gp4 = site.s.view(n, c, 1, 1), site.gp.view(n, c, 1, 1)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(n * h * w, c)  # noqa: E731
    return {"pooled": x4.mean((-1, -2)), "y": rows(s4 * x4), "ds": (dy4 * x4).sum_to_size(n, c, 1, 1).view(n, c),
            "dx": rows((dy4 * s4).add_(gp4.expand(n, c, h, w) / site.hw))}


def se_scratch(*shapes):
    """One zeroed scratch of the largest b200c_se_scratch_bytes of `shapes` ((n, c, hw)), then GUARD bytes of 0xA5."""
    need = max(int(N.load().b200c_se_scratch_bytes(n, c, hw)) for n, c, hw in shapes)
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    return buf, need


def se_site(site, scratch, place=None, stream=None):
    """NaN-filled pooled, y, ds and dx, and the four C-ABI calls of one site, each enqueued on `stream` (the current one
    by default) when called, with the operands and outputs named in `place` (name -> byte offset) moved off the
    16-byte grid.  Returns (calls, outputs, x as placed)."""
    place = place or {}
    lib, (buf, need) = N.load(), scratch
    n, c, hw = site.n, site.c, site.hw
    x, dy, s, gp = (placed(getattr(site, k), place.get(k, 0)) for k in ("x", "dy", "s", "gp"))
    out = {"pooled": nan_filled((n, c), place.get("pooled", 0)), "y": nan_filled((n * hw, c), place.get("y", 0)),
           "ds": nan_filled((n, c), place.get("ds", 0)), "dx": nan_filled((n * hw, c), place.get("dx", 0))}
    o = {k: p(v) for k, v in out.items()}
    st = lambda: (stream or torch.cuda.current_stream()).cuda_stream  # noqa: E731
    calls = [lambda: N.check(lib.b200c_se_pool(p(x), o["pooled"], n, c, hw, p(buf), need, st())),
             lambda: N.check(lib.b200c_se_scale(p(x), p(s), o["y"], n, c, hw, st())),
             lambda: N.check(lib.b200c_se_backward_reduce(p(dy), p(x), o["ds"], n, c, hw, p(buf), need, st())),
             lambda: N.check(lib.b200c_se_backward_elemt(p(dy), p(s), p(gp), o["dx"], n, c, hw, st()))]
    return calls, out, x


def run_se(site, scratch, place=None):
    """The four calls on the current stream, the guarded scratch checked after each.  Returns (outputs, x as placed)."""
    calls, out, x = se_site(site, scratch, place)
    for call in calls:
        call()
        torch.cuda.synchronize()
        check_scratch(*scratch)
    return out, x


def check_pooled_against_float64(site, x, pooled):
    """pooled against the float64 mean.  The fp32 sum of an output is a chain of at most ceil(rows per thread / 4)
    adds into one of the four accumulators, 3 to combine them, 2 log2(block_y) in the trees and ceil(ctas / block_y) in
    the staged walk; the factor and the product add 3 roundings more.  So |sum - exact| <= depth u sum|x|, and the bf16
    rounding adds half an ulp (at most |value| 2^-8)."""
    n, c, hw = site.n, site.c, site.hw
    l = device_launch(n, c, hw, x.data_ptr() % 16)
    rows = math.ceil(hw / (l.block_y * l.ctas)) if l.split else hw
    depth = math.ceil(rows / 4) + 3 + 2 * math.log2(l.block_y) + math.ceil(l.ctas / l.block_y) + 3
    x64 = x.view(n, hw, c).double()
    mean64, abs_mean = x64.mean(1), x64.abs().mean(1)
    got = pooled.double()
    bound = depth * U * abs_mean + torch.maximum(got.abs(), mean64.abs()) * 2.0 ** -8
    assert bool(((got - mean64).abs() <= bound).all()), (site.n, site.c, site.hw, float(((got - mean64).abs() / bound).max()))


def test_se_shapes_reach_every_launch_kind_on_this_device():
    kinds = {}
    for n, c, h, w, addr in SE_SHAPES:
        if h * w == 1:
            continue
        for a in (addr, 0):   # the pool at x's address, the backward reduce as torch's fresh product tensor
            l = device_launch(n, c, h * w, a)
            kinds.setdefault(l.vec, set()).add((l.split, l.ctas > 1))
            if l.ctas > 1:
                assert l.grid_x <= 4096, (n, c, h, w, l)
    for vec in (1, 2, 4):
        assert kinds.get(vec) == {(False, False), (True, False), (True, True)}, (vec, kinds.get(vec))


@pytest.mark.parametrize("n,c,h,w,addr", SE_SHAPES)
def test_se_calls_match_torch_at_every_placement(n, c, h, w, addr):
    site = SeSite(n, c, h, w, n * 1000 + c * 10 + h)
    hw = h * w
    scratch = se_scratch((n, c, hw))
    base = {"x": addr}
    want, x = run_se(site, scratch, base)
    assert_same(want, torch_se(site, x), f"x at {addr} mod 16 against torch")
    check_pooled_against_float64(site, x, want["pooled"])
    variants = [{out: off} for out in ("pooled", "ds") for off in (2, 4, 6)]
    variants += [{op: off} for op in SE_OPERANDS for off in (2, 8)]
    for v in variants:
        place = {**base, **v}
        got, xv = run_se(site, scratch, place)
        ref = torch_se(site, xv) if "x" in v else want
        assert_same(got, ref, f"{place} against torch")
        same_launch = device_launch(n, c, hw, place["x"]) == device_launch(n, c, hw, addr)
        for k in ("y", "ds", "dx") + (("pooled",) if same_launch else ()):
            assert same_bits(got[k], want[k]), f"{k} with {place} differs from the call at {base}"
        if "x" in v:
            check_pooled_against_float64(site, xv, got["pooled"])


def test_one_se_scratch_serves_every_site_on_a_stream():
    # split across blocks (196 and 49 blocks per output), then a narrow block, one row per sample, a split across
    # warps, and the first site again, all on one buffer of the largest size
    shapes = [(1, 32, 224, 224), (2, 6, 9, 9), (8, 64, 1, 1), (5, 3, 1, 1), (4, 100, 16, 16), (4, 100, 56, 56), (1, 32, 224, 224)]
    sites = [SeSite(*shape, i) for i, shape in enumerate(shapes)]
    scratch = se_scratch(*[(s.n, s.c, s.hw) for s in sites])
    assert device_launch(1, 32, 224 * 224).ctas > 1 and device_launch(4, 100, 56 * 56).ctas > 1
    for site, shape in zip(sites, shapes):
        got, x = run_se(site, scratch)
        assert_same(got, torch_se(site, x), f"{shape} on the shared scratch")


def test_se_sites_on_two_streams_with_their_own_scratch():
    sites = [SeSite(1, 32, 224, 224, 21), SeSite(8, 64, 56, 56, 22)]
    wants = [torch_se(site, site.x) for site in sites]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    scratches = [se_scratch((site.n, site.c, site.hw)) for site in sites]
    runs = [se_site(site, scratch, stream=st) for site, scratch, st in zip(sites, scratches, streams)]
    torch.cuda.synchronize()
    for _ in range(3):   # interleaved enqueues, so the two sites' kernels overlap on the device
        for i in range(4):
            for calls, _, _ in runs:
                calls[i]()
    torch.cuda.synchronize()
    for (_, got, _), want, scratch, site in zip(runs, wants, scratches, sites):
        check_scratch(*scratch)
        assert_same(got, want, (site.n, site.c, site.hw))


# ---- concatenation -------------------------------------------------------------------------------------------------
CAT_TABLES = {"64x8": (8,) * 64, "wide_first": (2048,) + (8,) * 63, "wide_last": (8,) * 63 + (2048,)}
CAT_NHW = (4, 14, 14)
NBT = 5


def cat_segments(m, chans, seed):
    """Seeded bf16 segments of m rows: 16-byte-aligned views into one NaN-filled buffer, laid out in reverse table order
    with gaps of 16 to 48 bytes between them."""
    gaps = [8 * (1 + i % 3) for i in range(len(chans))]   # elements
    buf = nan_filled((sum(m * k for k in chans) + sum(gaps),))
    segs, off = [None] * len(chans), 0
    for i in reversed(range(len(chans))):
        off += gaps[i]
        segs[i] = buf[off:off + m * chans[i]].view(m, chans[i])
        off += m * chans[i]
    g = torch.Generator(device="cuda").manual_seed(seed)
    for t in segs:
        t.copy_(torch.randn(t.shape, device="cuda", generator=g) * 2.0 + 0.5)
        assert t.data_ptr() % 16 == 0
    assert [t.data_ptr() for t in segs] == sorted((t.data_ptr() for t in segs), reverse=True)
    return segs


def cat_table(segs, chans):
    return (ctypes.c_void_p * len(segs))(*(t.data_ptr() for t in segs)), (ctypes.c_int * len(chans))(*chans), len(chans)


def cat_site(segs, chans, dy, bn, scratch, stream=None):
    """NaN-filled outputs (the mask 0xA5) of one training site and its two C-ABI calls, each enqueued on `stream` (the
    current one by default) when called.  Returns (forward, backward, outputs)."""
    lib, (buf, need) = N.load(), scratch
    m, c = dy.shape
    f32 = torch.float32
    out = {"y": nan_filled((m, c)), "mask": torch.full((m * c // 8,), 0xA5, dtype=torch.uint8, device="cuda"),
           "mean": nan_filled(c, dtype=f32), "invstd": nan_filled(c, dtype=f32), "running_mean": bn.running_mean.clone(),
           "running_var": bn.running_var.clone(), "num_batches_tracked": bn.num_batches_tracked.clone(),
           "dx": nan_filled((m, c)), "dweight": nan_filled(c, dtype=f32), "dbias": nan_filled(c, dtype=f32)}
    o = {k: p(v) for k, v in out.items()}
    table = cat_table(segs, chans)
    w, b = p(bn.weight), p(bn.bias)
    st = lambda: (stream or torch.cuda.current_stream()).cuda_stream  # noqa: E731

    def forward():
        N.check(lib.b200c_bn_forward_cat(*table, o["y"], o["mask"], w, b, o["running_mean"], o["running_var"], o["num_batches_tracked"],
                                         o["mean"], o["invstd"], m, c, 0.1, 1e-5, p(buf), st()))

    def backward():
        N.check(lib.b200c_bn_backward_cat(p(dy), o["mask"], *table, o["dx"], w, o["mean"], o["invstd"], o["dweight"], o["dbias"], m, c,
                                          p(buf), st()))

    return forward, backward, out


class CatSite:
    """Seeded segments of one table at CAT_NHW, an output gradient, a batch norm, and torch's results for them:
    `relu(bn(torch.cat(segs, 1)))` and its backward on channels-last tensors, as [m, c] rows."""

    def __init__(self, chans, seed):
        n, h, w = CAT_NHW
        self.m, self.c, self.chans = n * h * w, sum(chans), chans
        self.segs = cat_segments(self.m, chans, seed)
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.dy = torch.randn(self.m, self.c, device="cuda", generator=g).to(torch.bfloat16)
        self.bn = make_bn(self.c, seed, nbt=NBT)
        nchw = lambda t: t.view(n, h, w, t.shape[1]).permute(0, 3, 1, 2)  # noqa: E731
        rows = lambda t: t.permute(0, 2, 3, 1).reshape(self.m, t.shape[1])  # noqa: E731
        eager = eager_cat(make_bn(self.c, seed, nbt=NBT), [nchw(t) for t in self.segs], nchw(self.dy), False)
        self.x = torch.cat(self.segs, 1)
        _, mean, invstd = torch.native_batch_norm(nchw(self.x), self.bn.weight, self.bn.bias, self.bn.running_mean.clone(),
                                                  self.bn.running_var.clone(), True, 0.1, 1e-5)
        self.want = {"y": rows(eager["y"]), "mean": mean, "invstd": invstd, "running_mean": eager["running_mean"],
                     "running_var": eager["running_var"], "num_batches_tracked": eager["num_batches_tracked"],
                     "dweight": eager["dweight"], "dbias": eager["dbias"]}
        self.grads = [rows(eager[f"grad{i}"]) for i in range(len(chans))]

    def check(self, got, where, keys=None):
        check_mask(got["mask"], got["y"])
        for k in keys or self.want:
            same(got[k], self.want[k], f"{where}: {k}")
        c0 = 0
        for i, k in enumerate(self.chans):
            same(got["dx"][:, c0:c0 + k], self.grads[i], f"{where}: gradient of segment {i}")
            c0 += k


@pytest.mark.parametrize("table", sorted(CAT_TABLES))
def test_64_segments_through_the_c_abi_match_torch(table):
    chans = CAT_TABLES[table]
    site = CatSite(chans, len(chans) + chans[0])
    scratch = scratch_with_guard(site.c)
    forward, backward, got = cat_site(site.segs, chans, site.dy, site.bn, scratch)
    forward()
    torch.cuda.synchronize()
    check_scratch(*scratch)
    backward()
    torch.cuda.synchronize()
    check_scratch(*scratch)
    assert int(got["num_batches_tracked"]) == NBT + 1
    site.check(got, table)
    check_stats_against_float64(site.x, got)

    n, h, w = CAT_NHW
    lib = N.load()
    for dtype in (torch.float32, torch.bfloat16):
        bn = make_bn(site.c, 3, eps=1e-3).eval().to(dtype)
        y = nan_filled((site.m, site.c))
        N.check(lib.b200c_bn_infer_cat(*cat_table(site.segs, chans), p(y), p(bn.weight), p(bn.bias), p(bn.running_mean),
                                       p(bn.running_var), int(dtype == torch.bfloat16), bn.eps, site.m, site.c,
                                       torch.cuda.current_stream().cuda_stream))
        with torch.no_grad():
            want = torch.relu_(bn(site.x.view(n, h, w, site.c).permute(0, 3, 1, 2)))
        same(y, want.permute(0, 2, 3, 1).reshape(site.m, site.c), f"{table}: eval y ({dtype})")


def test_cat_sites_on_two_streams_with_their_own_scratch():
    sites = [CatSite(CAT_TABLES["wide_first"], 31), CatSite(CAT_TABLES["wide_last"], 32)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    scratches = [scratch_with_guard(site.c) for site in sites]
    runs = [cat_site(site.segs, site.chans, site.dy, site.bn, scratch, st) for site, scratch, st in zip(sites, scratches, streams)]
    torch.cuda.synchronize()
    for _ in range(3):   # interleaved enqueues, so the two sites' kernels overlap on the device
        for forward, backward, _ in runs:
            forward()
            backward()
    torch.cuda.synchronize()
    for (_, _, got), site, scratch in zip(runs, sites, scratches):
        check_scratch(*scratch)
        assert int(got["num_batches_tracked"]) == NBT + 3
        site.check(got, site.chans[0], keys=("y", "mean", "invstd", "dweight", "dbias"))
