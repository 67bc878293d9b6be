"""The activation and residual batch-norm sites (norm_act.cuh, norm_res.cuh) through the C-ABI, against torch's
functional chain, bit for bit.

b200c_bn_forward_act / b200c_bn_backward_act (ReLU6, SiLU, Hardswish) and b200c_bn_forward_res / b200c_bn_backward_res
(plain, `+ identity`, and stochastic depth then `+ identity`) run on one scratch buffer with guard bytes past
b200c_bn_scratch_bytes(c): after every call nothing past it is written and every semaphore is back at zero.  Every
output is filled with all-ones bits (a NaN) before its call, so an element no thread writes shows: y, the saved
statistics, g (the batch norm's output gradient, which the backward reduce writes for the elementwise kernel), dx,
dweight and dbias.  The running statistics and num_batches_tracked are checked as well.

- Merged grids of 128 and 8 rows of blocks, C = 16 to 131072, with stochastic depth over one sample, one row per sample
  and many samples; the saved statistics are also held to a float64 bound.
- Each operand a launcher checks before it takes its vector kernels, moved off the 16-byte grid alone (2 and 8 bytes
  past a boundary), must keep the all-aligned call's bits; the eval sites (b200c_bn_infer_act, b200c_bn_infer_res)
  with fp32 and bf16 parameters too.
- Two streams, each with its own scratch, with their kernels overlapping."""
import pytest
import torch
import torch.nn.functional as F

import test_gpu_fused_norm as L
from ant_ray_b200 import _native as N
from gpu_common import bn_launch_config
from test_gpu_bn_ring import ALONE_SHAPES, assert_same, nan_filled, p, placed
from test_gpu_fused_act import CODES, PARAMS

pytestmark = pytest.mark.gpu

RES = ("res_plain", "res_add", "res_drop")
KINDS = list(CODES) + list(RES)
ACT_FWD = {"relu6": lambda t: F.hardtanh(t, 0.0, 6.0), "silu": F.silu, "hardswish": F.hardswish}
ACT_BWD = {"relu6": lambda dy, t: torch.ops.aten.hardtanh_backward(dy, t, 0.0, 6.0), "silu": torch.ops.aten.silu_backward,
           "hardswish": torch.ops.aten.hardswish_backward}
SURVIVAL = 0.8
NBT = 5


def row_noise(samples, g):
    """Stochastic depth's per-sample noise as fused_norm._row_noise builds it (bernoulli_ of the survival rate, then
    div_ by it, in bf16), with sample 0 kept and, where there are two or more samples, the last one dropped."""
    noise = torch.empty(samples, dtype=torch.bfloat16, device="cuda").bernoulli_(SURVIVAL, generator=g).div_(SURVIVAL)
    noise[0] = torch.ones((), dtype=torch.bfloat16, device="cuda").div_(SURVIVAL)
    if samples > 1:
        noise[-1] = 0
    return noise


class Site:
    """Seeded inputs of one (M, C) site: x, dy and the batch norm of test_gpu_fused_norm.site_inputs, an identity,
    and stochastic depth's noise over M / rows_per_sample samples."""

    def __init__(self, m, c, rows_per_sample, seed):
        assert m % rows_per_sample == 0
        self.m, self.c, self.rows_per_sample = m, c, rows_per_sample
        self.x, self.dy, self.w, self.b, self.rm, self.rv = L.site_inputs(m, c, seed)
        g = torch.Generator(device="cuda").manual_seed(seed + 1)
        self.identity = (torch.randn(m, c, device="cuda", generator=g) - 0.2).to(torch.bfloat16)
        self.noise = row_noise(m // rows_per_sample, g)

    def noise_rows(self):
        """The noise of each row, [M, 1, 1, 1], as stochastic depth's [N, 1, 1, 1] noise broadcasts over H * W rows."""
        return self.noise.repeat_interleave(self.rows_per_sample).view(self.m, 1, 1, 1)


def torch_chain(site, kind):
    """torch's functional chain of one training site on x.view(m, c, 1, 1) (NCHW strides with stride(1) == 1: torch's
    channels-last kernels): native_batch_norm, then the activation, or stochastic depth's bf16 mul and the bf16 add of
    the identity; their backward; native_batch_norm_backward.  "g" is the batch norm's output gradient."""
    m, c = site.m, site.c
    x4, dy4 = site.x.view(m, c, 1, 1), site.dy.view(m, c, 1, 1)
    rm, rv = site.rm.clone(), site.rv.clone()
    t, mean, invstd = torch.native_batch_norm(x4, site.w, site.b, rm, rv, True, 0.1, 1e-5)
    if kind in CODES:
        y, g = ACT_FWD[kind](t), ACT_BWD[kind](dy4, t)
    else:
        y, g = t, dy4
        if kind == "res_drop":
            noise = site.noise_rows()
            y, g = y * noise, dy4 * noise
        if kind != "res_plain":
            y = y + site.identity.view(m, c, 1, 1)
    dx, dw, db = torch.ops.aten.native_batch_norm_backward(g, x4, site.w, rm, rv, mean, invstd, True, 1e-5, [True, True, True])
    # g before dx: an unwritten g shows as itself rather than as the dx computed from it
    return {"y": y.view(m, c), "mean": mean, "invstd": invstd, "running_mean": rm, "running_var": rv, "g": g.view(m, c),
            "dx": dx.view(m, c), "dweight": dw, "dbias": db}


def native_site(site, kind, scratch, stream=None, place=None):
    """NaN-filled outputs of one training site, allocated on the current stream, and its two C-ABI calls, each
    enqueued on `stream` (the current one by default) when called, with the operands named in `place` (name -> byte
    offset) moved off the 16-byte grid.  Returns (forward, backward, outputs); g is None where it is dy itself."""
    place = place or {}
    lib, m, c = N.load(), site.m, site.c
    on = lambda k, t: placed(t, place.get(k, 0))  # noqa: E731
    x, dy = on("x", site.x), on("dy", site.dy)
    identity = on("identity", site.identity) if kind in ("res_add", "res_drop") else None
    noise = site.noise if kind == "res_drop" else None
    f32 = torch.float32
    out = {"y": nan_filled((m, c), place.get("y", 0)), "mean": nan_filled(c, dtype=f32), "invstd": nan_filled(c, dtype=f32),
           "running_mean": site.rm.clone(), "running_var": site.rv.clone(),
           "num_batches_tracked": torch.full((), NBT, dtype=torch.int64, device="cuda"),
           "g": nan_filled((m, c), place.get("g", 0)) if kind in CODES or noise is not None else None,
           "dx": nan_filled((m, c), place.get("dx", 0)), "dweight": nan_filled(c, dtype=f32), "dbias": nan_filled(c, dtype=f32)}
    o = {k: p(v) for k, v in out.items()}
    stats = (o["running_mean"], o["running_var"], o["num_batches_tracked"], o["mean"], o["invstd"])

    def forward():
        s = (stream or torch.cuda.current_stream()).cuda_stream
        if kind in CODES:
            N.check(lib.b200c_bn_forward_act(p(x), o["y"], p(site.w), p(site.b), *stats, CODES[kind], m, c, 0.1, 1e-5, p(scratch), s))
        else:
            N.check(lib.b200c_bn_forward_res(p(x), p(identity), p(noise), site.rows_per_sample, o["y"], p(site.w), p(site.b), *stats, m,
                                             c, 0.1, 1e-5, p(scratch), s))

    def backward():
        s = (stream or torch.cuda.current_stream()).cuda_stream
        if kind in CODES:
            N.check(lib.b200c_bn_backward_act(p(dy), p(x), o["g"], o["dx"], p(site.w), p(site.b), o["mean"], o["invstd"], o["dweight"],
                                              o["dbias"], CODES[kind], m, c, p(scratch), s))
        else:
            N.check(lib.b200c_bn_backward_res(p(dy), p(noise), site.rows_per_sample, p(x), o["g"], o["dx"], p(site.w), o["mean"],
                                              o["invstd"], o["dweight"], o["dbias"], m, c, p(scratch), s))

    return forward, backward, out


def run(site, kind, scratch, place=None):
    """One training site on the current stream, the guarded scratch checked after each call."""
    buf, need = scratch
    forward, backward, out = native_site(site, kind, buf, place=place)
    forward()
    torch.cuda.synchronize()
    L.check_scratch(buf, need)
    backward()
    torch.cuda.synchronize()
    L.check_scratch(buf, need)
    return out


def against_torch(got, want, where):
    """Every output the native site wrote against torch's chain; num_batches_tracked is one past where it started."""
    assert int(got["num_batches_tracked"]) == NBT + 1, where
    assert_same({k: got[k] for k in want if got[k] is not None}, {k: v for k, v in want.items() if got[k] is not None}, where)


# (M, C, rows per sample): the shapes of test_gpu_fused_norm's scratch test, stochastic depth over 256 samples, 512
# samples, one row per sample and one sample
MERGED = [(65536, 16, 256), (32768, 100, 64), (32768, 2048, 1), (2048, 131072, 2048)]


@pytest.mark.parametrize("m,c,rows_per_sample", MERGED)
def test_act_and_res_sites_at_merged_grids(m, c, rows_per_sample):
    assert bn_launch_config(m, c).grid_y == (8 if c == 131072 else 128)
    site = Site(m, c, rows_per_sample, c)
    scratch = L.scratch_with_guard(c)
    for kind in KINDS:
        got = run(site, kind, scratch)
        against_torch(got, torch_chain(site, kind), kind)
        L.check_stats_against_float64(site.x, got)


# ---- each launcher operand off the 16-byte grid -----------------------------------------------------------------
# Each launcher takes its vector kernels when C % 8 == 0 and every operand it checks is on the 16-byte grid:
# forward_act x (statistics), x and y (transform); backward_act x, dx and g (elementwise; the reduce is scalar);
# forward_res x, y and the identity; backward_res with noise x, dx and g, without noise x and dy (reduce ring), x, dx
# and dy (elementwise).  An operand listed for a kind is moved in both of its calls.
OPERANDS = {**{a: ("x", "y", "dx", "g") for a in CODES}, "res_plain": ("x", "y", "dy", "dx"),
            "res_add": ("x", "y", "identity", "dy", "dx"), "res_drop": ("x", "y", "identity", "dx", "g")}
INFER_OPERANDS = {**{a: ("x", "y") for a in CODES}, "res_plain": ("x", "y"), "res_add": ("x", "y", "identity")}
# rows per sample of stochastic depth at test_gpu_bn_ring.ALONE_SHAPES: one sample, 99 and 11 samples
ALONE = [(c, m, r) for (c, m), r in zip(ALONE_SHAPES, (97, 331, 163))]


def eval_bn(c, params):
    return L.make_bn(c, c + 1, eps=1e-3).eval().to(PARAMS[params])


def infer(site, kind, bn, place=None):
    """b200c_bn_infer_act (an activation) or b200c_bn_infer_res (res_plain, res_add) into a NaN-filled y."""
    place = place or {}
    lib, m, c = N.load(), site.m, site.c
    x, y = placed(site.x, place.get("x", 0)), nan_filled((m, c), place.get("y", 0))
    params = (p(bn.weight), p(bn.bias), p(bn.running_mean), p(bn.running_var), int(bn.weight.dtype == torch.bfloat16), bn.eps)
    s = torch.cuda.current_stream().cuda_stream
    if kind in CODES:
        N.check(lib.b200c_bn_infer_act(p(x), p(y), *params, CODES[kind], m, c, s))
    else:
        identity = placed(site.identity, place.get("identity", 0)) if kind == "res_add" else None
        N.check(lib.b200c_bn_infer_res(p(x), p(identity), p(y), *params, m, c, s))
    torch.cuda.synchronize()
    return {"y": y}


def torch_eval(site, kind, bn):
    """The eval-mode module on x.view(m, c, 1, 1), then the activation or `+ identity`."""
    m, c = site.m, site.c
    x4 = site.x.view(m, c, 1, 1)
    assert torch._C._select_batch_norm_backend(x4, bn.weight, bn.bias, bn.running_mean, bn.running_var, False,
                                               bn.eps) == torch._C._BatchNormBackend.Native
    with torch.no_grad():
        t = bn(x4)
        y = ACT_FWD[kind](t) if kind in CODES else t if kind == "res_plain" else site.identity.view(m, c, 1, 1) + t
    return {"y": y.view(m, c)}


@pytest.mark.parametrize("offset", [2, 8])
@pytest.mark.parametrize("c,m,rows_per_sample", ALONE)
def test_each_launcher_operand_off_the_grid_alone(c, m, rows_per_sample, offset):
    """Every site once with all operands on the 16-byte grid (the vector kernels), compared with torch, then with each
    operand its launchers check alone 2 or 8 bytes past a 16-byte boundary (the scalar kernels): every output keeps
    the aligned call's bits."""
    assert c % 8 == 0
    site = Site(m, c, rows_per_sample, m + c)
    scratch = L.scratch_with_guard(c)
    for kind in KINDS:
        want = run(site, kind, scratch)
        against_torch(want, torch_chain(site, kind), f"{kind} against torch")
        for op in OPERANDS[kind]:
            assert_same(run(site, kind, scratch, {op: offset}), want, f"{kind} with {op} at {offset} mod 16")
    for params in PARAMS:
        bn = eval_bn(c, params)
        for kind, ops in INFER_OPERANDS.items():
            want = infer(site, kind, bn)
            assert_same(want, torch_eval(site, kind, bn), f"eval {kind} ({params}) against torch")
            for op in ops:
                assert_same(infer(site, kind, bn, {op: offset}), want, f"eval {kind} ({params}) with {op} at {offset} mod 16")


def test_two_streams_with_their_own_scratch():
    sites = [(Site(32768, 100, 1, 1), "silu"), (Site(32768, 2048, 64, 2), "res_drop")]
    wants = [torch_chain(site, kind) for site, kind in sites]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    scratches = [L.scratch_with_guard(site.c) for site, _ in sites]
    runs = [native_site(site, kind, buf, st) for (site, kind), (buf, _), st in zip(sites, scratches, streams)]
    torch.cuda.synchronize()
    for _ in range(3):   # interleaved enqueues, so the two sites' kernels overlap on the device
        for forward, backward, _ in runs:
            forward()
            backward()
    torch.cuda.synchronize()
    for (_, _, got), want, (buf, need), (_, kind) in zip(runs, wants, scratches, sites):
        L.check_scratch(buf, need)
        assert int(got["num_batches_tracked"]) == NBT + 3, kind
        keys = ("y", "mean", "invstd", "dx", "g", "dweight", "dbias")
        assert_same({k: got[k] for k in keys}, {k: want[k] for k in keys}, kind)
