"""Batch norm followed by a residual add, with or without stochastic depth (fused_norm.bn_res, norm_res.cuh), against
eager torch, bit for bit.

Training sites, four eager references: the batch norm alone ("plain"), `identity + bn(x)` as MobileNetV2 adds
("add"), `f = bn(x); f += identity` as MobileNetV3 adds ("iadd"), and torchvision's StochasticDepth(p, "row") then
`+=` as EfficientNet's MBConv runs it ("drop"), reseeded identically on both sides.  y, the running statistics,
num_batches_tracked, dx, d(identity), dweight and dbias must have the same bits (a NaN matching a NaN), at every
projection-site shape of mobilenet_v2, mobilenet_v3_large and efficientnet_b0 at 224 x 224 (batch 256 and 32), every
launch regime, C = 100, misaligned x, identity and dy (the scalar kernels), value edges of x and dy, every row dropped
and none, survival rates whose bf16 reciprocal is inexact, Inf and NaN gradients in dropped rows, a range of momentum
and eps, and an NCHW dy.  Eval sites: y, with fp32 and bf16 parameters, with and without an identity.  KERNELS names
every `b200c::bn_res` kernel with the case that launches it; the profiler traces and the whole models are in
test_gpu_zz_res_models.py."""
import copy
import json
import os
import re
import shutil
import subprocess

import pytest
import torch

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values, same_bits
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn, misaligned

StochasticDepth = pytest.importorskip("torchvision.ops").StochasticDepth

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")
KINDS = ["plain", "add", "iadd", "drop"]
PARAMS = {"fp32": torch.float32, "bf16": torch.bfloat16}
# (C, H, W) of every projection batch norm of mobilenet_v2, mobilenet_v3_large and efficientnet_b0 at 224 x 224
MODEL_SHAPES = [(16, 112, 112), (24, 56, 56), (32, 28, 28), (40, 28, 28), (64, 14, 14), (80, 14, 14), (96, 14, 14),
                (112, 14, 14), (160, 7, 7), (192, 7, 7), (320, 7, 7)]


def nhwc(t):
    """A bf16 copy of `t` with NHWC strides, stride(1) == 1 included (C = 1)."""
    n, c, h, w = t.shape
    return torch.empty(n, h, w, c, dtype=torch.bfloat16, device=t.device).permute(0, 3, 1, 2).copy_(t)


def gauss_inputs(n, c, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g) * 2 + 0.5)
    identity = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g) - 0.2)
    dy = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g))
    return x, identity, dy


def run(kind, bn, x, identity, dy, fused, p=0.2, seed=0, misalign=()):
    x = (misaligned(x) if "x" in misalign else x.clone()).requires_grad_()
    if kind == "plain":
        identity = None
    else:
        identity = (misaligned(identity) if "identity" in misalign else identity.clone()).requires_grad_()
    sd = StochasticDepth(p, "row")
    if fused:
        noise = None
        if kind == "drop":
            torch.manual_seed(seed)
            noise = fused_norm._row_noise(sd, x)
        y = fused_norm.bn_res(bn, x, identity, noise)
    elif kind == "plain":
        y = bn(x)
    elif kind == "add":
        y = identity + bn(x)
    else:
        y = bn(x)
        if kind == "drop":
            torch.manual_seed(seed)
            y = sd(y)
        y += identity
    y.backward(misaligned(dy) if "dy" in misalign else dy)
    return {"y": y.detach(), "dx": x.grad, "d_identity": identity.grad if identity is not None else None, "dweight": bn.weight.grad,
            "dbias": bn.bias.grad, "running_mean": bn.running_mean, "running_var": bn.running_var,
            "num_batches_tracked": bn.num_batches_tracked}


def check_site(kind, x, identity, dy, bn_setup=None, launches=4, seed=0, p=0.2, misalign=(), **bn_args):
    """One training site through bn_res and through eager torch's ops; every result must have the same bits (a NaN
    matching a NaN), and the fused site must make `launches` native launches."""
    c = x.shape[1]
    ref_bn = make_bn(c, seed, **bn_args).cuda()
    if bn_setup is not None:
        bn_setup(ref_bn)
    fused_bn = copy.deepcopy(ref_bn)
    want = run(kind, ref_bn, x, identity, dy, False, p, seed, misalign)
    before = N.launch_count()
    got = run(kind, fused_bn, x, identity, dy, True, p, seed, misalign)
    torch.cuda.synchronize()
    assert N.launch_count() - before == launches
    for k in want:
        if want[k] is None:
            assert got[k] is None, k
        else:
            assert_same_values(got[k], want[k], k)
    assert got["y"].is_contiguous(memory_format=CL) and got["dx"].is_contiguous(memory_format=CL)
    return want, got


def check_gauss_site(kind, n, c, h, w, seed=None, **kw):
    x, identity, dy = gauss_inputs(n, c, h, w, n * 7 + c * 13 + h)
    return check_site(kind, x, identity, dy, seed=c if seed is None else seed, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [256, 32])
@pytest.mark.parametrize("c,h,w", MODEL_SHAPES)
@pytest.mark.parametrize("kind", KINDS)
def test_model_site_shapes(kind, c, h, w, n):
    check_gauss_site(kind, n, c, h, w)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(BN_REGIME_SHAPES), ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", KINDS)
def test_launch_regimes(kind, shape):
    check_gauss_site(kind, *shape, p=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("misalign", [(), ("x",), ("identity",), ("dy",)], ids=["c100", "x", "identity", "dy"])
@pytest.mark.parametrize("kind", KINDS)
def test_scalar_kernels(kind, misalign):
    if misalign:
        if kind == "plain" and misalign == ("identity",):
            pytest.skip("no identity")
        check_gauss_site(kind, 8, 64, 16, 16, misalign=misalign)   # an operand off the 16-byte grid
    else:
        check_gauss_site(kind, 3, 100, 9, 9)                       # C % 8 != 0


@pytest.mark.gpu
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
@pytest.mark.parametrize("kind", KINDS)
def test_value_edges(kind, grad_edges):
    # NaN, +-Inf, near-max, subnormal and -0.0 batch-norm outputs and identities (input_edges); NaN, Inf and edge values
    # in dy and the identity (gradient_edges)
    x, dy, identity = edge_site_inputs(8, 64, 16, 16, 11 + grad_edges, grad_edges)
    check_site(kind, x, identity, dy, bn_setup=edge_bn_setup(grad_edges), p=0.5)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [1.0, 1e-6, 0.1, 0.025, 0.5], ids=["all_dropped", "none_dropped", "survive_0.9", "survive_0.975", "half"])
def test_stochastic_depth_rates(p):
    # 0.9 and 0.975 have inexact bf16 reciprocals; p = 1 drops every row (no division), p = 1e-6 none
    want, got = check_gauss_site("drop", 64, 24, 14, 14, p=p, seed=3)
    if p == 1.0:   # no gradient reaches the batch norm
        assert not got["dbias"].any() and not got["dweight"].any()


@pytest.mark.gpu
@pytest.mark.parametrize("p", [0.5, 1.0])
def test_inf_and_nan_gradients_in_dropped_rows(p):
    # every row's dy holds +-Inf and NaN: a dropped row's g is then NaN there (dy * 0), as torch's mul gives
    x, identity, dy = gauss_inputs(16, 32, 8, 8, 21)
    dy = dy.clone()
    dy[:, 0], dy[:, 1], dy[:, 2] = float("inf"), float("-inf"), float("nan")
    dy[:, 3, 0, 0] = float("nan")
    check_site("drop", x, identity, dy, p=p, seed=4)


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (0.01, 1e-3), (0.3, 0.5), (0.1, 1e-12)])
@pytest.mark.parametrize("kind", KINDS)
def test_hyperparameters(kind, momentum, eps):
    check_gauss_site(kind, 8, 40, 28, 28, momentum=momentum, eps=eps, nbt=2 ** 40)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 64, 100])
@pytest.mark.parametrize("kind", KINDS)
def test_nchw_gradient_keeps_eager_torch_s_backward(kind, c):
    # an NCHW dy: eager torch's mul writes g in NCHW and its batch-norm backward takes its NCHW kernels, so the site's
    # backward runs those torch ops.  With one channel NCHW strides (stride(1) == H * W) also pass the channels-last
    # check, so the site runs its native backward, and eager torch's kernels on that gradient must round alike.
    x, identity, dy = gauss_inputs(8, c, 7, 7, c)
    dy = torch.empty(dy.shape, dtype=dy.dtype, device=dy.device).copy_(dy)   # default strides, even where C == 1
    assert dy.stride(1) == 7 * 7 and dy.is_contiguous(memory_format=CL) == (c == 1)
    check_site(kind, x, identity, dy, launches=4 if c == 1 else 2, seed=c)


# ---- eval sites -------------------------------------------------------------------------------------------------
def check_eval_site(x, bn, identity=None):
    with torch.inference_mode():
        want = bn(x) if identity is None else identity + bn(x)
        buffers = [t.clone() for t in bn.buffers()]
        before = N.launch_count()
        got = fused_norm.bn_res(bn, x, identity)
        torch.cuda.synchronize()
    assert N.launch_count() - before == 1
    assert got.stride() == want.stride()
    assert_same_values(got, want, "y")
    assert all(same_bits(a, b) for a, b in zip(buffers, bn.buffers())), "a running statistic changed"
    return want, got


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("c,h,w", MODEL_SHAPES[::2] + [(100, 9, 9)])
@pytest.mark.parametrize("residual", [False, True], ids=["plain", "add"])
def test_eval_sites(residual, c, h, w, params):
    x, identity, _ = gauss_inputs(32, c, h, w, c)
    bn = make_bn(c, c + 1, eps=1e-3).cuda().eval().to(PARAMS[params])
    check_eval_site(x, bn, identity if residual else None)
    if c % 8 == 0:
        check_eval_site(misaligned(x), bn, identity if residual else None)
        if residual:
            check_eval_site(x, bn, misaligned(identity))


@pytest.mark.gpu
def test_eval_value_edges():
    x, _, identity = edge_site_inputs(8, 64, 16, 16, 11, False)
    bn = make_bn(64, 2).cuda().eval()
    edge_bn_setup(False)(bn)
    check_eval_site(x, bn)
    check_eval_site(x, bn, identity)


# ---- every b200c::bn_res kernel and the case that launches it ----------------------------------------------------
_T = "b200c::bn_res::k_res_transform<{}, (b200c::bn_res::Res){}>"
_R = "b200c::bn_res::k_res_bwd_reduce"
_I = "b200c::bn_res::k_res_infer<{}, (b200c::bn_res::Res){}, {}>"
_P = {"fp32": "float", "bf16": "__nv_bfloat16"}
KERNELS = {_R: "drop_c64"}
for _v, _c in ((8, 64), (1, 100)):
    KERNELS[_T.format(_v, 1)] = f"add_c{_c}"
    KERNELS[_T.format(_v, 2)] = f"drop_c{_c}"
    for _r, _kind in ((0, "plain"), (1, "add")):
        for _p in PARAMS:
            KERNELS[_I.format(_v, _r, _P[_p])] = f"eval_{_kind}_c{_c}_{_p}"


def kernel_name(signature):
    """`b200c::bn_res::k_...<template arguments>` of a demangled kernel signature."""
    name = signature[signature.index("b200c::bn_res::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_res_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted({f for f in re.findall(r"Function (\S+):", out) if f.startswith("_ZN5b200c6bn_res")})
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(mangled) == len(KERNELS) == 13
    assert names == set(KERNELS), {"without a case": sorted(names - set(KERNELS)), "not in the library": sorted(set(KERNELS) - names)}


def case_runs():
    runs = {}
    for kind in ("add", "drop"):
        runs[f"{kind}_c64"] = lambda kind=kind: check_gauss_site(kind, 8, 64, 16, 16)
        runs[f"{kind}_c100"] = lambda kind=kind: check_gauss_site(kind, 3, 100, 9, 9)
    for residual, kind in ((False, "plain"), (True, "add")):
        for c in (64, 100):
            for p in PARAMS:
                def eval_case(residual=residual, c=c, p=p):
                    x, identity, _ = gauss_inputs(4, c, 9, 9, c)
                    check_eval_site(x, make_bn(c, 3).cuda().eval().to(PARAMS[p]), identity if residual else None)
                runs[f"eval_{kind}_c{c}_{p}"] = eval_case
    return runs


def trace_cases():
    """Runs every case once under torch.profiler and prints {case: [b200c::bn_res kernels it launched]} as JSON."""
    launched = {}
    for case, run_case in case_runs().items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run_case()
            torch.cuda.synchronize()
        launched[case] = sorted({kernel_name(e.name) for e in prof.events()
                                 if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_res::" in e.name})
    print(json.dumps(launched))
