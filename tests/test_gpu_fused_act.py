"""Batch norm followed by ReLU6, SiLU or Hardswish (fused_norm.bn_act, norm_act.cuh) against eager torch, bit for bit.

Training sites: y, the running statistics, num_batches_tracked, dx, dweight and dbias against eager torch's batch norm
followed by the activation module (inplace and not), at every activation-site shape of mobilenet_v2,
mobilenet_v3_large, efficientnet_b0 and regnet_y_400mf at 224 x 224 (batch 256 and 32), every launch regime, the
scalar kernels, value edges of x and dy, and a range of momentum and eps.  Eval sites: y, with fp32 and bf16
parameters.  The epilogues exhaustively: every bf16 value of t through the eval site, and every bf16 value of t
through b200c_bn_backward_act against aten's silu_backward / hardswish_backward / hardtanh_backward.  KERNELS names
every `b200c::bn_act` kernel with the case that launches it; the profiler traces run in subprocesses from
test_gpu_zz_act_trace.py, and the whole models in test_gpu_zz_act_models.py."""
import copy
import json
import os
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values, same_bits
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn, misaligned

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")
ACTS = {"relu6": nn.ReLU6, "silu": nn.SiLU, "hardswish": nn.Hardswish}
CODES = {"relu6": N.ACT_RELU6, "silu": N.ACT_SILU, "hardswish": N.ACT_HARDSWISH}
PARAMS = {"fp32": torch.float32, "bf16": torch.bfloat16}
# (C, H, W) of every Conv2dNormActivation with an activation in mobilenet_v2, mobilenet_v3_large, efficientnet_b0 and
# regnet_y_400mf at 224 x 224
MODEL_SHAPES = [(16, 112, 112), (32, 112, 112), (48, 56, 56), (48, 112, 112), (64, 56, 56), (64, 112, 112), (72, 28, 28),
                (72, 56, 56), (96, 56, 56), (96, 112, 112), (104, 28, 28), (104, 56, 56), (120, 28, 28), (144, 28, 28),
                (144, 56, 56), (184, 14, 14), (192, 14, 14), (192, 28, 28), (200, 14, 14), (208, 14, 14), (208, 28, 28),
                (240, 14, 14), (240, 28, 28), (384, 14, 14), (440, 7, 7), (440, 14, 14), (480, 14, 14), (576, 7, 7),
                (576, 14, 14), (672, 7, 7), (672, 14, 14), (960, 7, 7), (1152, 7, 7), (1280, 7, 7)]


def nhwc(t):
    """A bf16 copy of `t` with NHWC strides, stride(1) == 1 included (C = 1)."""
    n, c, h, w = t.shape
    return torch.empty(n, h, w, c, dtype=torch.bfloat16, device=t.device).permute(0, 3, 1, 2).copy_(t)


def gauss_inputs(n, c, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    # centred near the activations' corners (0 and 6 for ReLU6, +-3 for Hardswish) and past them
    x = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g) * 3 + 0.5)
    dy = nhwc(torch.randn(n, c, h, w, device="cuda", generator=g))
    return x, dy


def run(bn, act, x, dy, fused):
    x = x.clone().requires_grad_() if x.data_ptr() % 16 == 0 else misaligned(x.detach()).requires_grad_()
    y = fused_norm.bn_act(bn, act, x) if fused else act(bn(x))
    y.backward(dy)
    return {"y": y.detach(), "dx": x.grad, "dweight": bn.weight.grad, "dbias": bn.bias.grad, "running_mean": bn.running_mean,
            "running_var": bn.running_var, "num_batches_tracked": bn.num_batches_tracked}


def check_site(act_name, x, dy, inplace=False, bn_setup=None, launches=4, seed=0, **bn_args):
    """One training site through bn_act and through eager torch's modules; every result must have the same bits
    (a NaN matching a NaN), and the fused site must make `launches` native launches."""
    c = x.shape[1]
    ref_bn = make_bn(c, seed, **bn_args).cuda()
    if bn_setup is not None:
        bn_setup(ref_bn)
    fused_bn = copy.deepcopy(ref_bn)
    want = run(ref_bn, ACTS[act_name](inplace=inplace), x, dy, fused=False)
    before = N.launch_count()
    got = run(fused_bn, ACTS[act_name](inplace=inplace), x, dy, fused=True)
    torch.cuda.synchronize()
    assert N.launch_count() - before == launches
    for k in want:
        assert_same_values(got[k], want[k], k)
    assert got["y"].is_contiguous(memory_format=CL) and got["dx"].is_contiguous(memory_format=CL)
    return want, got


def check_gauss_site(act_name, n, c, h, w, inplace=False, misalign=False, **bn_args):
    x, dy = gauss_inputs(n, c, h, w, n * 7 + c * 13 + h)
    if misalign:
        x = misaligned(x)
    return check_site(act_name, x, dy, inplace, seed=c, **bn_args)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [256, 32])
@pytest.mark.parametrize("c,h,w", MODEL_SHAPES)
@pytest.mark.parametrize("act", list(ACTS))
def test_model_site_shapes(act, c, h, w, n):
    check_gauss_site(act, n, c, h, w, inplace=(c // 8) % 2 == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(BN_REGIME_SHAPES), ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("act", list(ACTS))
def test_launch_regimes(act, shape):
    check_gauss_site(act, *shape, inplace=True)


@pytest.mark.gpu
@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("act", list(ACTS))
def test_scalar_kernels(act, inplace):
    check_gauss_site(act, 3, 100, 9, 9, inplace)              # C % 8 != 0
    check_gauss_site(act, 8, 64, 16, 16, inplace, misalign=True)   # x off the 16-byte grid


@pytest.mark.gpu
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
@pytest.mark.parametrize("act", list(ACTS))
def test_value_edges(act, grad_edges):
    # NaN, +-Inf, near-max, subnormal and -0.0 batch-norm outputs (input_edges); NaN, Inf and edge values in dy
    x, dy, _ = edge_site_inputs(8, 64, 16, 16, 11 + grad_edges, grad_edges)
    check_site(act, x, dy, bn_setup=edge_bn_setup(grad_edges))


@pytest.mark.gpu
@pytest.mark.parametrize("act", list(ACTS))
def test_outputs_at_the_corners_and_past_exp_overflow(act):
    # t = bf16(w * (x - mean) * invstd + b) near 0, on 6 and +-3, next to them, and beyond +-88 (where expf(-t) overflows
    # or is 0): channel k has weight 2^-20 and bias corners[k], so t is corners[k] plus an offset below 2^-17
    corners = torch.tensor([0.0, -0.0, 6.0, 3.0, -3.0, 100.0, -100.0, 89.0, -89.0, 1e30, -1e30, 2.0 ** -130, 5.96875, 6.03125,
                            -2.984375, 2.984375])

    def setup(bn):
        with torch.no_grad():
            bn.weight.fill_(2.0 ** -20)
            bn.bias.copy_(corners)
    x, dy = gauss_inputs(16, 16, 8, 8, 5)
    check_site(act, x, dy, bn_setup=setup)


@pytest.mark.gpu
@pytest.mark.parametrize("c", [1, 64, 100])
@pytest.mark.parametrize("act", list(ACTS))
def test_nchw_gradient_keeps_eager_torch_s_backward(act, c):
    # an NCHW dy (the gradient a model's average pool hands its last block): eager torch's activation backward writes g
    # in NCHW and its batch-norm backward takes its NCHW kernels, so the site's backward runs those torch ops.  With one
    # channel NCHW strides (stride(1) == H * W) also pass the channels-last check, so the site runs its native backward,
    # and eager torch's kernels on that gradient must round alike.
    x, dy = gauss_inputs(8, c, 7, 7, c)
    dy = torch.empty(dy.shape, dtype=dy.dtype, device=dy.device).copy_(dy)   # default strides, even where C == 1
    assert dy.stride(1) == 7 * 7 and dy.is_contiguous(memory_format=CL) == (c == 1)
    check_site(act, x, dy, launches=4 if c == 1 else 2, seed=c)


@pytest.mark.gpu
@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (0.01, 1e-3), (0.3, 0.5), (0.1, 1e-12)])
@pytest.mark.parametrize("act", list(ACTS))
def test_hyperparameters(act, momentum, eps):
    check_gauss_site(act, 8, 104, 28, 28, momentum=momentum, eps=eps, nbt=2 ** 40)


# ---- eval sites -------------------------------------------------------------------------------------------------
def check_eval_site(act_name, x, bn, inplace=False):
    with torch.inference_mode():
        want = ACTS[act_name](inplace=inplace)(bn(x))
        buffers = [t.clone() for t in bn.buffers()]
        before = N.launch_count()
        got = fused_norm.bn_act(bn, ACTS[act_name](inplace=inplace), x)
        torch.cuda.synchronize()
    assert N.launch_count() - before == 1
    assert got.stride() == want.stride()
    assert_same_values(got, want, "y")
    assert all(same_bits(a, b) for a, b in zip(buffers, bn.buffers())), "a running statistic changed"
    return want, got


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("c,h,w", MODEL_SHAPES[::3] + [(100, 9, 9)])
@pytest.mark.parametrize("act", list(ACTS))
def test_eval_sites(act, c, h, w, params):
    x, _ = gauss_inputs(32, c, h, w, c)
    bn = make_bn(c, c + 1, eps=1e-3).cuda().eval().to(PARAMS[params])
    check_eval_site(act, x, bn, inplace=c % 2 == 0)
    if c % 8 == 0:
        check_eval_site(act, misaligned(x), bn)


# ---- the epilogues, exhaustively ---------------------------------------------------------------------------------
def every_bf16():
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("act", list(ACTS))
def test_every_bf16_t_through_the_forward(act, params):
    # running_var 0.75 + eps 0.25 makes invstd exactly 1; weight 1, mean 0 and bias -0.0 make t = x for every x, -0.0
    # included (a NaN's payload aside: rounding t to bf16 makes every NaN torch's canonical one).  Eager torch's batch
    # norm must agree that t = x.
    x = nhwc(every_bf16().view(64, 16, 8, 8))
    bn = nn.BatchNorm2d(16, eps=0.25).cuda().eval()
    with torch.no_grad():
        bn.running_var.fill_(0.75)
        bn.bias.fill_(-0.0)
    bn = bn.to(PARAMS[params])
    with torch.inference_mode():
        assert_same_values(bn(x), x, "eager torch's t")
    check_eval_site(act, x, bn)


@pytest.mark.gpu
@pytest.mark.parametrize("act", list(ACTS))
def test_every_bf16_t_through_the_gradient(act):
    # 65,536 channels, 2 rows, saved mean 0 and invstd 1, weight 1, bias -0.0: row 0 holds t = x = every bf16 value and a
    # seeded dy, row 1 t = 0 and dy = 0 (g = +0).  The reduce writes every g; dbias[c] = 0 + g(dy[c], t[c]) (-0.0 as +0.0).
    c = 65536
    t = every_bf16()
    g = torch.Generator(device="cuda").manual_seed(9)
    dy0 = torch.randn(c, device="cuda", generator=g).to(torch.bfloat16)
    special = torch.tensor([float("nan"), float("inf"), -float("inf"), -0.0, 0.0, 2.0 ** -133, 1.0], device="cuda")
    every7 = torch.arange(0, c, 7, device="cuda")
    dy0[every7] = special[torch.arange(every7.numel(), device="cuda") % special.numel()].to(torch.bfloat16)
    x = torch.stack([t, torch.zeros_like(t)])
    dy = torch.stack([dy0, torch.zeros_like(dy0)])
    ones, zeros = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
    bias = torch.full((c,), -0.0, device="cuda")
    gx, dx, dw, db = torch.empty_like(x), torch.empty_like(x), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    scratch = torch.zeros(int(N.load().b200c_bn_scratch_bytes(c)), dtype=torch.uint8, device="cuda")
    N.check(N.load().b200c_bn_backward_act(dy.data_ptr(), x.data_ptr(), gx.data_ptr(), dx.data_ptr(), ones.data_ptr(), bias.data_ptr(),
                                           zeros.data_ptr(), ones.data_ptr(), dw.data_ptr(), db.data_ptr(), CODES[act], 2, c,
                                           scratch.data_ptr(), torch.cuda.current_stream().cuda_stream))
    if act == "silu":
        want = torch.ops.aten.silu_backward(dy0, t)
    elif act == "hardswish":
        want = torch.ops.aten.hardswish_backward(dy0, t)
    else:
        want = torch.ops.aten.hardtanh_backward(dy0, t, 0.0, 6.0)
    assert_same_values(gx[0], want, "g")                 # the g the reduce wrote, every bit
    assert_same_values(db, want.float() + 0.0, "dbias")


# ---- every b200c::bn_act kernel and the case that launches it ----------------------------------------------------
_T = "b200c::bn_act::k_act_transform<{}, (b200c::bn_act::Act){}>"
_R = "b200c::bn_act::k_act_bwd_reduce<(b200c::bn_act::Act){}>"
_I = "b200c::bn_act::k_act_infer<{}, (b200c::bn_act::Act){}, {}>"
_P = {"fp32": "float", "bf16": "__nv_bfloat16"}
KERNELS = {}
for _a, _code in CODES.items():
    KERNELS[_R.format(_code)] = f"{_a}_c64"
    for _v, _c in ((8, 64), (1, 100)):
        KERNELS[_T.format(_v, _code)] = f"{_a}_c{_c}"
        for _p in PARAMS:
            KERNELS[_I.format(_v, _code, _P[_p])] = f"eval_{_a}_c{_c}_{_p}"


def kernel_name(signature):
    """`b200c::bn_act::k_...<template arguments>` of a demangled kernel signature."""
    name = signature[signature.index("b200c::bn_act::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_act_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted({f for f in re.findall(r"Function (\S+):", out) if f.startswith("_ZN5b200c6bn_act")})
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(mangled) == len(KERNELS) == 21
    assert names == set(KERNELS), {"without a case": sorted(names - set(KERNELS)), "not in the library": sorted(set(KERNELS) - names)}


def case_runs():
    runs = {}
    for a in ACTS:
        runs[f"{a}_c64"] = lambda a=a: check_gauss_site(a, 8, 64, 16, 16)
        runs[f"{a}_c100"] = lambda a=a: check_gauss_site(a, 3, 100, 9, 9)
        for c in (64, 100):
            for p in PARAMS:
                runs[f"eval_{a}_c{c}_{p}"] = lambda a=a, c=c, p=p: check_eval_site(
                    a, gauss_inputs(4, c, 9, 9, c)[0], make_bn(c, 3).cuda().eval().to(PARAMS[p]))
    return runs


def trace_cases():
    """Runs every case once under torch.profiler and prints {case: [b200c::bn_act kernels it launched]} as JSON."""
    launched = {}
    for case, run_case in case_runs().items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run_case()
            torch.cuda.synchronize()
        launched[case] = sorted({kernel_name(e.name) for e in prof.events()
                                 if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_act::" in e.name})
    print(json.dumps(launched))
