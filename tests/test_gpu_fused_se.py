"""torchvision's SqueezeExcitation with its pool and scale on the squeeze-excitation kernels (fused_norm's
FusedSqueezeExcitation, se_kernels.cuh) against the eager module, bit for bit.

Under bf16 autocast with fp32 parameters: y, x's gradient and the fc1 / fc2 weight and bias gradients must have the
same bits (a NaN matching a NaN), and the site must make its four native launches, for SiLU / Sigmoid (EfficientNet)
and ReLU / Hardsigmoid (MobileNetV3) at every SE shape of efficientnet_b0, mobilenet_v3_large and efficientnet_v2_s at
224 x 224 (batch 256 and 32), every regime of test_fused_se_cpu.SE_REGIME_SHAPES (x placed at its address), C = 100
and C = 3, one row per sample, x and dy off the vector grids, value edges (+-Inf, NaN, sums of -0.0 and sums past the
bf16 maximum), eval with fp32 and bf16 parameters, retain_graph with two backwards, x without a gradient, frozen fc
parameters, an NCHW dy and a squeeze path returning fp32.  KERNELS names every `b200c::se` kernel with the case that
launches it; test_gpu_zz_se_trace.py runs the trace."""
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
from gpu_common import assert_same_values
from test_fused_se_cpu import SE_REGIME_SHAPES

SqueezeExcitation = pytest.importorskip("torchvision.ops.misc").SqueezeExcitation

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")
ACTS = {"silu_sigmoid": (nn.SiLU, nn.Sigmoid), "relu_hardsigmoid": (nn.ReLU, nn.Hardsigmoid)}
# (C, H, W, squeeze channels) of every SE module of efficientnet_b0, mobilenet_v3_large and efficientnet_v2_s at 224 x 224
MODEL_SHAPES = {
    "efficientnet_b0": [(32, 112, 112, 8), (96, 56, 56, 4), (144, 56, 56, 6), (144, 28, 28, 6), (240, 28, 28, 10),
                        (240, 14, 14, 10), (480, 14, 14, 20), (672, 14, 14, 28), (672, 7, 7, 28), (1152, 7, 7, 48)],
    "mobilenet_v3_large": [(72, 28, 28, 24), (120, 28, 28, 32), (480, 14, 14, 120), (672, 14, 14, 168), (672, 7, 7, 168),
                           (960, 7, 7, 240)],
    "efficientnet_v2_s": [(256, 14, 14, 16), (512, 14, 14, 32), (768, 14, 14, 32), (960, 14, 14, 40), (960, 7, 7, 40),
                          (1536, 7, 7, 64)],
}
MODEL_ACT = {"efficientnet_b0": "silu_sigmoid", "mobilenet_v3_large": "relu_hardsigmoid", "efficientnet_v2_s": "silu_sigmoid"}

_P = "b200c::se::k_se_pool<{}>"
_R = "b200c::se::k_se_bwd_reduce<{}, {}>"
# every b200c::se kernel, as the profiler names it, and the case of case_runs() that launches it
KERNELS = {
    _P.format(4): "c64",
    _P.format(2): "c64_x4",
    _P.format(1): "c64_x2",
    _R.format(4, "true"): "c64",
    _R.format(4, "false"): "c64_dy2",
    _R.format(2, "true"): "c6",
    _R.format(2, "false"): "c6_dy2",
    _R.format(1, "false"): "c3",
    "b200c::se::k_se_scale<8>": "c64",
    "b200c::se::k_se_scale<1>": "c64_x2",
    "b200c::se::k_se_bwd_elemt<8>": "c64",
    "b200c::se::k_se_bwd_elemt<1>": "c64_dy2",
}


def kernel_name(signature):
    """`b200c::se::k_...<template arguments>` of a demangled kernel signature: no return type, no parameter list."""
    name = signature[signature.index("b200c::se::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_se_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted({f for f in re.findall(r"Function (\S+):", out) if f.startswith("_ZN5b200c2se")})
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(mangled) == len(KERNELS) == 12
    assert names == set(KERNELS), {"without a case": sorted(names - set(KERNELS)), "not in the library": sorted(set(KERNELS) - names)}


def nhwc(t, offset=0):
    """A bf16 channels-last copy of `t` (stride(1) == 1) whose data pointer is `offset` elements past a 512-byte
    boundary."""
    n, c, h, w = t.shape
    v = torch.empty(t.numel() + offset, dtype=torch.bfloat16, device="cuda")[offset:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    assert v.is_contiguous(memory_format=CL) and v.stride(1) == 1 and v.data_ptr() % 16 == 2 * offset % 16
    return v


def make_se(c, sq, act, seed=0):
    torch.manual_seed(seed)
    a, s = ACTS[act]
    parent = SqueezeExcitation(c, sq, activation=a, scale_activation=s).cuda().to(memory_format=CL)
    fused = copy.deepcopy(parent)
    fused.__class__ = fused_norm.FusedSqueezeExcitation
    return parent, fused


def gauss(n, c, h, w, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, c, h, w, device="cuda", generator=g) * scale


def run(se, x, dy, x_grad=True, autocast=True, backwards=1):
    """y, dx, ds (the gradient reaching s, the scale activation's output) and the parameter gradients."""
    x = x.detach().clone() if x.data_ptr() % 16 == 0 else nhwc(x, (x.data_ptr() % 16) // 2)
    x.requires_grad_(x_grad)
    for p in se.parameters():
        p.grad = None
    ds = []

    def grab_ds(mod, inputs, out):
        if out.requires_grad:
            out.register_hook(ds.append)

    handle = se.scale_activation.register_forward_hook(grab_ds)
    try:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            y = se(x)
    finally:
        handle.remove()
    for i in range(backwards):
        y.backward(dy, retain_graph=i + 1 < backwards)
    grads = {f"{k}.grad": p.grad for k, p in se.named_parameters()}
    return {"y": y.detach(), "dx": x.grad, "ds": ds[-1] if ds else None, **grads}


def compare(got, want, where):
    assert got.keys() == want.keys()
    for k in want:
        if want[k] is None:
            assert got[k] is None, (where, k)
            continue
        assert got[k] is not None, (where, k)
        assert got[k].stride() == want[k].stride() or k not in ("y", "dx"), (where, k, got[k].stride(), want[k].stride())
        assert_same_values(got[k], want[k], f"{where} {k}")


def check_se(n, c, h, w, act="silu_sigmoid", sq=None, x_off=0, dy_off=0, x=None, dy=None, nchw=False, launches=4, seed=0,
             params="fp32", **kw):
    """One site against eager torch: x and dy (gaussian unless given) placed x_off / dy_off elements off the 512-byte
    grid in channels-last, or dy kept as given with `nchw`; with params "bf16" both modules are cast to bf16 and run
    without autocast.  Returns the fused module's results."""
    parent, fused = make_se(c, sq or max(1, c // 4), act, seed)
    if params == "bf16":
        parent, fused = parent.bfloat16(), fused.bfloat16()
        kw["autocast"] = False
    if x is None:
        x = gauss(n, c, h, w, seed + 1, 2.0) + 0.5
    if dy is None:
        dy = gauss(n, c, h, w, seed + 2)
    x = nhwc(x, x_off)
    dy = dy if nchw else nhwc(dy, dy_off)
    want = run(parent, x, dy, **kw)
    before = N.launch_count()
    got = run(fused, x, dy, **kw)
    torch.cuda.synchronize()
    assert N.launch_count() - before == launches, (n, c, h, w)
    compare(got, want, (n, c, h, w, act, x_off, dy_off))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("n", [256, 32])
@pytest.mark.parametrize("arch", sorted(MODEL_SHAPES))
def test_model_shapes(arch, n):
    for c, h, w, sq in MODEL_SHAPES[arch]:
        check_se(n, c, h, w, MODEL_ACT[arch], sq)


@pytest.mark.gpu
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("regime", sorted(SE_REGIME_SHAPES), ids=lambda r: f"{r[0]}@{r[1]}")
def test_regime_shapes(regime, act):
    (n, c, h, w), addr = regime
    check_se(n, c, h, w, act, x_off=addr // 2)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4, 100, 14, 14), (8, 100, 56, 56), (16, 3, 28, 28), (64, 3, 7, 7), (8, 64, 1, 1),
                                   (3, 100, 1, 1), (5, 3, 1, 1), (32, 2, 9, 9)])
def test_odd_channels_and_one_row(shape):
    check_se(*shape)
    check_se(*shape, act="relu_hardsigmoid", seed=5)


@pytest.mark.gpu
@pytest.mark.parametrize("x_off, dy_off", [(1, 0), (2, 0), (0, 1), (0, 2), (3, 5), (4, 4)])
@pytest.mark.parametrize("shape", [(8, 64, 28, 28), (4, 96, 56, 56), (8, 6, 16, 16)])
def test_misaligned_operands(shape, x_off, dy_off):
    check_se(*shape, x_off=x_off, dy_off=dy_off)


def edge_tensor(n, c, h, w, seed):
    """Gaussian values with, per channel group, +-Inf, NaN, all -0.0 and values whose sum passes the bf16 maximum."""
    t = gauss(n, c, h, w, seed)
    t[:, 0] = -0.0
    t[0, 1, 0, 0] = float("inf")
    t[1 % n, 2, -1, -1] = float("-inf")
    t[0, 3, 1 % h, 0] = float("nan")
    t[:, 4] = 3.0e38
    t[:, 5, 0] = -3.0e38
    t[:, 6] = 1.0e38
    t[0, 7, 0, 0], t[0, 7, -1, -1] = float("inf"), float("-inf")
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("shape", [(4, 64, 14, 14), (2, 16, 64, 64), (3, 12, 7, 7)])
def test_value_edges(shape, act):
    check_se(*shape, act=act, x=edge_tensor(*shape, 11))
    check_se(*shape, act=act, dy=edge_tensor(*shape, 12))
    check_se(*shape, act=act, x=edge_tensor(*shape, 13), dy=edge_tensor(*shape, 14))


@pytest.mark.gpu
@pytest.mark.parametrize("params", ["fp32", "bf16"])
@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
@pytest.mark.parametrize("shape", [(32, 672, 7, 7), (8, 100, 56, 56), (4, 3, 1, 1)])
def test_eval(shape, mode, params):
    n, c, h, w = shape
    parent, fused = make_se(c, max(1, c // 4), "silu_sigmoid")
    if params == "bf16":
        parent, fused = parent.bfloat16(), fused.bfloat16()
    x = nhwc(gauss(n, c, h, w, 3))
    ctx = torch.no_grad if mode == "no_grad" else torch.inference_mode
    outs = []
    for se in (parent, fused):
        se.eval()
        before = N.launch_count()
        with ctx(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=params == "fp32"):
            outs.append(se(x))
        launched = N.launch_count() - before
    assert launched == 2
    assert outs[0].stride() == outs[1].stride()
    assert_same_values(outs[1], outs[0], f"eval {shape} {params}")


@pytest.mark.gpu
def test_retain_graph_two_backwards():
    # the second backward adds to the first's gradients: 2 forward launches and 2 per backward
    check_se(8, 96, 28, 28, backwards=2, launches=6)
    check_se(4, 100, 14, 14, act="relu_hardsigmoid", backwards=2, launches=6)


@pytest.mark.gpu
def test_x_without_gradient():
    got = check_se(8, 96, 28, 28, x_grad=False, launches=3)
    assert got["dx"] is None and got["fc1.weight.grad"] is not None


@pytest.mark.gpu
def test_frozen_fc_parameters():
    n, c, h, w = 8, 96, 28, 28
    parent, fused = make_se(c, 24, "silu_sigmoid")
    for se in (parent, fused):
        for p in se.parameters():
            p.requires_grad_(False)
    x, dy = nhwc(gauss(n, c, h, w, 1)), nhwc(gauss(n, c, h, w, 2))
    want = run(parent, x, dy)
    before = N.launch_count()
    got = run(fused, x, dy)
    assert N.launch_count() - before == 4
    compare(got, want, "frozen")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(8, 96, 28, 28), (4, 100, 7, 7), (2, 3, 9, 9)])
def test_nchw_gradient_runs_torch_s_backward(shape):
    # the forward's 2 launches; the backward runs eager torch's ops in dy's layout
    n, c, h, w = shape
    dy = gauss(n, c, h, w, 9).bfloat16()
    assert dy.is_contiguous() and not dy.is_contiguous(memory_format=CL)
    check_se(*shape, dy=dy, nchw=True, launches=2)


class _Fp32Sigmoid(nn.Module):
    def forward(self, t):
        return torch.sigmoid(t).float()


@pytest.mark.gpu
def test_squeeze_path_returning_fp32_runs_torch_s_scale():
    n, c, h, w = 8, 64, 14, 14
    parent, fused = make_se(c, 16, "silu_sigmoid")
    parent.scale_activation, fused.scale_activation = _Fp32Sigmoid(), _Fp32Sigmoid()
    x, dy = nhwc(gauss(n, c, h, w, 1)), gauss(n, c, h, w, 2).contiguous(memory_format=CL)
    want = run(parent, x, dy)
    before = N.launch_count()
    got = run(fused, x, dy)
    assert N.launch_count() - before == 1   # the pool only
    assert got["y"].dtype == torch.float32
    compare(got, want, "fp32 squeeze path")


@pytest.mark.gpu
def test_too_little_scratch_is_rejected_before_the_launch():
    lib = fused_norm._native_lib()
    n, c, hw = 8, 64, 64 * 64
    need = lib.b200c_se_scratch_bytes(n, c, hw)
    assert need > 4096 * 4   # a split launch: semaphores and staging
    buf = torch.zeros(need, dtype=torch.uint8, device="cuda")
    x = torch.zeros(n * c * hw, dtype=torch.bfloat16, device="cuda")
    out = torch.zeros(n * c, dtype=torch.bfloat16, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    before = N.launch_count()
    assert lib.b200c_se_pool(x.data_ptr(), out.data_ptr(), n, c, hw, buf.data_ptr(), need - 1, stream) == N.EINVAL
    assert "scratch" in N.last_error()
    assert lib.b200c_se_backward_reduce(x.data_ptr(), x.data_ptr(), out.data_ptr(), n, c, hw, buf.data_ptr(), need - 1,
                                        stream) == N.EINVAL
    assert N.launch_count() == before
    N.check(lib.b200c_se_pool(x.data_ptr(), out.data_ptr(), n, c, hw, buf.data_ptr(), need, stream))
    torch.cuda.synchronize()
    assert not buf[:4096 * 4].any(), "the semaphores are left at zero"


def case_runs():
    return {
        "c64": lambda: check_se(8, 64, 32, 32),
        "c64_x4": lambda: check_se(8, 64, 32, 32, x_off=2),
        "c64_x2": lambda: check_se(8, 64, 32, 32, x_off=1),
        "c64_dy2": lambda: check_se(8, 64, 32, 32, dy_off=1),
        "c6": lambda: check_se(8, 6, 32, 32),
        "c6_dy2": lambda: check_se(8, 6, 32, 32, dy_off=1),
        "c3": lambda: check_se(8, 3, 32, 32),
    }


def trace_cases():
    """Runs every case once under torch.profiler and prints {case: [b200c::se kernels it launched]} as JSON."""
    launched = {}
    for case, fn in case_runs().items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        launched[case] = sorted({kernel_name(e.name) for e in prof.events()
                                 if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::se::" in e.name})
    print(json.dumps(launched))


@pytest.mark.gpu
@pytest.mark.parametrize("act", sorted(ACTS))
@pytest.mark.parametrize("shape", [(32, 672, 7, 7), (8, 96, 56, 56), (4, 100, 56, 56), (16, 3, 32, 32), (8, 64, 1, 1)])
def test_model_cast_to_bf16(shape, act):
    check_se(*shape, act=act, params="bf16")
    check_se(*shape, act=act, params="bf16", x_off=1, dy_off=2, seed=3)


@pytest.mark.gpu
@pytest.mark.parametrize("params", ["fp32", "bf16"])
@pytest.mark.parametrize("shape", [(8, 64, 1, 1), (5, 3, 1, 1), (4, 6, 1, 1)])
def test_one_row_keeps_the_sign_of_a_zero_product(shape, params):
    # sum_to hands back dy * x itself over one row: x = +0 against a negative dy must give ds = -0.0
    n, c, h, w = shape
    x = gauss(n, c, h, w, 4).abs()
    x[:, ::2] = 0.0
    dy = -gauss(n, c, h, w, 5).abs() - 0.25
    got = check_se(*shape, x=x, dy=dy, params=params)
    ds = got["ds"][:, ::2].contiguous().view(torch.int16)
    assert bool((ds == torch.tensor(-0.0, dtype=torch.bfloat16).view(torch.int16)).all())


def _site_graph_is_freed(backward):
    """Whether a fused training forward (with `backward`, its backward too) leaves nothing behind: s (the scale
    activation's output) is collected and the device memory is back where it started."""
    import gc
    import weakref

    n, c, h, w = 8, 96, 28, 28
    _, fused = make_se(c, 24, "silu_sigmoid")
    x = nhwc(gauss(n, c, h, w, 1)).requires_grad_()
    dy = nhwc(gauss(n, c, h, w, 2))
    refs = []
    handle = fused.scale_activation.register_forward_hook(lambda m, i, o: refs.append(weakref.ref(o)))

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = fused(x)
        if backward:
            y.backward(dy)
        del y
        x.grad = None
        for p in fused.parameters():
            p.grad = None

    step()   # the first steps allocate the site's scratch and settle cuDNN's and autocast's own buffers
    step()
    gc.collect()
    torch.cuda.synchronize()
    start = torch.cuda.memory_allocated()
    refs.clear()
    for _ in range(3):
        step()
    handle.remove()
    gc.collect()
    torch.cuda.synchronize()
    return len(refs) == 3 and all(r() is None for r in refs), torch.cuda.memory_allocated() - start


@pytest.mark.gpu
@pytest.mark.parametrize("backward", [True, False], ids=["training_step", "forward_without_backward"])
def test_a_site_s_graph_is_freed(backward):
    freed, grown = _site_graph_is_freed(backward)
    assert freed, "s outlived its step"
    assert grown <= 0, f"{grown} bytes of device memory left behind"
