"""The eval batch-norm sites (fused_norm.py, norm_infer.cuh) against eager torch's modules, bit for bit.

Each site kind runs through the public helpers in eval mode without autograd recording: BN -> ReLU (`bn_relu`),
BN -> `+= identity` -> ReLU (`bn_add_relu`), BN + downsample BN -> add -> ReLU (`bn_add_relu_downsample`) and the stem
BN -> ReLU -> max-pool 3/2/1 (`bn_relu_maxpool`).  The output must have eager torch's bits, dtype and strides, the site
must make exactly one native launch, and running_mean, running_var and num_batches_tracked must keep their bits.
Covered: every resnet18 / resnet50 batch-norm shape at batch 256, 32 and 1; fp32 and bf16 parameters; the scalar
kernels (C = 100, C = 4,104, operands off the 16-byte grid); value edges of running_var, eps, x and identity and pool
windows; no_grad and inference_mode; the sites that must stay on torch; whole torchvision models; a profiler trace
of a resnet50 eval forward; and a table naming every `b200c::bn_infer` kernel with the case that launches it.  The
two profiler traces run in subprocesses started from test_gpu_zz_infer_trace.py."""
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
from gpu_common import same_bits
from test_gpu_fused_norm import RESNET50_BN_SHAPES, edge_bn_setup, edge_site_inputs, make_bn, misaligned

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")
KINDS = ["relu", "tail", "dual", "stem"]
PARAMS = {"fp32": torch.float32, "bf16": torch.bfloat16}
# resnet18's batch-norm shapes are a subset of resnet50's
RESNET18_BN_SHAPES = [(64, 112, 112), (64, 56, 56), (128, 28, 28), (256, 14, 14), (512, 7, 7)]
assert set(RESNET18_BN_SHAPES) <= set(RESNET50_BN_SHAPES)
GRAD_MODES = {"inference_mode": torch.inference_mode, "no_grad": torch.no_grad}


def eval_bn(c, seed, params="fp32", eps=1e-5):
    return make_bn(c, seed, eps=eps).eval().to(PARAMS[params])


def inputs(kind, n, c, h, w, seed):
    """x, and the identity (a tail) or the downsample batch norm's input (a dual tail), bf16 channels-last."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(n, h, w, c, device="cuda", generator=g) * 2 + 0.3).to(torch.bfloat16).permute(0, 3, 1, 2)
    z = (torch.randn(n, h, w, c, device="cuda", generator=g) - 0.2).to(torch.bfloat16).permute(0, 3, 1, 2)
    return x, z if kind in ("tail", "dual") else None


def identity_conv(c):
    """An nn.Conv2d whose forward is the identity, so that the dual tail's downsample input is exactly the tensor given
    (including values a real convolution would spread over every channel)."""
    conv = nn.Conv2d(c, c, 1, bias=False).cuda()
    conv.forward = lambda t: t
    return conv


def torch_site(kind, bn, bn_ds, x, z, relu=None, pool=None, downsample=None):
    """What eager torch computes: the modules' own ops, in torchvision's order."""
    relu = relu or nn.ReLU(inplace=True)
    if kind == "relu":
        return relu(bn(x))
    if kind == "stem":
        return (pool or nn.MaxPool2d(3, 2, 1))(relu(bn(x)))
    out = bn(x)
    out += z if kind == "tail" else (downsample(z) if downsample is not None else bn_ds(z))
    return relu(out)


def fused_site(kind, bn, bn_ds, x, z, relu=None, pool=None, downsample=None):
    relu = relu or nn.ReLU(inplace=True)
    if kind == "relu":
        return fused_norm.bn_relu(bn, relu, x)
    if kind == "tail":
        return fused_norm.bn_add_relu(bn, relu, x, z)
    if kind == "dual":
        ds = downsample if downsample is not None else nn.Sequential(identity_conv(x.shape[1]), bn_ds)
        return fused_norm.bn_add_relu_downsample(bn, relu, x, ds, z)
    return fused_norm.bn_relu_maxpool(bn, relu, pool or nn.MaxPool2d(3, 2, 1), x)


def buffers(*bns):
    return [t.clone() for bn in bns if bn is not None for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)
            if t is not None]


def check_site(kind, x, z, bn, bn_ds=None, grad_mode="inference_mode", launches=1, **modules):
    """Runs the site through the fused helper and through eager torch's modules under `grad_mode`; returns both outputs."""
    before_buffers = buffers(bn, bn_ds)
    with GRAD_MODES[grad_mode]():
        want = torch_site(kind, bn, bn_ds, x, z, **modules)
        before = N.launch_count()
        got = fused_site(kind, bn, bn_ds, x, z, **modules)
        torch.cuda.synchronize()
        launched = N.launch_count() - before
    assert launched == launches, f"{launched} native launches, expected {launches}"
    assert got.dtype == want.dtype and got.shape == want.shape and got.stride() == want.stride()
    assert same_bits(got, want), "differs from eager torch"
    after = buffers(bn, bn_ds)
    assert all(same_bits(a, b) for a, b in zip(before_buffers, after)), "a running statistic changed"
    return want, got


def run_kind(kind, n, c, h, w, params="fp32", seed=0, grad_mode="inference_mode", misalign=()):
    x, z = inputs(kind, n, c, h, w, seed)
    if "x" in misalign:
        x = misaligned(x)
    if "z" in misalign:
        z = misaligned(z)
    bn_ds = eval_bn(c, seed + 2, params, eps=1e-3) if kind == "dual" else None
    return check_site(kind, x, z, eval_bn(c, seed + 1, params), bn_ds, grad_mode)


# ---- every resnet18 / resnet50 batch-norm shape ------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("n", [256, 32, 1])
@pytest.mark.parametrize("c,h,w", RESNET50_BN_SHAPES)
@pytest.mark.parametrize("kind", KINDS)
def test_site_is_bit_identical_to_eager_torch(kind, c, h, w, n, params):
    run_kind(kind, n, c, h, w, params, seed=c + h + n)


@pytest.mark.gpu
@pytest.mark.parametrize("grad_mode", list(GRAD_MODES))
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("kind", KINDS)
def test_both_grad_modes(kind, params, grad_mode):
    run_kind(kind, 8, 64, 14, 14, params, seed=5, grad_mode=grad_mode)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_grad_enabled_with_nothing_requiring_grad_runs_the_eval_site(kind):
    # frozen parameters and inputs that require no grad: the output would not require grad either
    x, z = inputs(kind, 4, 64, 14, 14, 6)
    bn, bn_ds = eval_bn(64, 7).requires_grad_(False), eval_bn(64, 8).requires_grad_(False) if kind == "dual" else None
    with torch.enable_grad():
        want = torch_site(kind, bn, bn_ds, x, z)
        before = N.launch_count()
        got = fused_site(kind, bn, bn_ds, x, z)
        torch.cuda.synchronize()
    assert N.launch_count() - before == 1
    assert same_bits(got, want) and not got.requires_grad and got.stride() == want.stride()


# ---- the scalar kernels ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("case", ["c100", "c4104", "x_off_grid", "identity_off_grid"])
@pytest.mark.parametrize("kind", KINDS)
def test_scalar_kernels(kind, case, params):
    if case == "identity_off_grid" and kind in ("relu", "stem"):
        pytest.skip("the site has no identity")
    shape = {"c100": (3, 100, 9, 9), "c4104": (8, 4104, 8, 8)}.get(case, (8, 64, 15, 15))
    run_kind(kind, *shape, params, seed=9, misalign={"x_off_grid": ("x",), "identity_off_grid": ("z",)}.get(case, ()))


# ---- value edges ------------------------------------------------------------------------------------------------------
VAR_EDGES = [0.0, -0.0, 1e-40, 3e38, -1.0, float("nan"), float("inf"), float("-inf"), 1e-45, 1.0, "-eps"]


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("eps", [1e-30, 1e-5, 1e-3, 1e-1])
@pytest.mark.parametrize("kind", KINDS)
def test_running_var_edges_and_eps(kind, eps, params):
    # running_var of 0, subnormal, huge, negative, NaN and +-Inf; var = -eps gives an infinite invstd (torch takes no
    # eps of 0: see the test below)
    c = 64
    x, z = inputs(kind, 4, c, 9, 9, 10)
    bns = [eval_bn(c, 11, params, eps), eval_bn(c, 12, params, eps) if kind == "dual" else None]
    with torch.no_grad():
        for k, bn in enumerate(b for b in bns if b is not None):
            edges = torch.tensor([-eps if v == "-eps" else v for v in VAR_EDGES], device="cuda").to(bn.running_var.dtype)
            bn.running_var[k * 8:k * 8 + len(edges)] = edges
            # x == mean at one element of each edge channel: 0 * Inf where the variance is -eps
            bn.running_mean[:20] = x[0, :20, 0, 0].to(bn.running_mean.dtype)
    check_site(kind, x, z, *bns)


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("edges", ["input_edges", "identity_edges"])
@pytest.mark.parametrize("kind", KINDS)
def test_value_edges_of_x_and_identity(kind, edges, params):
    # NaN, +-Inf, near-max, subnormal and -0.0 in x; edge values and -0.0 in the identity (gradient_edges of the
    # training tests puts them there)
    n, c, h, w = 8, 64, 16, 16
    x, _, identity = edge_site_inputs(n, c, h, w, 21, edges == "identity_edges")
    bn = make_bn(c, 22)
    edge_bn_setup(edges == "identity_edges")(bn)
    bn = bn.eval().to(PARAMS[params])
    bn_ds = eval_bn(c, 23, params) if kind == "dual" else None
    check_site(kind, x, identity if kind in ("tail", "dual") else None, bn, bn_ds)


@pytest.mark.gpu
@pytest.mark.parametrize("params", list(PARAMS))
def test_pool_windows_with_ties_nan_and_zero_maxima(params):
    from test_gpu_fused_norm import CONST, ONE_NAN, ZERO

    n, c, h, w = 8, 64, 16, 16
    x, _, _ = edge_site_inputs(n, c, h, w, 24, False)
    bn = make_bn(c, 25)
    with torch.no_grad():
        bn.bias[CONST] = 0.5         # a constant channel: every window a tie of one positive value
        bn.bias[ZERO] = -0.5         # a zero channel after the ReLU: every window's maximum is 0
        bn.running_var[ONE_NAN + 1] = float("nan")   # a NaN channel: NaN in every window
    bn = bn.eval().to(PARAMS[params])
    _, got = check_site("stem", x, None, bn)
    assert torch.isnan(got[:, ONE_NAN + 1]).all() and (got[:, ZERO] == 0).all()
    assert torch.isnan(got[:, ONE_NAN]).any()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_eps_of_zero_raises_as_torch_does(kind):
    x, z = inputs(kind, 2, 64, 8, 8, 13)
    bn, bn_ds = eval_bn(64, 14, eps=0.0), eval_bn(64, 15, eps=0.0) if kind == "dual" else None
    with torch.inference_mode():
        with pytest.raises(ValueError, match="eps must be positive"):
            torch_site(kind, bn, bn_ds, x, z)
        before = N.launch_count()
        with pytest.raises(ValueError, match="eps must be positive"):
            fused_site(kind, bn, bn_ds, x, z)
    assert N.launch_count() == before


# ---- sites that stay on torch ----------------------------------------------------------------------------------------
FALLBACKS = ["grad_recorded", "no_running_stats", "nchw", "fp32_input", "fp16", "mixed_params", "empty_batch", "bn_hook",
             "relu_hook", "global_hook", "pool_hook", "downsample_hook"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FALLBACKS)
@pytest.mark.parametrize("kind", KINDS)
def test_ineligible_sites_run_torch_s_ops(kind, case):
    if (case == "pool_hook" and kind != "stem") or (case == "downsample_hook" and kind != "dual"):
        pytest.skip("no such module at this site")
    n, c, h, w = 0 if case == "empty_batch" else 4, 64, 14, 14
    x, z = inputs(kind, n, c, h, w, 30)
    bn, bn_ds = eval_bn(c, 31), eval_bn(c, 32) if kind == "dual" else None
    modules, handles = {}, []
    if case == "no_running_stats":
        bn = nn.BatchNorm2d(c, track_running_stats=False).cuda().eval()
    elif case == "nchw":
        x = x.contiguous()
        z = z.contiguous() if z is not None else None
    elif case in ("fp32_input", "fp16"):
        dtype = torch.float32 if case == "fp32_input" else torch.float16
        x, z = x.to(dtype), z.to(dtype) if z is not None else None
        bn, bn_ds = bn.to(dtype), bn_ds.to(dtype) if bn_ds is not None else None
    elif case == "mixed_params":
        bn.running_mean, bn.running_var = bn.running_mean.bfloat16(), bn.running_var.bfloat16()
    elif case == "bn_hook":
        handles.append(bn.register_forward_hook(lambda *a: None))
    elif case == "relu_hook":
        modules["relu"] = nn.ReLU(inplace=True)
        handles.append(modules["relu"].register_forward_pre_hook(lambda *a: None))
    elif case == "global_hook":
        handles.append(torch.nn.modules.module.register_module_forward_hook(lambda *a: None))
    elif case == "pool_hook":
        modules["pool"] = nn.MaxPool2d(3, 2, 1)
        handles.append(modules["pool"].register_forward_hook(lambda *a: None))
    elif case == "downsample_hook":
        modules["downsample"] = nn.Sequential(identity_conv(c), bn_ds)
        handles.append(modules["downsample"].register_forward_pre_hook(lambda *a: None))
    # a hooked max-pool or downsample branch keeps its module call, and the batch norm before it runs as the ReLU or
    # add + ReLU eval site: one launch of a transform kernel, none of the stem or dual kernel
    launches = 1 if case in ("pool_hook", "downsample_hook") else 0
    try:
        if case == "grad_recorded":
            before = N.launch_count()
            got = fused_site(kind, bn, bn_ds, x, z)
            torch.cuda.synchronize()
            assert N.launch_count() == before and got.requires_grad
            assert same_bits(got.detach(), torch_site(kind, bn, bn_ds, x, z).detach())
        else:
            check_site(kind, x, z, bn, bn_ds, launches=launches, **modules)
    finally:
        for h in handles:
            h.remove()


# ---- whole models ------------------------------------------------------------------------------------------------------
SITES = {"resnet18": 17, "resnet50": 49, "resnext50_32x4d": 49}   # the stem plus 2 per BasicBlock, 3 per Bottleneck


def model_input(dtype=torch.float32):
    g = torch.Generator(device="cuda").manual_seed(40)
    return torch.randn(8, 3, 128, 128, device="cuda", generator=g).to(dtype).contiguous(memory_format=CL)


def eval_logits(model, x, autocast):
    with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        before = N.launch_count()
        out = model(x)
        torch.cuda.synchronize()
    return out, N.launch_count() - before


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["autocast", "bf16_model", "trained", "sync_converted"])
@pytest.mark.parametrize("arch", list(SITES))
def test_model_eval_logits_have_the_untouched_model_s_bits(arch, case):
    pytest.importorskip("torchvision")
    import test_gpu_fused_resnet as R
    from ant_ray_b200 import train

    base = R.make_model(arch).cuda().to(memory_format=CL)
    if case == "sync_converted":
        base = nn.SyncBatchNorm.convert_sync_batchnorm(base)
    if case == "bf16_model":
        base = base.to(torch.bfloat16)
    ref = copy.deepcopy(base)
    if case == "trained":
        data = R.batches()
        fused = train.prepare_model(copy.deepcopy(base), parallel_strategy=None)
        R.train_steps(ref, data)
        R.train_steps(fused, data)
    else:
        fused = fused_norm.fuse_resnet(copy.deepcopy(base))
    assert type(fused) is fused_norm.FusedResNet
    ref.eval()
    fused.eval()
    x = model_input(torch.bfloat16 if case == "bf16_model" else torch.float32)
    autocast = case != "bf16_model"
    want, _ = eval_logits(ref, x, autocast)
    buffers_before = [t.clone() for _, t in fused.named_buffers()]
    got, launched = eval_logits(fused, x, autocast)
    assert launched == SITES[arch], f"{launched} native launches, expected {SITES[arch]}"
    assert same_bits(got, want), "eval logits differ from the untouched model"
    assert all(same_bits(a, b) for a, (_, b) in zip(buffers_before, fused.named_buffers())), "a buffer changed"


@pytest.mark.gpu
def test_eval_with_autograd_recording_keeps_the_parent_forward():
    pytest.importorskip("torchvision")
    import test_gpu_fused_resnet as R

    base = R.make_model("resnet18").cuda().to(memory_format=CL).eval()
    fused = fused_norm.fuse_resnet(copy.deepcopy(base))
    x = model_input()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        want = base(x)
        before = N.launch_count()
        got = fused(x)
    assert N.launch_count() == before and got.requires_grad
    assert same_bits(got.detach(), want.detach())


def infer_trace_kernels():
    """Prints the CUDA kernel names of one fused resnet50 eval forward under inference_mode and bf16 autocast, as JSON."""
    import torchvision

    torch.manual_seed(0)
    model = fused_norm.fuse_resnet(torchvision.models.resnet50(num_classes=10).cuda().to(memory_format=CL)).eval()
    x = torch.randn(2, 3, 64, 64, device="cuda").contiguous(memory_format=CL)

    def forward():
        with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
            return model(x)

    forward()   # warm-up
    before = N.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        forward()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    print(json.dumps({"kernels": names, "launches": N.launch_count() - before}))


# ---- every b200c::bn_infer kernel and the case that launches it ------------------------------------------------------
_T = "b200c::bn_infer::k_infer_transform<{}, (b200c::bn::Tail){}, {}>"
_P = "b200c::bn_infer::k_infer_pool<{}, {}>"
_PTYPE = {"fp32": "float", "bf16": "__nv_bfloat16"}
# Tail: 1 ReLU, 2 add + ReLU, 3 a second batch norm + add + ReLU.  V = 8 at C = 64, 1 at C = 100.
KERNELS = {}
for _p, _ty in _PTYPE.items():
    for _v, _c in ((8, 64), (1, 100)):
        for _tail, _kind in ((1, "relu"), (2, "tail"), (3, "dual")):
            KERNELS[_T.format(_v, _tail, _ty)] = f"{_kind}_c{_c}_{_p}"
        KERNELS[_P.format(_v, _ty)] = f"stem_c{_c}_{_p}"


def kernel_name(signature):
    """`b200c::bn_infer::k_...<template arguments>` of a demangled kernel signature: no return type, no parameter list."""
    name = signature[signature.index("b200c::bn_infer::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_eval_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted({f for f in re.findall(r"Function (\S+):", out) if f.startswith("_ZN5b200c8bn_infer")})
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(mangled) == len(KERNELS) == 16
    assert names == set(KERNELS), {"without a case": sorted(names - set(KERNELS)), "not in the library": sorted(set(KERNELS) - names)}


def trace_cases():
    """Runs every case of KERNELS once under torch.profiler and prints {case: [b200c::bn_infer kernels]} as JSON."""
    launched = {}
    for case in sorted(set(KERNELS.values())):
        kind, c, params = case.split("_")
        shape = (2, 64, 8, 8) if c == "c64" else (3, 100, 9, 9)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run_kind(kind, *shape, params, seed=50)
            torch.cuda.synchronize()
        launched[case] = sorted({kernel_name(e.name) for e in prof.events()
                                 if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_infer::" in e.name})
    print(json.dumps(launched))
