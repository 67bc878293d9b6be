"""fuse_model and the ReLU6 / SiLU / Hardswish batch-norm sites without a GPU: the class swap keeps the model, the
swapped blocks compute their parent's bits where nothing is fused (CPU, NCHW, fp32), hooks decide between bn_act and
the parent's forward, and the three C-ABI calls reject bad arguments before any launch."""
import copy
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

torchvision = pytest.importorskip("torchvision")
from torchvision.ops.misc import Conv2dNormActivation  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["mobilenet_v2", "mobilenet_v3_small", "efficientnet_b0", "regnet_y_400mf"]


def make_model(arch):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10)


@pytest.mark.parametrize("arch", MODELS)
def test_fuse_model_keeps_the_model_and_is_idempotent(arch):
    model = make_model(arch)
    hook_calls = []
    blocks = [m for m in model.modules() if type(m) is Conv2dNormActivation]
    swapped = [m for m in blocks if len(m) == 3 and type(m[2]) in (nn.ReLU6, nn.SiLU, nn.Hardswish)]
    blocks[0].register_forward_hook(lambda *a: hook_calls.append(1))
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    # blocks ending in ReLU or without an activation keep torchvision's class
    assert all((type(m) is fused_norm.FusedConv2dNormActivation) == (m in swapped) for m in blocks)
    assert bool(swapped) == (arch != "regnet_y_400mf")
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    classes = [type(m) for m in model.modules()]
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == classes
    with torch.no_grad():
        model.eval()(torch.zeros(1, 3, 32, 32))
    assert hook_calls == [1]


def test_only_exact_conv2d_norm_activation_is_swapped():
    class Sub(Conv2dNormActivation):
        pass

    model = nn.Sequential(Conv2dNormActivation(3, 8, activation_layer=nn.SiLU), Sub(8, 8, activation_layer=nn.SiLU),
                          torchvision.models.resnet18(num_classes=10), Conv2dNormActivation(8, 8),
                          Conv2dNormActivation(8, 8, activation_layer=None))
    fused_norm.fuse_model(model)
    assert type(model[0]) is fused_norm.FusedConv2dNormActivation and type(model[1]) is Sub
    assert type(model[2]) is fused_norm.FusedResNet   # fuse_model includes fuse_resnet
    assert type(model[3]) is Conv2dNormActivation and type(model[4]) is Conv2dNormActivation   # ReLU, no activation


@pytest.mark.parametrize("arch", MODELS)
def test_swapped_blocks_compute_the_parent_s_bits_on_the_cpu(arch):
    ref = make_model(arch)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    x = torch.randn(2, 3, 48, 48, generator=torch.Generator().manual_seed(1))
    for train in (True, False):
        ref.train(train), fused.train(train)
        torch.manual_seed(5)
        want = ref(x)
        torch.manual_seed(5)
        got = fused(x)
        assert torch.equal(got, want), train
        if train:
            want.sum().backward()
            got.sum().backward()
            for (k, a), (_, b) in zip(ref.named_parameters(), fused.named_parameters()):
                assert torch.equal(a.grad, b.grad), k
    for a, b in zip(ref.buffers(), fused.buffers()):
        assert torch.equal(a, b)


@pytest.fixture
def bn_act_calls(monkeypatch):
    calls = []
    real = fused_norm.bn_act

    def spy(bn, act, x):
        calls.append(type(act))
        return real(bn, act, x)
    monkeypatch.setattr(fused_norm, "bn_act", spy)
    return calls


@pytest.mark.parametrize("act", [nn.ReLU6, nn.SiLU, nn.Hardswish])
@pytest.mark.parametrize("hooked", [None, "block", "conv", "bn", "act", "bn_pre", "global"])
def test_hooks_decide_between_the_site_and_the_parent_forward(act, hooked, bn_act_calls):
    block = fused_norm.fuse_model(Conv2dNormActivation(3, 8, activation_layer=act)).train()
    ran = []
    target = {"block": block, "conv": block[0], "bn": block[1], "act": block[2], "bn_pre": block[1]}.get(hooked)
    if hooked == "bn_pre":
        target.register_forward_pre_hook(lambda *a: ran.append(hooked))
    elif target is not None:
        target.register_forward_hook(lambda *a: ran.append(hooked))
    handle = nn.modules.module.register_module_forward_hook(lambda *a: ran.append("global")) if hooked == "global" else None
    try:
        x = torch.randn(2, 3, 8, 8)
        want = block[2](block[1](block[0](x)))
        got = block(x)
    finally:
        if handle is not None:
            handle.remove()
    assert torch.equal(got, want)
    assert bn_act_calls == [act]   # bn_act itself falls back to the modules' calls where one of them is hooked
    if hooked is not None:
        assert hooked in ran   # a hook is never skipped: either the site does not run, or the hook is outside it


@pytest.mark.parametrize("case", ["two_modules", "eval_with_grad", "gelu", "relu", "conv_subclass"])
def test_other_blocks_run_the_parent_forward(case, bn_act_calls):
    if case == "two_modules":
        block = Conv2dNormActivation(3, 8, activation_layer=None)
    elif case == "gelu":
        block = Conv2dNormActivation(3, 8, activation_layer=nn.GELU, inplace=None)
    elif case == "relu":
        block = Conv2dNormActivation(3, 8)
    else:
        block = Conv2dNormActivation(3, 8, activation_layer=nn.SiLU)
    if case == "conv_subclass":
        class Conv(nn.Conv2d):
            pass
        block[0].__class__ = Conv
    block.__class__ = fused_norm.FusedConv2dNormActivation   # as if swapped, whatever fuse_model would do
    block.train(case != "eval_with_grad")
    block(torch.randn(2, 3, 8, 8))
    assert bn_act_calls == []


def test_bn_act_routes_relu_to_bn_relu_and_leaves_other_activations(monkeypatch):
    seen = []
    monkeypatch.setattr(fused_norm, "bn_relu", lambda bn, relu, x: seen.append("bn_relu") or relu(bn(x)))
    bn, x = nn.BatchNorm2d(4), torch.randn(2, 4, 3, 3)
    fused_norm.bn_act(bn, nn.ReLU(), x)
    assert seen == ["bn_relu"]
    gelu = nn.GELU()
    assert torch.equal(fused_norm.bn_act(copy.deepcopy(bn), gelu, x), gelu(copy.deepcopy(bn)(x)))


def test_act_calls_reject_bad_arguments_before_any_launch():
    # as test_native_abi_infer: a made-up pointer in a process that sees no CUDA device
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_act_cpu as t; t.act_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def act_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()
    fwd_names = ("x", "y", "wt", "b", "rm", "rv", "sm", "si", "scratch")
    bwd_names = ("dy", "x", "g", "dx", "wt", "b", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("x", "y", "wt", "b", "rm", "rv")

    def fwd(m=64, c=8, act=N.ACT_SILU, **null):
        a = {k: None if k in null else p for k in fwd_names}
        return lib.b200c_bn_forward_act(a["x"], a["y"], a["wt"], a["b"], a["rm"], a["rv"], None, a["sm"], a["si"], act, m, c, 0.1,
                                        1e-5, a["scratch"], None)

    def bwd(m=64, c=8, act=N.ACT_SILU, **null):
        a = {k: None if k in null else p for k in bwd_names}
        return lib.b200c_bn_backward_act(a["dy"], a["x"], a["g"], a["dx"], a["wt"], a["b"], a["sm"], a["si"], a["gw"], a["gb"], act, m, c,
                                         a["scratch"], None)

    def infer(m=64, c=8, act=N.ACT_SILU, bf16=0, **null):
        a = {k: None if k in null else p for k in inf_names}
        return lib.b200c_bn_infer_act(a["x"], a["y"], a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-5, act, m, c, None)

    for call, names, site in ((fwd, fwd_names, "batch norm act"), (bwd, bwd_names, "batch norm act"),
                              (infer, inf_names, "batch norm infer act")):
        for act in (0, 4, -1, 1 << 20):
            assert call(act=act) == N.EINVAL and "unknown act" in N.last_error(), (call.__name__, act)
        # 1 <= channels <= 131072, m >= 1, fewer than 2^31 elements
        for m, c in ((0, 8), (-1, 8), (64, 0), (64, -8), (64, 131073), (1 << 28, 8), (65536, 32768), (2, 1 << 30)):
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
            assert site in N.last_error()
        for name in names:
            assert call(**{name: 1}) == N.EINVAL, (call.__name__, name)
            assert "null" in N.last_error()
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before
    # the largest accepted shapes get past the checks: without a device the launch itself fails, as a CUDA error
    assert infer(m=16383, c=131072) == N.ECUDA
    assert infer(m=(1 << 31) - 1, c=1) == N.ECUDA
    assert lib.b200c_launch_count() == before
