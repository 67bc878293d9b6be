"""fuse_model and the inverted-residual projection sites without a GPU: the class swap keeps the model and touches
neither Conv2dNormActivation nor RegNet, the swapped blocks compute their parent's bits where nothing is fused (CPU,
NCHW, fp32), hooks and module types decide between bn_res and the parent's forward, and the three C-ABI calls reject
bad arguments before any launch."""
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
from torchvision.models import efficientnet, mobilenetv2, mobilenetv3  # noqa: E402
from torchvision.ops.misc import Conv2dNormActivation  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["mobilenet_v2", "mobilenet_v3_small", "mobilenet_v3_large", "efficientnet_b0"]
PARENTS = (mobilenetv2.InvertedResidual, mobilenetv3.InvertedResidual, efficientnet.MBConv)


def make_model(arch, **kw):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10, **kw)


@pytest.mark.parametrize("arch", MODELS)
def test_fuse_model_swaps_the_blocks_and_keeps_the_model(arch):
    model = make_model(arch)
    blocks = [m for m in model.modules() if type(m) in PARENTS]
    plain = [m for m in model.modules() if type(m) is Conv2dNormActivation and len(m) == 2]
    hook_calls = []
    blocks[-1].register_forward_hook(lambda *a: hook_calls.append(1))
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    assert blocks and all(type(b) is fused_norm._RES_SWAP[type(b).__mro__[1]] for b in blocks)
    # the projections (Conv2dNormActivation without activation) keep torchvision's class
    assert all(type(m) is Conv2dNormActivation for m in plain)
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    classes = [type(m) for m in model.modules()]
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == classes
    with torch.no_grad():
        model.eval()(torch.zeros(1, 3, 32, 32))
    assert hook_calls == [1]


def test_only_exact_classes_are_swapped_and_regnet_is_untouched():
    class Sub(mobilenetv2.InvertedResidual):
        pass

    model = nn.Sequential(mobilenetv2.InvertedResidual(8, 8, 1, 6), Sub(8, 8, 1, 6), make_model("regnet_y_400mf"))
    regnet_classes = [type(m) for m in model[2].modules()]
    fused_norm.fuse_model(model)
    assert type(model[0]) is fused_norm.FusedInvertedResidualV2 and type(model[1]) is Sub
    assert [type(m) for m in model[2].modules()] == regnet_classes


@pytest.mark.parametrize("arch", MODELS)
def test_swapped_blocks_compute_the_parent_s_bits_on_the_cpu(arch):
    # stochastic depth raised so that rows are dropped at batch 4
    ref = make_model(arch, **({"stochastic_depth_prob": 0.9} if arch.startswith("efficientnet") else {}))
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    x = torch.randn(4, 3, 48, 48, generator=torch.Generator().manual_seed(1))
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


def test_row_noise_is_torchvision_s():
    from torchvision.ops import StochasticDepth, stochastic_depth

    t = torch.ones(16, 3, 2, 2)
    for p in (0.0, 0.1, 0.5, 1.0):
        sd = StochasticDepth(p, "row")
        torch.manual_seed(3)
        want = stochastic_depth(t, p, "row")
        torch.manual_seed(3)
        noise = fused_norm._row_noise(sd, t)
        assert torch.equal(t if noise is None else t * noise, want), p
        assert (noise is None) == (p == 0.0)
        assert fused_norm._row_noise(sd.eval(), t) is None


@pytest.fixture
def bn_res_calls(monkeypatch):
    calls = []
    real = fused_norm.bn_res

    def spy(bn, x, identity=None, noise=None):
        calls.append((identity is not None, noise is not None))
        return real(bn, x, identity, noise)
    monkeypatch.setattr(fused_norm, "bn_res", spy)
    return calls


def small_block(kind):
    if kind == "v2":
        return mobilenetv2.InvertedResidual(8, 8, 1, 2)
    if kind == "v3":
        cnf = mobilenetv3.InvertedResidualConfig(8, 3, 16, 8, True, "HS", 1, 1, 1.0)
        return mobilenetv3.InvertedResidual(cnf, nn.BatchNorm2d)
    cnf = efficientnet.MBConvConfig(2, 3, 1, 8, 8, 1)
    return efficientnet.MBConv(cnf, 0.5, nn.BatchNorm2d)


def parts(block):
    """(sequential, projection Conv2dNormActivation or None, conv, batch norm) of a block."""
    if isinstance(block, mobilenetv2.InvertedResidual):
        return block.conv, None, block.conv[-2], block.conv[-1]
    return block.block, block.block[-1], block.block[-1][0], block.block[-1][1]


@pytest.mark.parametrize("kind", ["v2", "v3", "mbconv"])
@pytest.mark.parametrize("hooked", [None, "block", "conv", "seq", "proj", "bn", "bn_pre", "sd", "global"])
def test_hooks_decide_between_the_site_and_the_parent_forward(kind, hooked, bn_res_calls):
    block = fused_norm.fuse_model(small_block(kind)).train()
    seq, proj, conv, bn = parts(block)
    if hooked == "proj" and proj is None or hooked == "sd" and kind != "mbconv":
        pytest.skip("the block has no such module")
    ran = []
    target = {"block": block, "conv": conv, "seq": seq, "proj": proj, "bn": bn, "bn_pre": bn,
              "sd": getattr(block, "stochastic_depth", None)}.get(hooked)
    if hooked == "bn_pre":
        target.register_forward_pre_hook(lambda *a: ran.append(hooked))
    elif target is not None:
        target.register_forward_hook(lambda *a: ran.append(hooked))
    handle = nn.modules.module.register_module_forward_hook(lambda *a: ran.append("global")) if hooked == "global" else None
    x = torch.randn(4, 8, 6, 6)
    parent = copy.deepcopy(block)
    parent.__class__ = type(block).__mro__[1]
    try:
        torch.manual_seed(2)
        want = parent(x)
        torch.manual_seed(2)
        got = block(x)
    finally:
        if handle is not None:
            handle.remove()
    assert torch.equal(got, want)
    skipped = hooked in ("seq", "proj", "bn", "bn_pre", "sd", "global")
    assert bn_res_calls == ([] if skipped else [(True, kind == "mbconv")])
    if hooked is not None:
        assert hooked in ran   # a hook is never skipped: either the site does not run, or the hook is outside it


@pytest.mark.parametrize("case", ["eval_with_grad", "sync_bn", "batch_mode", "conv_subclass", "bn_subclass", "projection_relu"])
@pytest.mark.parametrize("kind", ["v2", "v3", "mbconv"])
def test_other_blocks_run_the_parent_forward(kind, case, bn_res_calls):
    block = small_block(kind)
    seq, proj, conv, bn = parts(block)
    if case == "batch_mode":
        if kind != "mbconv":
            pytest.skip("no stochastic depth")
        block.stochastic_depth.mode = "batch"
    elif case == "sync_bn":
        bn.__class__ = nn.SyncBatchNorm
    elif case == "conv_subclass":
        conv.__class__ = type("Conv", (nn.Conv2d,), {})
    elif case == "bn_subclass":
        bn.__class__ = type("BN", (nn.BatchNorm2d,), {})
    elif case == "projection_relu":
        seq.append(nn.ReLU())   # the last modules are no longer the convolution and the batch norm
    fused_norm.fuse_model(block)
    block.train(case != "eval_with_grad")
    x = torch.randn(4, 8, 6, 6)
    if case == "sync_bn":   # a SyncBatchNorm's forward wants a GPU input: the block's decision is taken before any module runs
        assert fused_norm._res_forward(block, seq, kind != "v2", x, x) is None
    else:
        block(x)
    assert bn_res_calls == []


def test_bn_res_runs_the_modules_where_nothing_is_fused():
    bn, x, identity = nn.BatchNorm2d(4), torch.randn(2, 4, 3, 3), torch.randn(2, 4, 3, 3)
    noise = torch.tensor([0.0, 2.0]).view(2, 1, 1, 1)
    for args, want in (((), lambda b: b(x)), ((identity,), lambda b: b(x) + identity),
                       ((identity, noise), lambda b: b(x) * noise + identity)):
        b1, b2 = copy.deepcopy(bn), copy.deepcopy(bn)
        assert torch.equal(fused_norm.bn_res(b1, x, *args), want(b2))


def test_res_calls_reject_bad_arguments_before_any_launch():
    # as test_native_abi_infer: a made-up pointer in a process that sees no CUDA device
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_res_cpu as t; t.res_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def res_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()
    fwd_names = ("x", "y", "wt", "b", "rm", "rv", "sm", "si", "scratch")
    bwd_names = ("dy", "x", "g", "dx", "wt", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("x", "y", "wt", "b", "rm", "rv")

    def fwd(m=64, c=8, identity=p, noise=p, rps=16, **null):
        a = {k: None if k in null else p for k in fwd_names}
        return lib.b200c_bn_forward_res(a["x"], identity, noise, rps, a["y"], a["wt"], a["b"], a["rm"], a["rv"], None, a["sm"], a["si"],
                                        m, c, 0.1, 1e-5, a["scratch"], None)

    def bwd(m=64, c=8, noise=p, rps=16, **null):
        a = {k: None if k in null else p for k in bwd_names}
        return lib.b200c_bn_backward_res(a["dy"], noise, rps, a["x"], a["g"], a["dx"], a["wt"], a["sm"], a["si"], a["gw"], a["gb"], m, c,
                                         a["scratch"], None)

    def infer(m=64, c=8, identity=p, bf16=0, **null):
        a = {k: None if k in null else p for k in inf_names}
        return lib.b200c_bn_infer_res(a["x"], identity, a["y"], a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-5, m, c, None)

    for call, names, site in ((fwd, fwd_names, "batch norm res"), (bwd, bwd_names, "batch norm res"),
                              (infer, inf_names, "batch norm infer res")):
        # 1 <= channels <= 131072, m >= 1, fewer than 2^31 elements
        for m, c in ((0, 8), (-1, 8), (64, 0), (64, -8), (64, 131073), (1 << 28, 8), (65536, 32768), (2, 1 << 30)):
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
            assert site in N.last_error()
        for name in names:
            assert call(**{name: 1}) == N.EINVAL, (call.__name__, name)
            assert "null" in N.last_error()
    assert fwd(identity=None) == N.EINVAL and "noise without an identity" in N.last_error()
    for call in (fwd, bwd):
        for rps in (0, -1, 3, 128):   # rows_per_sample below 1 or not dividing m = 64
            assert call(rps=rps) == N.EINVAL and "rows_per_sample" in N.last_error(), (call.__name__, rps)
    assert bwd(noise=None) == N.EINVAL and "g without noise" in N.last_error()
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before
    # the largest accepted shapes get past the checks: without a device the launch itself fails, as a CUDA error
    assert infer(m=16383, c=131072) == N.ECUDA
    assert infer(m=(1 << 31) - 1, c=1, identity=None) == N.ECUDA
    assert fwd(rps=64, noise=p) == N.ECUDA and fwd(noise=None, identity=None, rps=0) == N.ECUDA
    assert bwd(noise=None, g=1) == N.ECUDA
    assert lib.b200c_launch_count() == before
