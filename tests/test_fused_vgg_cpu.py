"""The VGG swap and the stage-end batch-norm sites without a GPU: fuse_model swaps exactly torchvision's VGG class and
keeps the model; vgg11_bn .. vgg19_bn run 5 stage-end sites and 3, 5, 8 or 11 ReLU sites (all their batch norms) and
plain vgg16 none; at every hook position the modules run and each hook is called as often as in the untouched model;
the CPU fallbacks keep torchvision's bits; `_pool2_fusable` takes exactly nn.MaxPool2d(2, 2); the C-ABI calls reject
every bad argument before any launch; and KERNELS is the library's `b200c::bn_pool2` kernels, none with a stack."""
import copy
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

torchvision = pytest.importorskip("torchvision")
from torchvision.models import vgg  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

# every b200c::bn_pool2 kernel, as the profiler names it, and the case of test_gpu_fused_vgg.trace_cases() that launches it
KERNELS = {
    "b200c::bn_pool2::k_pool2_fwd<8>": "train_vec",
    "b200c::bn_pool2::k_pool2_bwd_reduce<4>": "train_vec",
    "b200c::bn_pool2::k_pool2_bwd_elemt<8>": "train_vec",
    "b200c::bn_pool2::k_pool2_fwd<1>": "train_scalar",
    "b200c::bn_pool2::k_pool2_bwd_reduce<1>": "train_scalar",
    "b200c::bn_pool2::k_pool2_bwd_elemt<1>": "train_scalar",
    "b200c::bn_pool2::k_pool2_infer<8, float>": "eval_vec_fp32",
    "b200c::bn_pool2::k_pool2_infer<1, float>": "eval_scalar_fp32",
    "b200c::bn_pool2::k_pool2_infer<8, __nv_bfloat16>": "eval_vec_bf16",
    "b200c::bn_pool2::k_pool2_infer<1, __nv_bfloat16>": "eval_scalar_bf16",
}

# model -> (stage-end sites, ReLU sites)
SITES = {"vgg11_bn": (5, 3), "vgg13_bn": (5, 5), "vgg16_bn": (5, 8), "vgg19_bn": (5, 11), "vgg16": (0, 0)}


def make_model(arch, num_classes=10):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=num_classes)


def inputs(seed=1, size=32):
    return torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("arch", list(SITES))
def test_fuse_model_swaps_exact_classes_keeps_the_model_and_is_idempotent(arch):
    model = make_model(arch)
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    before = [type(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    after = [type(m) for m in model.modules()]
    assert after == [fused_norm.FusedVGG if t is vgg.VGG else t for t in before]
    assert after.count(fused_norm.FusedVGG) == 1
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == after


def test_subclasses_are_not_swapped():
    class Net(vgg.VGG):
        pass

    model = nn.ModuleList([Net(nn.Sequential(nn.Conv2d(3, 8, 3)), num_classes=2), make_model("vgg11_bn")])
    fused_norm.fuse_model(model)
    assert type(model[0]) is Net and type(model[1]) is fused_norm.FusedVGG


def count_sites(model, x, monkeypatch, train=True):
    """The site entry points one forward calls: bn_relu_maxpool and bn_relu (the stage end's fallback calls bn_relu
    inside it, which is not a site of its own)."""
    counts = {"pool": 0, "relu": 0}
    depth = []

    def counting(key, real):
        def call(*a, **k):
            if not depth:
                counts[key] += 1
            depth.append(key)
            try:
                return real(*a, **k)
            finally:
                depth.pop()
        return call

    for name, key in (("bn_relu_maxpool", "pool"), ("bn_relu", "relu")):
        monkeypatch.setattr(fused_norm, name, counting(key, getattr(fused_norm, name)))
    model.train(train)
    with torch.no_grad() if not train else torch.enable_grad():
        model(x)
    return counts


@pytest.mark.parametrize("arch", list(SITES))
def test_every_batch_norm_is_one_site(arch, monkeypatch):
    model = fused_norm.fuse_model(make_model(arch))
    counts = dict(count_sites(model, inputs(), monkeypatch))
    assert (counts["pool"], counts["relu"]) == SITES[arch]
    n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in model.modules())
    assert sum(counts.values()) == n_bn
    monkeypatch.undo()
    # eval without gradients recorded walks the same sites
    assert count_sites(model, inputs(), monkeypatch, train=False) == counts


def run(model, x, train):
    """Logits, and with `train` every parameter's gradient from one backward pass of the summed logits."""
    model.train(train)
    out = model(x)
    if train:
        out.float().sum().backward()
    return out


def compare(ref, fused, x, train=True):
    torch.manual_seed(7)   # the classifier's dropout draws the same masks in both models
    want = run(ref, x, train)
    torch.manual_seed(7)
    got = run(fused, x, train)
    assert torch.equal(want, got)
    if train:
        for (k, a), (_, b) in zip(ref.named_parameters(), fused.named_parameters()):
            assert torch.equal(a.grad, b.grad), k
    for (k, a), (_, b) in zip(ref.named_buffers(), fused.named_buffers()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("arch", ["vgg11_bn", "vgg16"])
def test_swapped_model_computes_torchvision_s_bits_on_the_cpu(arch, train):
    ref = make_model(arch)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    compare(ref, fused, inputs(), train)
    if train:   # a second step from the updated running statistics
        compare(ref, fused, inputs(seed=2), train)


def test_eval_with_gradients_recorded_runs_the_parent_forward(monkeypatch):
    seen = []
    monkeypatch.setattr(fused_norm, "bn_relu_maxpool", lambda *a: seen.append(1))
    monkeypatch.setattr(fused_norm, "bn_relu", lambda *a: seen.append(1))
    model = fused_norm.fuse_model(make_model("vgg11_bn")).eval()
    model(inputs())
    assert seen == []


def hook_positions(model):
    f = model.features
    return {"features": f, "conv": f[0], "bn": f[1], "relu": f[2], "pool": f[3], "inner_bn": f[5], "inner_relu": f[6],
            "avgpool": model.avgpool, "classifier": model.classifier}


# the positions where the untouched model runs a full backward hook (no inplace ReLU modifies the hooked output)
BACKWARD_HOOKABLE = {"features", "pool", "avgpool", "classifier"}


@pytest.mark.parametrize("kind", ["forward", "pre", "backward"])
@pytest.mark.parametrize("where", [*hook_positions(make_model("vgg11_bn")), "global"])
def test_every_hook_position_runs_the_modules_and_the_hook(where, kind):
    if kind == "backward" and where not in BACKWARD_HOOKABLE:
        pytest.skip("torch refuses a full backward hook whose output an inplace ReLU modifies, in the untouched model too")
    ref = make_model("vgg11_bn")
    fused = fused_norm.fuse_model(copy.deepcopy(ref))

    def register(mod, calls):
        if kind == "forward":
            return mod.register_forward_hook(lambda *a: calls.append(1))
        if kind == "pre":
            return mod.register_forward_pre_hook(lambda *a: calls.append(1))
        return mod.register_full_backward_hook(lambda *a: calls.append(1))

    if where == "global":
        reg = {"forward": nn.modules.module.register_module_forward_hook,
               "pre": nn.modules.module.register_module_forward_pre_hook,
               "backward": nn.modules.module.register_module_full_backward_hook}[kind]
        calls = []
        handle = reg(lambda *a: calls.append(1))
        try:
            compare(ref, fused, inputs(seed=2))
            n_both = len(calls)
            calls.clear()
            torch.manual_seed(7)
            run(ref, inputs(seed=2), True)
            assert n_both == 2 * len(calls)   # the fused model makes every module call of the untouched one, no more
        finally:
            handle.remove()
        return
    calls, ref_calls = [], []
    handle = register(hook_positions(fused)[where], calls)
    ref_handle = register(hook_positions(ref)[where], ref_calls)
    try:
        compare(ref, fused, inputs(seed=2))
    finally:
        handle.remove()
        ref_handle.remove()
    assert len(calls) == len(ref_calls) >= 1


def test_pool2_fusable_takes_exactly_vgg_s_max_pool():
    ok = [nn.MaxPool2d(2, 2), nn.MaxPool2d(2), nn.MaxPool2d((2, 2), (2, 2)), nn.MaxPool2d(2, 2, 0, 1)]
    bad = [nn.MaxPool2d(3, 2, 1), nn.MaxPool2d(2, 1), nn.MaxPool2d(2, 2, 1), nn.MaxPool2d(2, 2, dilation=2),
           nn.MaxPool2d(2, 2, ceil_mode=True), nn.MaxPool2d(2, 2, return_indices=True), nn.MaxPool2d((2, 3), 2),
           nn.MaxPool2d(2, (2, 1)), nn.AvgPool2d(2, 2), nn.AdaptiveMaxPool2d(1)]

    class Sub(nn.MaxPool2d):
        pass

    bad.append(Sub(2, 2))
    hooked = nn.MaxPool2d(2, 2)
    hooked.register_forward_hook(lambda *a: None)
    bad.append(hooked)
    assert all(fused_norm._pool2_fusable(p) for p in ok)
    assert not any(fused_norm._pool2_fusable(p) for p in bad)
    # the stem's predicate is unchanged: it takes neither
    assert not any(fused_norm._pool_fusable(p) for p in ok)


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_cpu_fallback_keeps_eager_bits(train):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 7, 9, generator=g).contiguous(memory_format=torch.channels_last).requires_grad_(train)
    bn = nn.BatchNorm2d(8).train(train)
    ref_bn = copy.deepcopy(bn)
    pool = nn.MaxPool2d(2, 2)
    want = pool(nn.ReLU()(ref_bn(x)))
    got = fused_norm.bn_relu_maxpool(bn, nn.ReLU(inplace=True), pool, x)
    assert torch.equal(got, want) and got.stride() == want.stride()
    assert torch.equal(bn.running_mean, ref_bn.running_mean) and torch.equal(bn.running_var, ref_bn.running_var)
    if train:
        dy = torch.randn(want.shape, generator=g)
        (wx,) = torch.autograd.grad(want, x, dy)
        (gx,) = torch.autograd.grad(got, x, dy)
        assert torch.equal(gx, wx)


@pytest.mark.parametrize("h,w", [(1, 8), (8, 1), (1, 1)])
def test_a_side_of_one_leaves_torch_s_error_to_torch(h, w):
    x = torch.randn(2, 8, h, w)
    with pytest.raises(RuntimeError) as want:
        nn.MaxPool2d(2, 2)(nn.ReLU()(nn.BatchNorm2d(8)(x)))
    with pytest.raises(RuntimeError) as got:
        fused_norm.bn_relu_maxpool(nn.BatchNorm2d(8), nn.ReLU(), nn.MaxPool2d(2, 2), x)
    assert str(got.value) == str(want.value)


def test_pool2_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_vgg_cpu as t; t.pool2_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def pool2_argument_checks():
    lib = N.load()
    p = 16   # never dereferenced: each call is rejected first, or fails to launch without a device
    before = lib.b200c_launch_count()
    fwd_names = ("x", "y", "argmax", "wt", "b", "rm", "rv", "sm", "si", "scratch")
    bwd_names = ("dy", "argmax", "x", "dx", "wt", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("x", "y", "wt", "b", "rm", "rv")
    fp32 = {"wt", "b", "rm", "rv", "sm", "si", "gw", "gb"}

    def ptrs(names, null, at):
        return [None if k in null else at.get(k, p) for k in names]

    def fwd(n=2, h=8, w=8, c=64, at=None, nbt=None, **null):
        a = ptrs(fwd_names, null, at or {})
        return lib.b200c_bn_forward_pool2(*a[:7], nbt, *a[7:9], n, h, w, c, 0.1, 1e-5, a[9], None)

    def bwd(n=2, h=8, w=8, c=64, at=None, **null):
        a = ptrs(bwd_names, null, at or {})
        return lib.b200c_bn_backward_pool2(*a[:9], n, h, w, c, a[9], None)

    def infer(n=2, h=8, w=8, c=64, at=None, bf16=0, **null):
        a = ptrs(inf_names, null, at or {})
        return lib.b200c_bn_infer_pool2(*a, bf16, 1e-5, n, h, w, c, None)

    for call, names in ((fwd, fwd_names), (bwd, bwd_names), (infer, inf_names)):
        # the shape passes; without a device the launch fails
        assert call() == N.ECUDA and call(c=1) == N.ECUDA and call(c=131072, h=2, w=2) == N.ECUDA, call.__name__
        assert call(h=2, w=2) == N.ECUDA and call(h=3, w=5, c=100) == N.ECUDA
        for name in names:
            assert call(**{name: 1}) == N.EINVAL and "null" in N.last_error(), (call.__name__, name)
        for n, h, w, c in ((0, 8, 8, 64), (-1, 8, 8, 64), (2, 1, 8, 64), (2, 8, 1, 64), (2, 0, 8, 64), (2, 8, 8, 0),
                           (2, 8, 8, -1), (2, 8, 8, 131073)):
            assert call(n=n, h=h, w=w, c=c) == N.EINVAL and "bad shape" in N.last_error(), (call.__name__, n, h, w, c)
        # n * h * w * c below 2^31
        assert call(n=1, h=2, w=(1 << 24), c=64) == N.EINVAL and "bad shape" in N.last_error()
        assert call(n=1, h=2, w=(1 << 24) - 1, c=64) == N.ECUDA
        # operands on their element's grid; off the 16-byte grid they take the one-channel kernels
        for name in names:
            if name in ("argmax", "scratch"):
                continue
            off = 2 if name in fp32 else 1
            if call is infer and name in fp32:
                assert call(at={name: p + 2}, bf16=1) == N.ECUDA, name   # bf16 parameters sit on the 2-byte grid
                assert call(at={name: p + 1}, bf16=1) == N.EINVAL and "grid" in N.last_error(), name
            assert call(at={name: p + off}) == N.EINVAL and "grid" in N.last_error(), (call.__name__, name)
            if name not in fp32:
                assert call(at={name: p + 2}) == N.ECUDA, (call.__name__, name)
    assert fwd(nbt=p) == N.ECUDA and fwd(nbt=p + 4) == N.EINVAL and "num_batches_tracked" in N.last_error()
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before


def kernel_name(signature):
    name = signature[signature.index("b200c::bn_pool2::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_pool2_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (_ZN5b200c8bn_pool2\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(usage)), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(usage) == len(KERNELS) == 10
    assert names == set(KERNELS)
    assert all(v == "0" for v in usage.values()), usage
