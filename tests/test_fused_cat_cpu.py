"""The DenseNet swap and the concatenation batch-norm site without a GPU: fuse_model swaps exactly torchvision's
_DenseLayer, _DenseBlock and DenseNet and keeps the model; at every hook position the modules run and the hook is
called; the memory_efficient path and the CPU fallback keep torchvision's bits; the three C-ABI calls reject every bad
argument before any launch; and test_gpu_fused_cat.KERNELS is the library's `b200c::bn_cat` kernels."""
import copy
import ctypes
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
from torchvision.models import densenet  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

# every b200c::bn_cat kernel, as the profiler names it, and the case of test_gpu_fused_cat.trace_cases() that launches it
KERNELS = {
    "b200c::bn_cat::k_cat_stats": "train",
    "b200c::bn_cat::k_cat_transform": "train",
    "b200c::bn_cat::k_cat_bwd_reduce": "train",
    "b200c::bn_cat::k_cat_bwd_elemt": "train",
    "b200c::bn_cat::k_cat_infer<float>": "eval_fp32",
    "b200c::bn_cat::k_cat_infer<__nv_bfloat16>": "eval_bf16",
}


def make_model(arch="densenet121", **kw):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10, **kw)


def test_fuse_model_keeps_the_model_and_is_idempotent():
    model = make_model()
    hook_calls = []
    model.features.denseblock1.denselayer1.register_forward_hook(lambda *a: hook_calls.append(1))
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    assert type(model) is fused_norm.FusedDenseNet
    assert all(type(m) is fused_norm.FusedDenseBlock for m in model.features if isinstance(m, densenet._DenseBlock))
    assert sum(type(m) is fused_norm.FusedDenseLayer for m in model.modules()) == 58
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    classes = [type(m) for m in model.modules()]
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == classes
    with torch.no_grad():
        model.eval()(torch.zeros(1, 3, 32, 32))
    assert hook_calls == [1]


def test_only_exact_classes_are_swapped():
    class Layer(densenet._DenseLayer):
        pass

    class Net(densenet.DenseNet):
        pass

    layer = Layer(64, 32, 4, 0.0)
    net = Net(block_config=(1, 1), num_init_features=16, growth_rate=8)
    model = nn.ModuleList([layer, net])
    fused_norm.fuse_model(model)
    assert type(layer) is Layer and type(net) is Net
    assert type(net.features.denseblock1) is fused_norm.FusedDenseBlock
    assert type(net.features.denseblock1.denselayer1) is fused_norm.FusedDenseLayer


def compare(ref, fused, x, train=True):
    ref.train(train), fused.train(train)
    torch.manual_seed(5)
    want = ref(x)
    torch.manual_seed(5)
    got = fused(x)
    assert torch.equal(got, want)
    if train:
        want.sum().backward()
        got.sum().backward()
        for (k, a), (_, b) in zip(ref.named_parameters(), fused.named_parameters()):
            assert torch.equal(a.grad, b.grad), k
    for (k, a), (_, b) in zip(ref.named_buffers(), fused.named_buffers()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("kw", [{}, {"drop_rate": 0.3}, {"memory_efficient": True}], ids=["plain", "dropout", "memory_efficient"])
@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
def test_swapped_model_computes_torchvision_s_bits_on_the_cpu(kw, train):
    ref = make_model(**kw)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    compare(ref, fused, torch.randn(2, 3, 48, 48, generator=torch.Generator().manual_seed(1)), train)


def test_bn_relu_cat_falls_back_to_cat_and_bn_relu(monkeypatch):
    seen = []
    monkeypatch.setattr(fused_norm, "bn_relu", lambda bn, relu, x: seen.append(x.shape) or relu(bn(x)))
    segs = [torch.randn(2, 8, 3, 3), torch.randn(2, 16, 3, 3)]
    bn = nn.BatchNorm2d(24)
    want = nn.ReLU()(copy.deepcopy(bn)(torch.cat(segs, 1)))
    assert torch.equal(fused_norm.bn_relu_cat(bn, nn.ReLU(), segs), want)
    assert seen == [torch.Size([2, 24, 3, 3])]
    # the functional ReLU of DenseNet.forward (norm5)
    assert torch.equal(fused_norm.bn_relu_cat(copy.deepcopy(bn), None, segs), torch.relu(copy.deepcopy(bn)(torch.cat(segs, 1))))


def positions(model):
    f = model.features
    return {"norm1": f.denseblock1.denselayer2.norm1, "relu1": f.denseblock1.denselayer2.relu1, "block": f.denseblock2,
            "transition": f.transition1, "features": f, "norm5": f.norm5}


@pytest.mark.parametrize("where", ["norm1", "relu1", "block", "transition", "features", "norm5", "global"])
def test_every_hook_position_runs_the_modules_and_the_hook(where, monkeypatch):
    ref = make_model()
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    calls = []
    walks = []
    real_walk = fused_norm._dense_walk
    monkeypatch.setattr(fused_norm, "_dense_walk", lambda f: walks.append(real_walk(f) is not None) or real_walk(f))
    hook = lambda *a: calls.append(1)  # noqa: E731
    if where == "global":
        handle = nn.modules.module.register_module_forward_hook(hook)
    else:
        handle = positions(fused)[where].register_forward_hook(hook)
    try:
        compare(ref, fused, torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(2)))
    finally:
        handle.remove()
    assert calls if where == "global" else calls == [1]
    # the walk skips the calls of `features`, the blocks and transitions: their hooks send the model to the parent
    assert walks == [where not in ("block", "transition", "features")]


def test_memory_efficient_runs_the_parent_forward_where_torchvision_checkpoints(monkeypatch):
    seen = []
    real = fused_norm.bn_relu_cat
    monkeypatch.setattr(fused_norm, "bn_relu_cat", lambda *a: seen.append(1) or real(*a))
    model = fused_norm.fuse_model(make_model(memory_efficient=True))
    layer = model.features.denseblock1.denselayer1
    x = torch.randn(2, 64, 8, 8, requires_grad=True)
    layer([x]).sum().backward()
    assert seen == []   # checkpointed: torchvision's bn_function
    with torch.no_grad():
        layer([x.detach()])
    assert seen == [1]  # nothing to checkpoint: the site


def test_cat_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_cat_cpu as t; t.cat_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def cat_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def table(chans, ptrs=None):
        k = len(chans)
        ptrs = ptrs or [16 * (i + 1) for i in range(k)]
        return (ctypes.c_void_p * max(k, 1))(*ptrs), (ctypes.c_int * max(k, 1))(*chans), k

    fwd_names = ("y", "mask", "wt", "b", "rm", "rv", "sm", "si", "scratch")
    bwd_names = ("dy", "mask", "dx", "wt", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("y", "wt", "b", "rm", "rv")

    def fwd(m=64, c=48, chans=(32, 16), tab=None, **null):
        a = {k: None if k in null else (null.get("at", {}).get(k) or p) for k in fwd_names}
        return lib.b200c_bn_forward_cat(*(tab or table(chans)), a["y"], a["mask"], a["wt"], a["b"], a["rm"], a["rv"], None, a["sm"], a["si"],
                                        m, c, 0.1, 1e-5, a["scratch"], None)

    def bwd(m=64, c=48, chans=(32, 16), tab=None, **null):
        a = {k: None if k in null else (null.get("at", {}).get(k) or p) for k in bwd_names}
        return lib.b200c_bn_backward_cat(a["dy"], a["mask"], *(tab or table(chans)), a["dx"], a["wt"], a["sm"], a["si"], a["gw"], a["gb"],
                                         m, c, a["scratch"], None)

    def infer(m=64, c=48, chans=(32, 16), tab=None, bf16=0, **null):
        a = {k: None if k in null else (null.get("at", {}).get(k) or p) for k in inf_names}
        return lib.b200c_bn_infer_cat(*(tab or table(chans)), a["y"], a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-5, m, c, None)

    for call, names, site in ((fwd, fwd_names, "batch norm cat"), (bwd, bwd_names, "batch norm cat"),
                              (infer, inf_names, "batch norm infer cat")):
        for name in names:
            assert call(**{name: 1}) == N.EINVAL and "null" in N.last_error(), (call.__name__, name)
        # a null segment table, and a null segment
        assert call(tab=(None, None, 2)) == N.EINVAL and "null segment table" in N.last_error()
        assert call(tab=table((32, 16), [16, 0])) == N.EINVAL and "segment 1 is null" in N.last_error()
        # 1..64 segments
        assert call(tab=table(())) == N.EINVAL and "nsegs=0" in N.last_error()
        assert call(c=520, tab=table((8,) * 65)) == N.EINVAL and "nsegs=65" in N.last_error()
        assert call(c=512, tab=table((8,) * 64)) == N.ECUDA   # 64 segments pass the checks; without a device the launch fails
        # the channels add up, each a positive multiple of 8, each segment on the 16-byte grid
        assert call(c=56) == N.EINVAL and "sum to 48" in N.last_error()
        for chans in ((36, 12), (32, 0), (56, -8)):
            assert call(chans=chans) == N.EINVAL and "not a positive multiple of 8" in N.last_error(), chans
        assert call(tab=table((32, 16), [16, 40])) == N.EINVAL and "segment 1 is off the 16-byte grid" in N.last_error()
        # the whole-tensor operands on the grid
        out = "y" if call is not bwd else "dx"
        assert call(at={out: 24}) == N.EINVAL and "off the 16-byte grid" in N.last_error()
        # channels 1..131072, fewer than 2^31 elements, m >= 2 in training (m >= 1 in eval)
        for m, c in ((64, 0), (64, -8), (64, 131080), (1 << 28, 8), (0, 48), (-1, 48)):
            assert call(m=m, c=c, chans=(max(c, 8),)) == N.EINVAL and site in N.last_error(), (call.__name__, m, c)
        assert call(m=1) == (N.EINVAL if call is not infer else N.ECUDA), call.__name__
    assert bwd(at={"dy": 8}) == N.EINVAL and "off the 16-byte grid" in N.last_error()
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before


def kernel_name(signature):
    name = signature[signature.index("b200c::bn_cat::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_cat_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (_ZN5b200c6bn_cat\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(usage)), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(usage) == len(KERNELS) == 6
    assert names == set(KERNELS)
    assert all(v == "0" for v in usage.values()), usage
