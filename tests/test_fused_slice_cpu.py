"""The Inception and GoogLeNet swaps and the slice batch-norm sites without a GPU: fuse_model swaps exactly
torchvision's BasicConv2d and Inception module classes and keeps the model; at every hook position the modules run
and the hook is called; the CPU fallbacks keep torchvision's bits; the three C-ABI calls reject every bad argument
before any launch; and KERNELS is the library's `b200c::bn_slice` kernels, none with a stack."""
import copy
import importlib
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
inception = importlib.import_module("torchvision.models.inception")
googlenet = importlib.import_module("torchvision.models.googlenet")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

# every b200c::bn_slice kernel, as the profiler names it, and the case of test_gpu_fused_slice.trace_cases() that
# launches it
KERNELS = {
    "b200c::bn_slice::k_slice_transform": "train",
    "b200c::bn_slice::k_slice_bwd_reduce": "train",
    "b200c::bn_slice::k_slice_bwd_elemt": "train",
    "b200c::bn_slice::k_slice_infer<float>": "eval_fp32",
    "b200c::bn_slice::k_slice_infer<__nv_bfloat16>": "eval_bf16",
}

# fused class of every torchvision class fuse_model swaps here
SWAPS = {inception.BasicConv2d: fused_norm.FusedInceptionBasicConv2d, googlenet.BasicConv2d: fused_norm.FusedGoogLeNetBasicConv2d,
         inception.InceptionA: fused_norm.FusedInceptionA, inception.InceptionB: fused_norm.FusedInceptionB,
         inception.InceptionC: fused_norm.FusedInceptionC, inception.InceptionD: fused_norm.FusedInceptionD,
         inception.InceptionE: fused_norm.FusedInceptionE, googlenet.Inception: fused_norm.FusedInception}


def make_model(arch, **kw):
    torch.manual_seed(0)
    kw.setdefault("init_weights", True)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10, **kw)


@pytest.mark.parametrize("arch,counts", [("googlenet", {googlenet.BasicConv2d: 59, googlenet.Inception: 9}),
                                         ("inception_v3", {inception.BasicConv2d: 96, inception.InceptionA: 3, inception.InceptionB: 1,
                                                           inception.InceptionC: 4, inception.InceptionD: 1, inception.InceptionE: 2})])
def test_fuse_model_swaps_exact_classes_keeps_the_model_and_is_idempotent(arch, counts):
    model = make_model(arch, aux_logits=True)
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    before = [type(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    after = [type(m) for m in model.modules()]
    assert after == [SWAPS.get(t, t) for t in before]
    for cls, n in counts.items():
        assert after.count(SWAPS[cls]) == n, cls
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == after


def test_subclasses_are_not_swapped():
    class Block(inception.BasicConv2d):
        pass

    class Mixed(inception.InceptionA):
        pass

    model = nn.ModuleList([Block(8, 8, kernel_size=1), Mixed(16, 8), googlenet.Inception(16, 8, 8, 8, 8, 8, 8)])
    fused_norm.fuse_model(model)
    assert type(model[0]) is Block and type(model[1]) is Mixed
    assert type(model[1].branch1x1) is fused_norm.FusedInceptionBasicConv2d
    assert type(model[2]) is fused_norm.FusedInception


def run(model, x, train):
    """Outputs, and with `train` every parameter's gradient from one backward pass of the summed logits."""
    model.train(train)
    torch.manual_seed(5)
    out = model(x)
    logits = out if isinstance(out, torch.Tensor) else [t for t in out if t is not None]
    if train:
        sum(t.float().sum() for t in ([logits] if isinstance(logits, torch.Tensor) else logits)).backward()
    return logits


def compare(ref, fused, x, train=True):
    want, got = run(ref, x, train), run(fused, x, train)
    if isinstance(want, torch.Tensor):
        want, got = [want], [got]
    assert len(want) == len(got) and all(torch.equal(a, b) for a, b in zip(want, got))
    if train:
        for (k, a), (_, b) in zip(ref.named_parameters(), fused.named_parameters()):
            assert torch.equal(a.grad, b.grad), k
    for (k, a), (_, b) in zip(ref.named_buffers(), fused.named_buffers()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("arch,size", [("googlenet", 64), ("inception_v3", 80)])
def test_swapped_model_computes_torchvision_s_bits_on_the_cpu(arch, size, train):
    ref = make_model(arch, aux_logits=False)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    compare(ref, fused, torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(1)), train)


def test_bn_relu_concat_falls_back_to_the_module_ops_and_cat():
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(2, c, 3, 3, generator=g, requires_grad=True) for c in (8, 16)]
    ready = torch.randn(2, 5, 3, 3, generator=g, requires_grad=True)
    bns = [nn.BatchNorm2d(8), nn.BatchNorm2d(16)]
    ref_bns = copy.deepcopy(bns)
    want = torch.cat([torch.relu(ref_bns[0](xs[0])), ready, torch.relu(ref_bns[1](xs[1]))], 1)
    got = fused_norm.bn_relu_concat([(bns[0], xs[0]), ready, (bns[1], xs[1], ())])
    assert torch.equal(got, want)
    for a, b in zip(bns, ref_bns):
        assert torch.equal(a.running_mean, b.running_mean) and torch.equal(a.running_var, b.running_var)


def hook_positions(arch, model):
    if arch == "googlenet":
        m = model.inception3b
        return {"bn": m.branch2[1].bn, "tail": m.branch1, "inner": m.branch2[0], "sequential": m.branch3, "module": m,
                "standalone": model.conv2}
    m = model.Mixed_7b
    return {"bn": m.branch3x3_2a.bn, "tail": m.branch_pool, "inner": m.branch3x3_1, "module": m, "standalone": model.Conv2d_3b_1x1}


@pytest.mark.parametrize("where", ["bn", "tail", "inner", "sequential", "module", "standalone", "global"])
@pytest.mark.parametrize("arch,size", [("googlenet", 64), ("inception_v3", 80)])
def test_every_hook_position_runs_the_modules_and_the_hook(arch, size, where, monkeypatch):
    ref = make_model(arch, aux_logits=False)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    positions = hook_positions(arch, fused)
    if where not in positions and where != "global":
        pytest.skip(f"{arch} has no branch Sequential")
    hooked = positions.get(where)
    # the modules whose forward bn_relu_concat's callers bypass send their module to the parent's forward
    concats = []
    real = fused_norm.bn_relu_concat
    monkeypatch.setattr(fused_norm, "bn_relu_concat", lambda branches: concats.append(1) or real(branches))
    calls, ref_calls = [], []
    if where == "global":
        handle = nn.modules.module.register_module_forward_hook(lambda *a: calls.append(1))
        try:
            compare(ref, fused, torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(2)))
            n_both = len(calls)
            calls.clear()
            run(ref, torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(2)), True)
            assert n_both == 2 * len(calls)   # the fused model makes every module call of the untouched one, no more
        finally:
            handle.remove()
        assert concats == []
        return
    handle = hooked.register_forward_hook(lambda *a: calls.append(1))
    ref_handle = dict(zip(positions, hook_positions(arch, ref).values()))[where].register_forward_hook(lambda *a: ref_calls.append(1))
    try:
        compare(ref, fused, torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(2)))
    finally:
        handle.remove()
        ref_handle.remove()
    assert calls == ref_calls == [1]
    n_modules = 9 if arch == "googlenet" else 11
    bypassed = where in ("bn", "tail", "sequential")
    assert len(concats) == n_modules - bypassed


def test_eval_with_gradients_recorded_runs_the_parent_forward(monkeypatch):
    seen = []
    monkeypatch.setattr(fused_norm, "bn_relu_concat", lambda branches: seen.append(1))
    model = fused_norm.fuse_model(make_model("googlenet", aux_logits=False)).eval()
    model.inception3a(torch.randn(2, 192, 8, 8))
    assert seen == []
    with torch.no_grad():
        model.inception3a(torch.randn(2, 192, 8, 8))
    assert seen == [1]


def test_slice_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_slice_cpu as t; t.slice_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def slice_argument_checks():
    lib = N.load()
    p = 16   # never dereferenced: each call is rejected first, or fails to launch without a device
    before = lib.b200c_launch_count()
    fwd_names = ("x", "y", "mask", "wt", "b", "rm", "rv", "sm", "si", "scratch")
    bwd_names = ("dy", "mask", "x", "dx", "wt", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("x", "y", "wt", "b", "rm", "rv")

    def ptrs(names, null, at):
        return {k: None if k in null else at.get(k, p) for k in names}

    def fwd(m=64, c=48, ld=96, at=None, **null):
        a = ptrs(fwd_names, null, at or {})
        return lib.b200c_bn_forward_slice(a["x"], a["y"], ld, a["mask"], a["wt"], a["b"], a["rm"], a["rv"], None, a["sm"], a["si"], m, c,
                                          0.1, 1e-3, a["scratch"], None)

    def bwd(m=64, c=48, ld=96, at=None, **null):
        a = ptrs(bwd_names, null, at or {})
        return lib.b200c_bn_backward_slice(a["dy"], ld, a["mask"], a["x"], a["dx"], a["wt"], a["sm"], a["si"], a["gw"], a["gb"], m, c,
                                           a["scratch"], None)

    def infer(m=64, c=48, ld=96, at=None, bf16=0, **null):
        a = ptrs(inf_names, null, at or {})
        return lib.b200c_bn_infer_slice(a["x"], a["y"], ld, a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-3, m, c, None)

    for call, names, site in ((fwd, fwd_names, "batch norm slice"), (bwd, bwd_names, "batch norm slice"),
                              (infer, inf_names, "batch norm infer slice")):
        assert call() == N.ECUDA   # the arguments pass; without a device the launch fails
        assert call(ld=48) == N.ECUDA and call(c=131072, ld=131072, m=16) == N.ECUDA and call(c=8, ld=8) == N.ECUDA
        for name in names:
            assert call(**{name: 1}) == N.EINVAL and "null" in N.last_error(), (call.__name__, name)
        # channels 1..131072 and a multiple of 8
        for c in (0, -8, 131080):
            assert call(c=c, ld=max(c, 8)) == N.EINVAL and "bad shape" in N.last_error(), (call.__name__, c)
        for c in (4, 12, 100):
            assert call(c=c, ld=104) == N.EINVAL and "not a multiple of 8" in N.last_error(), (call.__name__, c)
        # the row stride: a multiple of 8, at least the channels
        for ld in (40, 100, 0, -96):
            assert call(ld=ld) == N.EINVAL and "row stride" in N.last_error(), (call.__name__, ld)
        # m >= 2 in training, m >= 1 in eval; m * c and m * ld below 2^31
        for m in (0, -1):
            assert call(m=m) == N.EINVAL and "bad shape" in N.last_error(), (call.__name__, m)
        assert call(m=1) == (N.EINVAL if call is not infer else N.ECUDA), call.__name__
        assert call(m=1 << 26, c=32, ld=32) == N.EINVAL and "bad shape" in N.last_error()
        assert call(m=(1 << 26) - 1, c=32, ld=32) == N.ECUDA   # m * c = 2^31 - 32
        assert call(m=1 << 24, c=64, ld=128) == N.EINVAL and "row stride" in N.last_error()   # m * c = 2^30, m * ld = 2^31
        assert call(m=(1 << 24) - 1, c=64, ld=128) == N.ECUDA
        # every bf16 operand on the 16-byte grid
        for name in ("x", "y", "dy", "dx"):
            if name in names:
                for off in (2, 8):
                    assert call(at={name: 16 + off}) == N.EINVAL and "16-byte grid" in N.last_error(), (call.__name__, name, off)
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before


def kernel_name(signature):
    name = signature[signature.index("b200c::bn_slice::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_slice_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (_ZN5b200c8bn_slice\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(usage)), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(usage) == len(KERNELS) == 5
    assert names == set(KERNELS)
    assert all(v == "0" for v in usage.values()), usage
