"""The ShuffleNetV2 swaps and the shuffle batch-norm sites without a GPU: fuse_model swaps exactly torchvision's
ShuffleNetV2 and InvertedResidual classes and keeps the model; a model's 56 batch norms split into 1 stem, 17 ReLU,
19 plain and 16 tail sites (13 stride-1, 3 stride-2); at every hook position the modules run and each hook is called
as often as in the untouched model; the CPU fallbacks keep torchvision's bits; the C-ABI calls reject every bad
argument before any launch; and KERNELS is the library's `b200c::bn_shuffle` kernels, none with a stack."""
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
from torchvision.models import shufflenetv2  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

# every b200c::bn_shuffle kernel, as the profiler names it, and the case of test_gpu_fused_shuffle.trace_cases() that
# launches it
KERNELS = {
    "b200c::bn_shuffle::k_shuffle_transform<false>": "train_one",
    "b200c::bn_shuffle::k_shuffle_transform<true>": "train_two",
    "b200c::bn_shuffle::k_shuffle_bwd_reduce<false>": "train_one",
    "b200c::bn_shuffle::k_shuffle_bwd_reduce<true>": "train_two",
    "b200c::bn_shuffle::k_shuffle_bwd_elemt<false>": "train_one",
    "b200c::bn_shuffle::k_shuffle_bwd_elemt<true>": "train_two",
    "b200c::bn_shuffle::k_shuffle_infer<false, float>": "eval_one_fp32",
    "b200c::bn_shuffle::k_shuffle_infer<true, float>": "eval_two_fp32",
    "b200c::bn_shuffle::k_shuffle_infer<false, __nv_bfloat16>": "eval_one_bf16",
    "b200c::bn_shuffle::k_shuffle_infer<true, __nv_bfloat16>": "eval_two_bf16",
}

SWAPS = {shufflenetv2.InvertedResidual: fused_norm.FusedShuffleInvertedResidual,
         shufflenetv2.ShuffleNetV2: fused_norm.FusedShuffleNetV2}
ARCHS = ["shufflenet_v2_x0_5", "shufflenet_v2_x1_0", "shufflenet_v2_x1_5", "shufflenet_v2_x2_0"]


def make_model(arch):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10)


def inputs(seed=1, size=64):
    return torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("arch", ARCHS)
def test_fuse_model_swaps_exact_classes_keeps_the_model_and_is_idempotent(arch):
    model = make_model(arch)
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    before = [type(m) for m in model.modules()]
    assert sum(isinstance(m, nn.BatchNorm2d) for m in model.modules()) == 56
    assert fused_norm.fuse_model(model) is model
    after = [type(m) for m in model.modules()]
    assert after == [SWAPS.get(t, t) for t in before]
    assert after.count(fused_norm.FusedShuffleInvertedResidual) == 16 and after.count(fused_norm.FusedShuffleNetV2) == 1
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == after


def test_subclasses_are_not_swapped():
    class Block(shufflenetv2.InvertedResidual):
        pass

    model = nn.ModuleList([Block(8, 8, 1), shufflenetv2.InvertedResidual(8, 16, 2)])
    fused_norm.fuse_model(model)
    assert type(model[0]) is Block and type(model[1]) is fused_norm.FusedShuffleInvertedResidual


def count_sites(model, x, monkeypatch):
    """The site entry points one training forward calls: bn_relu_maxpool, bn_relu, bn_res, and bn_relu_shuffle split
    by its form."""
    counts = {"stem": 0, "relu": 0, "plain": 0, "tail1": 0, "tail2": 0}
    depth = []   # the stem's CPU fallback runs bn_relu inside it, which is not a site of its own

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

    for name, key in (("bn_relu_maxpool", "stem"), ("bn_relu", "relu"), ("bn_res", "plain")):
        monkeypatch.setattr(fused_norm, name, counting(key, getattr(fused_norm, name)))
    real = fused_norm.bn_relu_shuffle

    def shuffle(first, second):
        key = "tail2" if isinstance(first, tuple) else "tail1"
        counts[key] += 1
        return real(first, second)

    monkeypatch.setattr(fused_norm, "bn_relu_shuffle", shuffle)
    model.train()
    model(x)
    return counts


@pytest.mark.parametrize("arch", ARCHS)
def test_every_batch_norm_is_one_site(arch, monkeypatch):
    model = fused_norm.fuse_model(make_model(arch))
    counts = count_sites(model, inputs(), monkeypatch)
    assert counts == {"stem": 1, "relu": 17, "plain": 19, "tail1": 13, "tail2": 3}
    # 1 + 17 + 19 + 13 + 2 * 3 batch norms
    assert sum(counts.values()) + counts["tail2"] == 56


def run(model, x, train):
    """Logits, and with `train` every parameter's gradient from one backward pass of the summed logits."""
    model.train(train)
    out = model(x)
    if train:
        out.float().sum().backward()
    return out


def compare(ref, fused, x, train=True):
    want, got = run(ref, x, train), run(fused, x, train)
    assert torch.equal(want, got)
    if train:
        for (k, a), (_, b) in zip(ref.named_parameters(), fused.named_parameters()):
            assert torch.equal(a.grad, b.grad), k
    for (k, a), (_, b) in zip(ref.named_buffers(), fused.named_buffers()):
        assert torch.equal(a, b), k


@pytest.mark.parametrize("train", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("arch", ["shufflenet_v2_x0_5", "shufflenet_v2_x1_0"])
def test_swapped_model_computes_torchvision_s_bits_on_the_cpu(arch, train):
    ref = make_model(arch)
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    compare(ref, fused, inputs(), train)
    if train:   # a second step from the updated running statistics
        compare(ref, fused, inputs(seed=2), train)


def test_bn_relu_shuffle_falls_back_to_the_module_ops_cat_and_channel_shuffle():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 10, 3, 3, generator=g, requires_grad=True)
    u, t = (torch.randn(2, 5, 3, 3, generator=g, requires_grad=True) for _ in range(2))
    bns = [nn.BatchNorm2d(5), nn.BatchNorm2d(5)]
    ref_bns = copy.deepcopy(bns)
    x1 = x.chunk(2, 1)[0]
    want = shufflenetv2.channel_shuffle(torch.cat((x1, torch.relu(ref_bns[1](t))), 1), 2)
    got = fused_norm.bn_relu_shuffle(x1, (bns[1], t, ()))
    assert torch.equal(got, want) and got.stride() == want.stride()
    (want * want).sum().backward()
    grads = [x.grad.clone(), t.grad.clone()]
    x.grad = t.grad = None
    (got * got).sum().backward()
    assert torch.equal(x.grad, grads[0]) and torch.equal(t.grad, grads[1])
    want = shufflenetv2.channel_shuffle(torch.cat((torch.relu(ref_bns[0](u)), torch.relu(ref_bns[1](t))), 1), 2)
    got = fused_norm.bn_relu_shuffle((bns[0], u, ()), (bns[1], t, ()))
    assert torch.equal(got, want) and got.stride() == want.stride()
    for a, b in zip(bns, ref_bns):
        assert torch.equal(a.running_mean, b.running_mean) and torch.equal(a.running_var, b.running_var)
        assert torch.equal(a.num_batches_tracked, b.num_batches_tracked)


def hook_positions(model):
    s1, s2 = model.stage2[1], model.stage3[0]   # a stride-1 and a stride-2 block
    return {"tail_bn": s1.branch2[6], "tail_relu": s1.branch2[7], "branch2": s1.branch2, "branch1": s2.branch1,
            "branch1_bn": s2.branch1[3], "branch1_relu": s2.branch1[4], "first_bn": s1.branch2[1], "first_relu": s1.branch2[2],
            "dw_bn": s1.branch2[4], "conv": s1.branch2[5], "block": s1, "stage": model.stage2, "conv1": model.conv1,
            "conv1_bn": model.conv1[1], "maxpool": model.maxpool, "conv5": model.conv5, "conv5_relu": model.conv5[2], "fc": model.fc}


# the positions where a hook sends its block (or the model) to the parent's forward
BYPASSED = {"tail_bn", "tail_relu", "branch2", "branch1", "branch1_bn", "branch1_relu"}
# the positions where the untouched model runs a full backward hook (no inplace ReLU modifies the hooked output)
BACKWARD_HOOKABLE = {"branch2", "branch1", "dw_bn", "conv", "block", "stage", "conv1", "maxpool", "conv5", "fc"}


@pytest.mark.parametrize("kind", ["forward", "pre", "backward"])
@pytest.mark.parametrize("where", [*hook_positions(make_model("shufflenet_v2_x0_5")), "global"])
def test_every_hook_position_runs_the_modules_and_the_hook(where, kind, monkeypatch):
    if kind == "backward" and where not in BACKWARD_HOOKABLE:
        pytest.skip("torch refuses a full backward hook whose output an inplace ReLU modifies, in the untouched model too")
    ref = make_model("shufflenet_v2_x0_5")
    fused = fused_norm.fuse_model(copy.deepcopy(ref))
    shuffles = []
    real = fused_norm.bn_relu_shuffle
    monkeypatch.setattr(fused_norm, "bn_relu_shuffle", lambda a, b: shuffles.append(1) or real(a, b))

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
            run(ref, inputs(seed=2), True)
            assert n_both == 2 * len(calls)   # the fused model makes every module call of the untouched one, no more
        finally:
            handle.remove()
        assert shuffles == []
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
    assert len(shuffles) == 16 - (where in BYPASSED)


def test_eval_with_gradients_recorded_runs_the_parent_forward(monkeypatch):
    seen = []
    monkeypatch.setattr(fused_norm, "bn_relu_shuffle", lambda a, b: seen.append(1))
    monkeypatch.setattr(fused_norm, "bn_relu_maxpool", lambda *a: seen.append(1))
    model = fused_norm.fuse_model(make_model("shufflenet_v2_x0_5")).eval()
    model(inputs())
    assert seen == []
    with torch.no_grad():
        model.stage2[1](torch.randn(2, 48, 8, 8))
    assert seen == [1]


def test_shuffle_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_shuffle_cpu as t; t.shuffle_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def shuffle_argument_checks():
    lib = N.load()
    p = 16   # never dereferenced: each call is rejected first, or fails to launch without a device
    before = lib.b200c_launch_count()
    bn_names = ("mask", "wt", "b", "rm", "rv", "sm", "si")
    fwd_names = ("t", "y", "scratch") + bn_names
    bwd_names = ("dy", "t", "mask", "dt", "wt", "sm", "si", "gw", "gb", "scratch")
    inf_names = ("t", "y", "wt", "b", "rm", "rv")

    def ptr(a, k, null):
        return None if k in null else a.get(k, p)

    def fwd(n=4, hw=16, c=58, x1=p, x1_stride=None, u=None, at=None, **null):
        a = at or {}
        x1_stride = 2 * c * hw if x1_stride is None else x1_stride
        ub = [ptr(a, k + "_u", null) for k in bn_names] if u else [None] * 7
        lead = (x1, x1_stride, u, ub[0], *ub[1:5], None, *ub[5:], 0.1, 1e-5)
        tb = [ptr(a, k, null) for k in bn_names]
        return lib.b200c_bn_forward_shuffle(*lead, ptr(a, "t", null), tb[0], *tb[1:5], None, *tb[5:], 0.1, 1e-5, ptr(a, "y", null),
                                            n, hw, c, ptr(a, "scratch", null), None)

    def bwd(m=64, c=58, u=None, at=None, **null):
        a = at or {}
        ub = (u, *(ptr(a, k, null) for k in ("mask_u", "du", "wt_u", "sm_u", "si_u", "gw_u", "gb_u"))) if u else (None,) * 8
        return lib.b200c_bn_backward_shuffle(ptr(a, "dy", null), *ub, *(ptr(a, k, null) for k in bwd_names[1:-1]), m, c,
                                             ptr(a, "scratch", null), None)

    def infer(n=4, hw=16, c=58, x1=p, x1_stride=None, u=None, bf16=0, **null):
        x1_stride = 2 * c * hw if x1_stride is None else x1_stride
        ub = [None if k + "_u" in null else p for k in ("wt", "b", "rm", "rv")] if u else [None] * 4
        return lib.b200c_bn_infer_shuffle(x1, x1_stride, u, *ub, 1e-5, *(None if k in null else p for k in inf_names[:1]),
                                          *(None if k in null else p for k in inf_names[2:]), 1e-5, None if "y" in null else p, bf16,
                                          n, hw, c, None)

    # both forms pass; without a device the launch fails
    for call in (fwd, infer):
        assert call() == N.ECUDA and call(x1=None, u=p) == N.ECUDA
        assert call(c=1, x1_stride=32) == N.ECUDA and call(c=65536, hw=1, n=2) == N.ECUDA
        assert call(x1=None) == N.EINVAL and "exactly one" in N.last_error()
        assert call(u=p) == N.EINVAL and "exactly one" in N.last_error()
        for c in (0, -1, 65537):
            assert call(c=c, x1_stride=2 * max(c, 1) * 16) == N.EINVAL and "bad shape" in N.last_error(), (call.__name__, c)
        for n, hw in ((0, 16), (4, 0), (-1, 16)):
            assert call(n=n, hw=hw) == N.EINVAL and "bad shape" in N.last_error(), (call.__name__, n, hw)
        # one row: training needs two, eval one
        assert call(n=1, hw=1) == (N.EINVAL if call is fwd else N.ECUDA)
        # n * 2B * hw below 2^31
        assert call(n=1 << 10, hw=1 << 10, c=1 << 10, x1=None, u=p) == N.EINVAL and "bad shape" in N.last_error()
        assert call(n=(1 << 10) - 1, hw=1 << 10, c=1 << 10, x1=None, u=p) == N.ECUDA
        # x1's sample stride: at least B * hw, its last element below 2^31
        assert call(x1_stride=58 * 16 - 1) == N.EINVAL and "sample stride" in N.last_error()
        assert call(x1_stride=58 * 16) == N.ECUDA
        assert call(n=3, x1_stride=(1 << 30)) == N.EINVAL and "sample stride" in N.last_error()
        assert call(n=2, x1_stride=(1 << 30)) == N.ECUDA
    for name in fwd_names:
        assert fwd(**{name: 1}) == N.EINVAL and "null" in N.last_error(), name
        assert fwd(x1=None, u=p, **{name: 1}) == N.EINVAL and "null" in N.last_error(), name
    for name in bn_names:
        assert fwd(x1=None, u=p, **{name + "_u": 1}) == N.EINVAL and "null" in N.last_error(), name
        assert fwd(**{name + "_u": 1}) == N.ECUDA   # the one-batch-norm form reads no u pointer
    for name in inf_names:
        assert infer(**{name: 1}) == N.EINVAL and "null" in N.last_error(), name
    for name in ("wt", "b", "rm", "rv"):
        assert infer(x1=None, u=p, **{name + "_u": 1}) == N.EINVAL and "null" in N.last_error(), name
    for bf16 in (2, -1):
        assert infer(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    # the backward: pointers, m >= 2, channels 1..65536, m * 2B below 2^31, dy on the 4-byte grid
    assert bwd() == N.ECUDA and bwd(u=p) == N.ECUDA and bwd(c=1) == N.ECUDA and bwd(c=65536) == N.ECUDA
    for name in bwd_names:
        assert bwd(**{name: 1}) == N.EINVAL and "null" in N.last_error(), name
    for name in ("mask_u", "du", "wt_u", "sm_u", "si_u", "gw_u", "gb_u"):
        assert bwd(u=p, **{name: 1}) == N.EINVAL and "null" in N.last_error(), name
    for m, c in ((1, 58), (0, 58), (64, 0), (64, 65537), (1 << 24, 64)):
        assert bwd(m=m, c=c) == N.EINVAL and "bad shape" in N.last_error(), (m, c)
    assert bwd(m=(1 << 24) - 1, c=64) == N.ECUDA
    for off in (1, 2, 3):
        assert bwd(at={"dy": 16 + off}) == N.EINVAL and "4-byte grid" in N.last_error(), off
    assert bwd(at={"dy": 20}) == N.ECUDA
    assert lib.b200c_launch_count() == before
    # the mask: ceil(B / 8) bytes per row
    for m, c in ((3, 1), (3, 8), (3, 58), (7, 116), (1, 65536)):
        assert lib.b200c_bn_shuffle_mask_bytes(m, c) == m * ((c + 7) // 8)
    for m, c in ((0, 8), (4, 0), (4, 65537), (1 << 24, 128)):
        assert lib.b200c_bn_shuffle_mask_bytes(m, c) == 0


def kernel_name(signature):
    name = signature[signature.index("b200c::bn_shuffle::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_shuffle_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (_ZN5b200c10bn_shuffle\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    demangled = subprocess.run(["c++filt"], input="\n".join(sorted(usage)), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(usage) == len(KERNELS) == 10
    assert names == set(KERNELS)
    assert all(v == "0" for v in usage.values()), usage
