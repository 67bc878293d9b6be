"""Whole torchvision ShuffleNetV2 models with fused block ends against the untouched models, bit for bit:
shufflenet_v2_x0_5, x1_0 and x2_0 at 64 x 64, each after `fuse_model` and after `prepare_model`: three reseeded
SGD-momentum steps under bf16 autocast, channels-last, then an eval forward under inference_mode.  Losses, gradients,
parameters, buffers and logits must have the same bits.  Every block end's output gradient arrives channels-last
where the next module is conv5 or a stride-2 block, and NCHW where it is a stride-1 block, whose SplitBackward concatenates
x1's NCHW gradient with the branch's channels-last one (the block end then copies it channels-last).

`trace_cases` is the traced code of test_gpu_zz_trace_shuffle.py."""
import copy
import json
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits

pytestmark = pytest.mark.gpu
CL = torch.channels_last
ARCHS = ["shufflenet_v2_x0_5", "shufflenet_v2_x1_0", "shufflenet_v2_x2_0"]


@pytest.fixture(scope="module")
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def make_model(arch):
    import torchvision

    torch.manual_seed(0)
    model = getattr(torchvision.models, arch)(weights=None, num_classes=10)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                c = m.num_features
                m.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
                m.bias.copy_(0.2 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                m.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
    return model.cuda().to(memory_format=CL)


def batches(steps=3, n=16, size=64):
    g = torch.Generator(device="cuda").manual_seed(3)
    return [(torch.randn(n, 3, size, size, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (n,), device="cuda", generator=g)) for _ in range(steps)]


def train_steps(model, data):
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    model.train()
    losses = []
    for i, (x, y) in enumerate(data):
        torch.manual_seed(100 + i)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x).float(), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        losses.append(loss.detach())
    model.eval()
    with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
        out = model(data[0][0])
    return losses, out


def mismatches(a_named, b_named):
    a, b = dict(a_named), dict(b_named)
    assert a.keys() == b.keys()
    return [k for k in a if not same_bits(a[k], b[k])]


@pytest.mark.parametrize("entry", ["fuse_model", "prepare_model"])
@pytest.mark.parametrize("arch", ARCHS)
def test_model_trains_and_evaluates_bit_identically(arch, entry, deterministic_cudnn, monkeypatch):
    pytest.importorskip("torchvision")
    base = make_model(arch)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert sum(type(m) is fused_norm.FusedShuffleInvertedResidual for m in fused.modules()) == 16
    layouts = []
    real = fused_norm._rows_of
    monkeypatch.setattr(fused_norm, "_rows_of", lambda dy: layouts.append(fused_norm._activation(dy)) or real(dy))
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"
    # backward order: stage4's last block first.  dy arrives channels-last from conv5's dgrad and from a stride-2 block's
    # two branch convolutions; a stride-1 block hands its predecessor SplitBackward's cat of x1's NCHW gradient and the
    # branch's channels-last one, which torch.cat writes contiguous (NCHW), as in eager torch
    assert layouts == [True, False, False, False, True, *[False] * 7, True, False, False, False] * len(data), layouts


FAMILIES = {"shuffle_transform": r"b200c::bn_shuffle::k_shuffle_transform", "shuffle_reduce": r"b200c::bn_shuffle::k_shuffle_bwd_reduce",
            "shuffle_elemt": r"b200c::bn_shuffle::k_shuffle_bwd_elemt", "bn_stats": r"b200c::bn::k_bn_stats<",
            "bn_stats_dual": r"b200c::bn::k_bn_stats_dual<", "bn_pool": r"b200c::bn::k_bn_pool_fwd<",
            "bn_transform": r"b200c::bn::k_bn_transform<", "bn_reduce": r"b200c::bn::k_bn_bwd_reduce<",
            "bn_elemt": r"b200c::bn::k_bn_bwd_elemt<", "res_transform": r"b200c::bn_res::k_res_transform<",
            "torch_bn": r"batch_norm", "torch_cat": r"CatArrayBatchedCopy", "torch_relu": r"clamp_min|threshold"}


def trace_counts(arch):
    """Kernels per family of a bf16-autocast training step of the fused model, the most of three traced steps after one
    untraced step (as test_gpu_zz_dense_models.trace_counts)."""
    model = fused_norm.fuse_model(make_model(arch)).train()
    (x, y), = batches(1)
    counts = dict.fromkeys(FAMILIES, 0)
    for step in range(4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            torch.cuda.synchronize()
        if step:
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            for f, p in FAMILIES.items():
                counts[f] = max(counts[f], sum(bool(re.search(p, k)) for k in names))
    counts["batch_norms"] = sum(isinstance(m, nn.BatchNorm2d) for m in model.modules())
    return counts


def trace_cases():
    print(json.dumps({arch: trace_counts(arch) for arch in ("shufflenet_v2_x0_5", "shufflenet_v2_x1_0")}))
