"""Whole torchvision DenseNets with fused concatenation sites against the untouched models, bit for bit: densenet121
and densenet161 at 64 x 64, and densenet121 with drop_rate > 0 and with memory_efficient=True, after `fuse_model` and
after `prepare_model`: three reseeded SGD-momentum steps under bf16 autocast, channels-last, then an eval forward
under inference_mode.  Losses, gradients, parameters, buffers and logits must have the same bits.

`trace_cases` is the traced code of test_gpu_zz_trace_dense.py."""
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
CASES = {"densenet121": {}, "densenet161": {}, "densenet121_drop": {"drop_rate": 0.2},
         "densenet121_memory_efficient": {"memory_efficient": True}}


@pytest.fixture(scope="module")
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def make_model(case):
    import torchvision

    torch.manual_seed(0)
    model = getattr(torchvision.models, case.split("_")[0])(weights=None, num_classes=10, **CASES[case])
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


def batches(n=8, size=64):
    g = torch.Generator(device="cuda").manual_seed(3)
    return [(torch.randn(n, 3, size, size, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (n,), device="cuda", generator=g)) for _ in range(3)]


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
@pytest.mark.parametrize("case", list(CASES))
def test_densenet_trains_and_evaluates_bit_identically(case, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(case)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert type(fused) is fused_norm.FusedDenseNet
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


FAMILIES = {"cat_stats": r"b200c::bn_cat::k_cat_stats", "cat_transform": r"b200c::bn_cat::k_cat_transform",
            "cat_reduce": r"b200c::bn_cat::k_cat_bwd_reduce", "cat_elemt": r"b200c::bn_cat::k_cat_bwd_elemt",
            "bn_stats": r"b200c::bn::k_bn_stats<", "bn_transform": r"b200c::bn::k_bn_transform<",
            "bn_reduce": r"b200c::bn::k_bn_bwd_reduce<", "pool_fwd": r"b200c::bn::k_bn_pool_fwd<",
            "torch_bn": r"batch_norm", "torch_cat": r"CatArrayBatchedCopy", "torch_relu": r"clamp_min|threshold"}


def trace_counts(case):
    """Kernels per family of a bf16-autocast training step of the fused model, and its site counts.  Every step launches
    the same kernels, and a profiler session now and then arrives without its first kernel records
    (test_gpu_fused_norm_paths.reducing_kernels), so after one untraced step each family counts the most of three
    traced steps."""
    model = fused_norm.fuse_model(make_model(case)).train()
    (x, y), = batches(4, 64)[:1]
    counts = dict.fromkeys(FAMILIES, 0)
    for step in range(4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.manual_seed(7)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            torch.cuda.synchronize()
        if step:
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            for f, p in FAMILIES.items():
                counts[f] = max(counts[f], sum(bool(re.search(p, k)) for k in names))
    layers = [m for m in model.modules() if type(m) is fused_norm.FusedDenseLayer]
    counts["layers"] = len(layers)
    counts["transitions"] = sum(type(m).__name__ == "_Transition" for m in model.modules())
    return counts


def trace_cases():
    print(json.dumps({case: trace_counts(case) for case in ("densenet121", "densenet121_memory_efficient")}))
