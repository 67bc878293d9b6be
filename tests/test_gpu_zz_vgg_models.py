"""Whole torchvision VGG-BN models with fused stage ends against the untouched models, bit for bit: vgg11_bn and
vgg16_bn at 64 x 64, each after `fuse_model` and after `prepare_model`: three reseeded SGD-momentum steps under bf16
autocast, channels-last, then an eval forward under inference_mode.  Losses, gradients, parameters, buffers and logits
must have the same bits.

`trace_cases` is the traced code of test_gpu_zz_trace_vgg.py."""
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
ARCHS = ["vgg11_bn", "vgg16_bn"]


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
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    model.train()
    losses = []
    for i, (x, y) in enumerate(data):
        torch.manual_seed(100 + i)   # the classifier's dropout draws the same masks in both models
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
def test_model_trains_and_evaluates_bit_identically(arch, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(arch)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert type(fused) is fused_norm.FusedVGG
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]  # noqa: E731
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


FAMILIES = {"pool2_fwd": r"b200c::bn_pool2::k_pool2_fwd<", "pool2_reduce": r"b200c::bn_pool2::k_pool2_bwd_reduce<",
            "pool2_elemt": r"b200c::bn_pool2::k_pool2_bwd_elemt<", "bn_stats": r"b200c::bn::k_bn_stats<",
            "bn_transform": r"b200c::bn::k_bn_transform<", "bn_reduce": r"b200c::bn::k_bn_bwd_reduce<",
            "bn_elemt": r"b200c::bn::k_bn_bwd_elemt<", "torch_bn": r"batch_norm", "torch_relu": r"clamp_min|threshold",
            "torch_max_pool": r"max_pool"}


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
    print(json.dumps({"vgg16_bn": trace_counts("vgg16_bn")}))
