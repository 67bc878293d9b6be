"""Whole torchvision Inception v3 and GoogLeNet models with fused slice sites against the untouched models, bit for bit:
googlenet with its aux heads at 64 x 64, inception_v3 with its aux head at 299 x 299 (the aux head needs Mixed_6e at
17 x 17) and without it at 139 x 139, each after `fuse_model` and after `prepare_model`: three reseeded SGD-momentum
steps under bf16 autocast, channels-last, whose loss sums the main and aux logits' cross-entropies, then an eval
forward under inference_mode.  Losses, gradients, parameters, buffers and logits must have the same bits.  A module
input's gradient is a bf16 sum over its branches, so these also hold the sum's order to eager torch's.

`trace_cases` is the traced code of test_gpu_zz_trace_slice.py."""
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
# case -> (architecture, aux heads, batch, input size)
CASES = {"googlenet": ("googlenet", True, 8, 64), "inception_v3": ("inception_v3", True, 2, 299),
         "inception_v3_no_aux": ("inception_v3", False, 4, 139)}


@pytest.fixture(scope="module")
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def make_model(case):
    import torchvision

    arch, aux = CASES[case][:2]
    torch.manual_seed(0)
    model = getattr(torchvision.models, arch)(weights=None, num_classes=10, aux_logits=aux, init_weights=True)
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


def batches(case, steps=3):
    _, _, n, size = CASES[case]
    g = torch.Generator(device="cuda").manual_seed(3)
    return [(torch.randn(n, 3, size, size, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (n,), device="cuda", generator=g)) for _ in range(steps)]


def loss_of(out, y):
    """The cross-entropy of the main logits plus those of the aux heads, as a user trains with them."""
    logits = [out] if isinstance(out, torch.Tensor) else [t for t in out if t is not None]
    return sum(F.cross_entropy(t.float(), y) for t in logits)


def train_steps(model, data):
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    model.train()
    losses = []
    for i, (x, y) in enumerate(data):
        torch.manual_seed(100 + i)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = loss_of(model(x), y)
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
def test_model_trains_and_evaluates_bit_identically(case, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(case)
    data = batches(case)
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert any(type(m) in (fused_norm.FusedInception, fused_norm.FusedInceptionE) for m in fused.modules())
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


FAMILIES = {"slice_transform": r"b200c::bn_slice::k_slice_transform", "slice_reduce": r"b200c::bn_slice::k_slice_bwd_reduce",
            "slice_elemt": r"b200c::bn_slice::k_slice_bwd_elemt", "bn_stats": r"b200c::bn::k_bn_stats<",
            "bn_transform": r"b200c::bn::k_bn_transform<", "bn_reduce": r"b200c::bn::k_bn_bwd_reduce<",
            "bn_elemt": r"b200c::bn::k_bn_bwd_elemt<",
            "torch_bn": r"batch_norm", "torch_cat": r"CatArrayBatchedCopy", "torch_relu": r"clamp_min|threshold"}


def trace_counts(case):
    """Kernels per family of a bf16-autocast training step of the fused model, the most of three traced steps after one
    untraced step (as test_gpu_zz_dense_models.trace_counts), and the model's batch norms."""
    model = fused_norm.fuse_model(make_model(case)).train()
    (x, y), = batches(case, 1)
    counts = dict.fromkeys(FAMILIES, 0)
    for step in range(4):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.manual_seed(7)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = loss_of(model(x), y)
            loss.backward()
            torch.cuda.synchronize()
        if step:
            names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            for f, p in FAMILIES.items():
                counts[f] = max(counts[f], sum(bool(re.search(p, k)) for k in names))
    counts["batch_norms"] = sum(isinstance(m, nn.BatchNorm2d) for m in model.modules())
    counts["slice_sites"] = sum(len(t) for t in _tails(model))
    return counts


def _tails(model):
    """Each swapped Inception module's branch-ending BasicConv2d blocks (its slice sites)."""
    out = []
    for m in model.modules():
        if type(m) is fused_norm.FusedInception:
            out.append([m.branch1, m.branch2[-1], m.branch3[-1], m.branch4[-1]])
        elif type(m) in (fused_norm.FusedInceptionA, fused_norm.FusedInceptionC):
            out.append([c for n, c in m.named_children() if n in ("branch1x1", "branch5x5_2", "branch3x3dbl_3", "branch_pool",
                                                                 "branch7x7_3", "branch7x7dbl_5")])
        elif type(m) is fused_norm.FusedInceptionB:
            out.append([m.branch3x3, m.branch3x3dbl_3])
        elif type(m) is fused_norm.FusedInceptionD:
            out.append([m.branch3x3_2, m.branch7x7x3_4])
        elif type(m) is fused_norm.FusedInceptionE:
            out.append([m.branch1x1, m.branch3x3_2a, m.branch3x3_2b, m.branch3x3dbl_3a, m.branch3x3dbl_3b, m.branch_pool])
    return out


def trace_cases():
    print(json.dumps({case: trace_counts(case) for case in ("googlenet", "inception_v3")}))
