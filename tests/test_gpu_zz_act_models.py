"""Whole torchvision models with fused Conv2dNormActivation sites against the untouched models, bit for bit:
mobilenet_v2, mobilenet_v3_large, efficientnet_b0 and regnet_y_400mf (num_classes 10, 96 x 96) after `fuse_model` and
after `prepare_model`, three reseeded SGD-momentum steps under bf16 autocast, channels-last, then an eval forward under
inference_mode.  Losses, gradients, parameters, buffers and logits must have the same bits.  `trace_models` is the
traced code of test_gpu_zz_act_trace.py.

These run after the files with in-process profiler sessions: after these models' steps, a later in-process session
(test_gpu_fused_norm_paths.py) was seen to lose kernel records."""
import copy
import json
import re

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits
from test_gpu_fused_act import ACTS, CODES

CL = torch.channels_last
MODELS = ["mobilenet_v2", "mobilenet_v3_large", "efficientnet_b0", "regnet_y_400mf"]


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


def batches(n=8, size=96):
    g = torch.Generator(device="cuda").manual_seed(3)
    return [(torch.randn(n, 3, size, size, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (n,), device="cuda", generator=g)) for _ in range(3)]


def train_steps(model, data):
    """Three SGD-momentum steps under bf16 autocast, each reseeded (dropout, stochastic depth), then an eval forward
    under inference_mode; returns the losses and the logits."""
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


def sites(model):
    return [m for m in model.modules() if type(m) is fused_norm.FusedConv2dNormActivation]


def mismatches(a_named, b_named):
    a, b = dict(a_named), dict(b_named)
    assert a.keys() == b.keys()
    return [k for k in a if not same_bits(a[k], b[k])]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["fuse_model", "prepare_model"])
@pytest.mark.parametrize("arch", MODELS)
def test_model_trains_and_evaluates_bit_identically(arch, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(arch)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert bool(sites(fused)) == (arch != "regnet_y_400mf")   # regnet's blocks all end in ReLU and stay torchvision's
    before = N.launch_count()
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert (N.launch_count() > before) == bool(sites(fused))
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


def model_trace_counts(arch):
    """Per family, the number of kernels one bf16-autocast training step (forward and backward) launches, fused and
    unfused, the model's fused sites per activation, and how many of them received their gradient in NCHW."""
    counts = {}
    base = make_model(arch)
    (x, y), = batches(4, 64)[:1]
    families = {"act_transform": r"b200c::bn_act::k_act_transform", "act_reduce": r"b200c::bn_act::k_act_bwd_reduce",
                **{f"act_reduce_{a}": rf"k_act_bwd_reduce<\(b200c::bn_act::Act\){code}>" for a, code in CODES.items()},
                "silu": r"::silu_kernel\(", "silu_backward": r"::silu_backward_kernel\(",
                "hardswish": r"::hardswish_kernel\(", "hardswish_backward": r"::hardswish_backward_kernel\(",
                "clamp": r"clamp_scalar", "hardtanh_backward": r"hardtanh_backward_kernel"}
    nchw = []   # per fused site and step: whether its output's gradient arrived in another layout than channels-last
    for name, model in (("unfused", copy.deepcopy(base)), ("fused", fused_norm.fuse_model(copy.deepcopy(base)))):
        model.train()
        if name == "fused":
            # a block's own hook keeps the block fused; it records the layout of each site's incoming gradient
            def record(mod, inputs, out):
                out.register_hook(lambda g: nchw.append(not g.is_contiguous(memory_format=CL)))

            for m in sites(model):
                m.register_forward_hook(record)
        for step in range(2):   # the second step is traced
            nchw.clear()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                torch.manual_seed(7)
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    loss = F.cross_entropy(model(x).float(), y)
                loss.backward()
                torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        counts[name] = {f: sum(bool(re.search(p, k)) for k in names) for f, p in families.items()}
        if name == "fused":
            counts["sites"] = {a: sum(len(m) == 3 and type(m[2]) is cls for m in sites(model)) for a, cls in ACTS.items()}
            counts["nchw_gradient_sites"] = sum(nchw)
    return counts


def trace_models():
    print(json.dumps({arch: model_trace_counts(arch) for arch in MODELS}))
