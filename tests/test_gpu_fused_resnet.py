"""Fused ResNet blocks and models (fused_norm.py) against the untouched torchvision classes, bit for bit.

bf16 autocast on channels-last models, as in the training step.  Per block: torchvision's BasicBlock at stride 1
and at stride 2 with a downsample, and Bottleneck with and without a downsample; the output, the input gradient,
every parameter gradient and every buffer must have the same bits, and each fused site makes 4 native launches.
Per model: resnet18 and resnet50 after `train.prepare_model`, three SGD-momentum steps and an eval forward; the
loss of every step, the parameters, the buffers and the eval output must have the same bits as the untouched model.
A model with bf16 parameters, and an fp32 model without autocast, make no native launch and match too."""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits

torchvision = pytest.importorskip("torchvision")
from torchvision.models.resnet import BasicBlock, Bottleneck  # noqa: E402

pytestmark = pytest.mark.gpu

CL = torch.channels_last
SITES = {"resnet18": 17, "resnet50": 49}   # the stem plus 2 per BasicBlock, 3 per Bottleneck


@pytest.fixture(scope="module", autouse=True)
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def randomize_bn(model, seed):
    # non-trivial affine parameters and running statistics, so that every batch-norm term matters
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                c = m.num_features
                m.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
                m.bias.copy_(0.2 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                m.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
    return model


def mismatches(a_named, b_named):
    a, b = dict(a_named), dict(b_named)
    assert a.keys() == b.keys()
    return [k for k in a if not same_bits(a[k], b[k])]


def make_block(kind, seed):
    torch.manual_seed(seed)
    if kind == "basic":
        return BasicBlock(64, 64), (8, 64, 16, 16), 2
    if kind == "basic_stride2":
        ds = nn.Sequential(nn.Conv2d(64, 128, 1, stride=2, bias=False), nn.BatchNorm2d(128))
        return BasicBlock(64, 128, stride=2, downsample=ds), (8, 64, 16, 16), 2
    if kind == "bottleneck":
        return Bottleneck(256, 64), (8, 256, 14, 14), 3
    ds = nn.Sequential(nn.Conv2d(64, 256, 1, bias=False), nn.BatchNorm2d(256))
    return Bottleneck(64, 64, downsample=ds), (8, 64, 14, 14), 3


def run_block(block, x, dy):
    x = x.clone().requires_grad_()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = block(x)
    out.backward(dy)
    return out.detach(), x.grad


@pytest.mark.parametrize("kind", ["basic", "basic_stride2", "bottleneck", "bottleneck_downsample"])
def test_fused_block_is_bit_identical(kind):
    ref, shape, sites = make_block(kind, 0)
    ref = randomize_bn(ref, 1).cuda().to(memory_format=CL).train()
    fused = fused_norm.fuse_resnet(copy.deepcopy(ref))
    assert type(fused) in (fused_norm.FusedBasicBlock, fused_norm.FusedBottleneck)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        out_shape = ref.eval()(x).shape   # eval mode: the running statistics stay as they are
    ref.train()
    dy = torch.randn(out_shape, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    out_ref, dx_ref = run_block(ref, x, dy)
    before = N.launch_count()
    out, dx = run_block(fused, x, dy)
    torch.cuda.synchronize()
    assert N.launch_count() - before == 4 * sites
    assert same_bits(out, out_ref) and same_bits(dx, dx_ref)
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "parameter gradients differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"


def make_model(arch):
    torch.manual_seed(0)
    return randomize_bn(getattr(torchvision.models, arch)(weights=None, num_classes=10), 1)


def batches():
    g = torch.Generator(device="cuda").manual_seed(3)
    return [(torch.randn(8, 3, 96, 96, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (8,), device="cuda", generator=g)) for _ in range(3)]


def train_steps(model, data, autocast=True, per_step_launches=None):
    """Three SGD-momentum steps, then an eval forward; returns the losses, the eval output and the model."""
    opt = torch.optim.SGD(model.parameters(), lr=0.05, momentum=0.9)
    model.train()
    losses = []
    for x, y in data:
        before = N.launch_count()
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            loss = F.cross_entropy(model(x.to(next(model.parameters()).dtype)).float(), y)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        if per_step_launches is not None:
            assert N.launch_count() - before == per_step_launches
        losses.append(loss.detach())
    model.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        out = model(data[0][0].to(next(model.parameters()).dtype))
    return losses, out


def assert_same_training(got, want, got_model, want_model):
    (got_losses, got_out), (want_losses, want_out) = got, want
    assert [same_bits(a, b) for a, b in zip(got_losses, want_losses)] == [True] * 3, "losses differ"
    assert not mismatches(got_model.named_parameters(), want_model.named_parameters()), "parameters differ"
    assert not mismatches(got_model.named_buffers(), want_model.named_buffers()), "buffers differ"
    assert same_bits(got_out, want_out), "eval output differs"


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_fused_model_trains_bit_identically(arch):
    base = make_model(arch).cuda().to(memory_format=CL)
    data = batches()
    # the reference is reproducible run to run, so a difference below belongs to the fused path
    refs = [copy.deepcopy(base) for _ in range(2)]
    want = [train_steps(r, data) for r in refs]
    assert_same_training(want[0], want[1], refs[0], refs[1])

    fused = train.prepare_model(copy.deepcopy(base), parallel_strategy=None)
    assert type(fused) is fused_norm.FusedResNet
    blocks = [m for m in fused.modules() if isinstance(m, (BasicBlock, Bottleneck))]
    assert blocks and all(type(m) in (fused_norm.FusedBasicBlock, fused_norm.FusedBottleneck) for m in blocks)
    got = train_steps(fused, data, per_step_launches=4 * SITES[arch])
    assert_same_training(got, want[0], fused, refs[0])


@pytest.mark.parametrize("case", ["bf16_params", "fp32_no_autocast"])
def test_ineligible_models_make_no_native_launch(case):
    base = make_model("resnet18").cuda().to(memory_format=CL)
    if case == "bf16_params":
        base = base.to(torch.bfloat16)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data, autocast=False)
    fused = fused_norm.fuse_resnet(copy.deepcopy(base))
    got = train_steps(fused, data, autocast=False, per_step_launches=0)
    assert_same_training(got, want, fused, ref)
