"""The fused batch-norm sites (fused_norm.py, norm_kernels.cuh) against eager torch, bit for bit.

For every distinct batch-norm shape of ResNet-50, at batch 256 and 32, and for an odd shape (batch 3, 100 channels:
a single-row grid, a partial channel tile and the scalar elementwise path): `BatchNorm2d` -> ReLU and
`BatchNorm2d` -> `+= identity` -> ReLU on bf16 channels-last inputs, forward and backward.  The output, the
running statistics, num_batches_tracked and the gradients of the input, the identity, the weight and the bias must
have the same bits as eager torch's.  Sites that must not run fused (eval mode, fp32, NCHW) fall back without a
native launch."""
import copy

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

pytestmark = pytest.mark.gpu

CL = torch.channels_last
# (C, H, W) of the 53 batch norms of torchvision's resnet50 at 224 x 224
RESNET50_BN_SHAPES = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28),
                      (256, 28, 28), (256, 14, 14), (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]
CASES = [(n, c, h, w) for c, h, w in RESNET50_BN_SHAPES for n in (256, 32)] + [(3, 100, 9, 9)]


def same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    view = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[a.dtype]
    return torch.equal(a.contiguous().view(view), b.contiguous().view(view))


def make_bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
        bn.bias.copy_(0.2 * torch.randn(c, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
        bn.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
        bn.num_batches_tracked.fill_(5)
    return bn.cuda()


def run(bn, x, identity, dy, fused):
    x = x.clone().requires_grad_()
    identity = identity.clone().requires_grad_() if identity is not None else None
    relu = nn.ReLU(inplace=True)
    if fused:
        y = fused_norm.bn_relu(bn, relu, x) if identity is None else fused_norm.bn_add_relu(bn, relu, x, identity)
    else:
        out = bn(x)
        if identity is not None:
            out += identity
        y = relu(out)
    y.backward(dy)
    return {"y": y.detach(), "running_mean": bn.running_mean, "running_var": bn.running_var,
            "num_batches_tracked": bn.num_batches_tracked, "dx": x.grad, "d_identity": identity.grad if identity is not None else None,
            "dweight": bn.weight.grad, "dbias": bn.bias.grad}


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("n,c,h,w", CASES)
def test_fused_site_is_bit_identical_to_eager_torch(n, c, h, w, residual):
    check_site(n, c, h, w, residual)


def test_one_scratch_serves_every_channel_count():
    # A narrow site whose grid merge spans many rows stages its partial sums in the scratch buffer that the
    # semaphores of a later wide site share (one buffer per stream); every site must still merge correctly.
    fused_norm._scratch.clear()
    for n, c, h, w in [(256, 16, 56, 56), (256, 2048, 7, 7), (256, 32, 56, 56), (256, 2048, 7, 7), (3, 100, 9, 9)]:
        for residual in (False, True):
            check_site(n, c, h, w, residual)
    assert len(fused_norm._scratch) == 1


def test_one_value_per_channel_raises_as_torch_does():
    bn = make_bn(64, 0)
    x = torch.randn(1, 64, 1, 1, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    before = N.launch_count()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        fused_norm.bn_relu(bn, nn.ReLU(), x)
    assert N.launch_count() == before


def check_site(n, c, h, w, residual):
    seed = n * 100003 + c * 101 + h + residual
    g = torch.Generator(device="cuda").manual_seed(seed)

    def act(scale, shift):
        return (torch.randn(n, c, h, w, device="cuda", generator=g) * scale + shift).to(torch.bfloat16).contiguous(memory_format=CL)

    x, dy = act(2.0, 0.5), act(1.0, 0.0)
    identity = act(1.0, -0.2) if residual else None
    ref_bn = make_bn(c, seed)
    fused_bn = copy.deepcopy(ref_bn)
    assert torch._C._select_batch_norm_backend(x, ref_bn.weight, ref_bn.bias, ref_bn.running_mean, ref_bn.running_var, True,
                                               ref_bn.eps) == torch._C._BatchNormBackend.Native
    want = run(ref_bn, x, identity, dy, fused=False)
    before = N.launch_count()
    got = run(fused_bn, x, identity, dy, fused=True)
    torch.cuda.synchronize()
    assert N.launch_count() - before == 4, "the site did not run on the fused kernels"
    assert got["y"].is_contiguous(memory_format=CL) and got["dx"].is_contiguous(memory_format=CL)
    bad = [k for k in want if not same_bits(got[k], want[k])]
    assert not bad, f"differs from eager torch: {bad}"


@pytest.mark.parametrize("case", ["eval", "fp32", "nchw"])
def test_ineligible_sites_fall_back_to_torch(case):
    n, c, h, w = 8, 64, 14, 14
    g = torch.Generator(device="cuda").manual_seed(3)
    dtype = torch.float32 if case == "fp32" else torch.bfloat16
    fmt = torch.contiguous_format if case == "nchw" else CL
    x = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
    identity = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
    ref_bn = make_bn(c, 1)
    fused_bn = copy.deepcopy(ref_bn)
    if case == "eval":
        ref_bn.eval()
        fused_bn.eval()
    relu = nn.ReLU()
    before = N.launch_count()
    got = fused_norm.bn_add_relu(fused_bn, relu, x, identity)
    assert N.launch_count() == before, "an ineligible site ran the fused kernels"
    out = ref_bn(x)
    out += identity
    assert same_bits(got, relu(out))
    assert same_bits(fused_bn.running_mean, ref_bn.running_mean) and same_bits(fused_bn.running_var, ref_bn.running_var)
