"""The fused batch norm's 1-bit ReLU mask and the block tail's two gradients, against eager torch, bit for bit.

A tail called with `pair=True` returns its output twice; autograd hands the backward each consumer's gradient
apart and the kernel sums them as autograd's bf16 accumulation does.  Checked for every tail shape of ResNet-50 at
batch 256 and one shape per launch regime of the reducing kernels (gpu_common.BN_REGIME_SHAPES), with only one of the two outputs used, with a channel count that has no mask (C % 8 != 0), and at
value edges of the two gradients.  Through the C-ABI: the mask's bits and layout for the vector and the scalar
transform (a guard past the mask stays untouched), and the mask backward against the backward that reads y.  In a
fused resnet50 training step, the blocks chained in pairs leave one elementwise add in the backward, the maxpool
output's, where chaining them one tensor at a time leaves 16."""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values
from test_gpu_fused_norm import make_bn, misaligned

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CL = torch.channels_last
BF16_MAX = torch.finfo(torch.bfloat16).max
TAIL_SHAPES = [(256, 256, 56, 56), (256, 512, 28, 28), (256, 1024, 14, 14), (256, 2048, 7, 7)]


def nhwc(t):
    n, c, h, w = t.shape
    return torch.empty(n, h, w, c, dtype=t.dtype, device=t.device).permute(0, 3, 1, 2).copy_(t)


def gauss(shape, g, scale=1.0, shift=0.0):
    return nhwc((torch.randn(shape, device="cuda", generator=g) * scale + shift).to(torch.bfloat16))


def two_gradient_site(bn, x, identity, dy1, dy2, used, fused):
    """Runs one tail; `used` names the outputs whose gradient is given: "both", "first" or "second"."""
    x, identity = x.clone().requires_grad_(), identity.clone().requires_grad_()
    relu = nn.ReLU(inplace=True)
    if fused:
        y, y_id = fused_norm.bn_add_relu(bn, relu, x, identity, pair=True)
    else:
        out = bn(x)
        out += identity
        y = y_id = relu(out)
    outs, grads = {"both": ([y, y_id], [dy1, dy2]), "first": ([y], [dy1]), "second": ([y_id], [dy2])}[used]
    torch.autograd.backward(outs, grads)
    return {"y": y.detach(), "running_mean": bn.running_mean, "running_var": bn.running_var, "dx": x.grad,
            "d_identity": identity.grad, "dweight": bn.weight.grad, "dbias": bn.bias.grad}


def check_two_gradients(n, c, h, w, used, edges=False):
    g = torch.Generator(device="cuda").manual_seed(n * 7 + c)
    shape = (n, c, h, w)
    x, identity, dy1, dy2 = gauss(shape, g, 2.0, 0.5), gauss(shape, g, 1.0, -0.2), gauss(shape, g), gauss(shape, g)
    if edges:
        # per 8 channels: -0 + -0, -0 + +0, +Inf + -Inf, a sum past the bf16 maximum, NaN in either gradient; the
        # ReLU passes about half of every channel's rows, so each pair meets masked and unmasked positions
        pairs = [(-0.0, -0.0), (-0.0, 0.0), (float("inf"), float("-inf")), (BF16_MAX, BF16_MAX / 2),
                 (float("nan"), None), (None, float("nan")), (0.0, -0.0), (-BF16_MAX, -BF16_MAX)]
        with torch.no_grad():
            for k, (a, b) in enumerate(pairs):
                if a is not None:
                    dy1[:, 8 * k:8 * k + 8] = a
                if b is not None:
                    dy2[:, 8 * k:8 * k + 8] = b
    ref_bn = make_bn(c, c)
    fused_bn = copy.deepcopy(ref_bn)
    want = two_gradient_site(ref_bn, x, identity, dy1, dy2, used, fused=False)
    before = N.launch_count()
    got = two_gradient_site(fused_bn, x, identity, dy1, dy2, used, fused=True)
    torch.cuda.synchronize()
    assert N.launch_count() - before == 4
    for k in want:
        assert_same_values(got[k], want[k], k)


@pytest.mark.parametrize("n,c,h,w", TAIL_SHAPES + [(3, 100, 9, 9)] + list(BN_REGIME_SHAPES))
def test_two_gradients_match_eager_accumulation(n, c, h, w):
    check_two_gradients(n, c, h, w, "both")


@pytest.mark.parametrize("used", ["first", "second"])
@pytest.mark.parametrize("n,c,h,w", [(8, 64, 16, 16), (32, 2048, 7, 7), (3, 100, 9, 9)])
def test_one_gradient_is_taken_as_it_is(n, c, h, w, used):
    check_two_gradients(n, c, h, w, used)


@pytest.mark.parametrize("used", ["both", "first", "second"])
def test_two_gradient_value_edges(used):
    check_two_gradients(8, 64, 16, 16, used, edges=True)


# ---- the mask through the C-ABI ----------------------------------------------------------------------
GUARD = 4096


def expected_mask(y):
    m, c = y.shape
    bits = (~(y.float() <= 0)).to(torch.int32).view(m * c // 8, 8)
    return (bits << torch.arange(8, device=y.device, dtype=torch.int32)).sum(1).to(torch.uint8)


@pytest.mark.parametrize("residual", [False, True])
@pytest.mark.parametrize("m,c", [(2048, 64), (1000, 264), (77, 8), (130, 24), (96, 2048)])
@pytest.mark.parametrize("aligned", [True, False], ids=["vector", "scalar"])
def test_mask_bits_and_mask_backward(m, c, residual, aligned):
    lib = N.load()
    g = torch.Generator(device="cuda").manual_seed(m + c)
    x = (torch.randn(m, c, device="cuda", generator=g) * 2 + 0.3).to(torch.bfloat16)
    x[:, 5] = float("nan")    # a NaN channel: y is NaN, whose gradient the ReLU passes
    x[:, 3] = 0.75            # a constant channel: y = relu(bias) (+ identity)
    if not aligned:
        x = misaligned(x.view(m, 1, 1, c).permute(0, 3, 1, 2)).permute(0, 2, 3, 1).reshape(m, c)
        assert x.data_ptr() % 16 == 2
    identity = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16) if residual else None
    dy = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    dy2 = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    bn = make_bn(c, c)
    w, b = bn.weight.detach(), bn.bias.detach()
    scratch = torch.zeros(int(lib.b200c_bn_scratch_bytes(c)), dtype=torch.uint8, device="cuda")
    out = {}
    for variant in ("y", "mask"):
        rm, rv = bn.running_mean.clone(), bn.running_var.clone()
        y = torch.empty_like(dy)
        mask = torch.full((m * c // 8 + GUARD,), 0xA5, dtype=torch.uint8, device="cuda")
        stats = torch.empty(2, c, device="cuda")
        fwd = (w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(), None, stats[0].data_ptr(), stats[1].data_ptr(), m, c,
               0.1, 1e-5, scratch.data_ptr(), None)
        id_ptr = identity.data_ptr() if residual else None
        dx, d_id = torch.empty_like(dy), torch.empty_like(dy) if residual else None
        dw, db = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
        bwd = (x.data_ptr(), d_id.data_ptr() if residual else None, dx.data_ptr(), w.data_ptr(), stats[0].data_ptr(),
               stats[1].data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, scratch.data_ptr(), None)
        if variant == "y":
            dy_sum = (dy.float() + dy2.float()).to(torch.bfloat16)
            N.check(lib.b200c_bn_forward(x.data_ptr(), id_ptr, y.data_ptr(), *fwd))
            N.check(lib.b200c_bn_backward(dy_sum.data_ptr(), y.data_ptr(), *bwd))
        else:
            N.check(lib.b200c_bn_forward_mask(x.data_ptr(), id_ptr, y.data_ptr(), mask.data_ptr(), *fwd))
            N.check(lib.b200c_bn_backward_mask(dy.data_ptr(), dy2.data_ptr(), mask.data_ptr(), *bwd))
        torch.cuda.synchronize()
        out[variant] = {"y": y, "mask": mask, "dx": dx, "d_identity": d_id, "dweight": dw, "dbias": db, "stats": stats}
    got = out["mask"]
    assert torch.isnan(got["y"][:, 5]).all()
    assert torch.equal(got["mask"][:m * c // 8], expected_mask(got["y"])), "mask bits"
    assert (got["mask"][m * c // 8:] == 0xA5).all(), "a write past the mask"
    for k in ("y", "dx", "d_identity", "dweight", "dbias", "stats"):
        if got[k] is not None:
            assert_same_values(got[k], out["y"][k], k)


# ---- which path the fused resnet50 step runs -------------------------------------------------------
def backward_add_kernels(model, x, target):
    with torch.autocast("cuda", dtype=torch.bfloat16):
        loss = F.cross_entropy(model(x).float(), target)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        loss.backward()
        torch.cuda.synchronize()
    model.zero_grad(set_to_none=True)
    return sorted(e.name for e in prof.events()
                  if e.device_type == torch.autograd.DeviceType.CUDA and "CUDAFunctor_add" in e.name)


def paired_and_chained_add_kernels():
    import torchvision

    torch.manual_seed(0)
    model = fused_norm.fuse_resnet(torchvision.models.resnet50(weights=None, num_classes=10)).cuda().to(memory_format=CL).train()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(2, 3, 64, 64, device="cuda", generator=g).contiguous(memory_format=CL)
    target = torch.randint(0, 10, (2,), device="cuda", generator=g)
    backward_add_kernels(model, x, target)   # warm-up
    paired = backward_add_kernels(model, x, target)
    # a hook on each layer makes the model call the layer as a module, which chains its blocks one tensor at a time
    hooks = [layer.register_forward_hook(lambda mod, args, out: None)
             for layer in (model.layer1, model.layer2, model.layer3, model.layer4)]
    chained = backward_add_kernels(model, x, target)
    for h in hooks:
        h.remove()
    print(json.dumps({"paired": paired, "chained": chained}))


def test_paired_blocks_leave_only_the_maxpool_accumulation():
    pytest.importorskip("torchvision")
    # in a process of its own, so that this whole-model profiler session shares no process with other tests' sessions
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_gpu_fused_norm_bits as t; t.paired_and_chained_add_kernels()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    got = json.loads(out.stdout.strip().splitlines()[-1])
    paired, chained = got["paired"], got["chained"]
    assert len(chained) - len(paired) == 15, (len(chained), len(paired))
    assert len(paired) == 1 and "BFloat16" in paired[0], paired
