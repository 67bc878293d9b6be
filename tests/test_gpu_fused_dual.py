"""The dual tail, relu(bn3(x3) + bn_ds(x_ds)) of a block whose identity is its downsample branch, against eager torch's
own modules and autograd, bit for bit: y, dx3, dx_ds, both batch norms' dweight, dbias, running statistics and
num_batches_tracked.  One gradient, two gradients (the tail's `pair`) and one of the pair unused; every ResNet-18 and
ResNet-50 downsample shape at batch 256 and 32, C = 100 (y read instead of the mask), one shape per launch regime of the
reducing kernels up to the dual limit of 65536 channels (gpu_common.BN_DUAL_REGIME_SHAPES), misaligned inputs (the
scalar kernels), value edges and the momentum / eps range.  Each site makes 4 native launches, and the downsample
output is never written.  Above the dual limit the downsample's batch norm runs on torch and the tail alone is fused."""
import copy

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_DUAL_REGIME_SHAPES, same_bits
from test_gpu_fused_norm import (check_scratch, check_stats_against_float64, edge_bn_setup, edge_site_inputs, make_bn,
                                 misaligned)

pytestmark = pytest.mark.gpu
CL = torch.channels_last

# (C, H, W) of the downsample sites: resnet50's four, resnet18's three
DOWNSAMPLE_SHAPES = [(256, 56, 56), (512, 28, 28), (1024, 14, 14), (2048, 7, 7), (128, 28, 28), (256, 14, 14), (512, 7, 7)]
KEYS = ("y", "dx", "dx_ds", "dweight", "dbias", "dweight_ds", "dbias_ds", "running_mean", "running_var", "num_batches_tracked",
        "running_mean_ds", "running_var_ds", "num_batches_tracked_ds")


def inputs(n, c, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = lambda s, o: (torch.randn(n, h, w, c, device="cuda", generator=g) * s + o).to(torch.bfloat16).permute(0, 3, 1, 2)  # noqa: E731
    return t(2.0, 0.5), t(1.5, -0.3), t(1.0, 0.0), t(1.0, 0.0)


def run(bn, bn_ds, x3, x_ds, dy1, dy2, mode, fused):
    x3 = (x3.clone() if x3.data_ptr() % 16 == 0 else x3.detach()).requires_grad_()
    x_ds = (x_ds.clone() if x_ds.data_ptr() % 16 == 0 else x_ds.detach()).requires_grad_()
    relu = nn.ReLU(inplace=True)
    before = N.launch_count()
    if fused:
        ys = fused_norm._FusedBatchNormDual.apply(x3, x_ds, bn.weight, bn.bias, bn_ds.weight, bn_ds.bias, bn, bn_ds, mode != "one")
        y = ys[0] if mode != "one" else ys
    else:
        out = bn(x3)
        out += bn_ds(x_ds)
        y = ys = relu(out)
    if mode == "pair":
        torch.autograd.backward([ys[0], ys[1]] if fused else [y, y], [dy1, dy2])
    else:
        y.backward(dy1)
    torch.cuda.synchronize()
    launched = N.launch_count() - before
    return {"y": y.detach(), "dx": x3.grad, "dx_ds": x_ds.grad, "dweight": bn.weight.grad, "dbias": bn.bias.grad,
            "dweight_ds": bn_ds.weight.grad, "dbias_ds": bn_ds.bias.grad, "running_mean": bn.running_mean,
            "running_var": bn.running_var, "num_batches_tracked": bn.num_batches_tracked, "running_mean_ds": bn_ds.running_mean,
            "running_var_ds": bn_ds.running_var, "num_batches_tracked_ds": bn_ds.num_batches_tracked}, launched


def check_dual(x3, x_ds, dy1, dy2, mode, bn, bn_ds):
    want, _ = run(copy.deepcopy(bn), copy.deepcopy(bn_ds), x3, x_ds, dy1, dy2, mode, False)
    got, launched = run(copy.deepcopy(bn), copy.deepcopy(bn_ds), x3, x_ds, dy1, dy2, mode, True)
    assert launched == 4, launched
    bad = [k for k in KEYS if not same_bits(got[k], want[k])]
    assert not bad, f"differs from eager torch: {bad}"
    return want, got


@pytest.mark.parametrize("mode", ["one", "pair", "pair_unused"])
@pytest.mark.parametrize("n", [256, 32])
@pytest.mark.parametrize("c,h,w", DOWNSAMPLE_SHAPES)
def test_downsample_tail_is_bit_identical_to_eager_torch(c, h, w, n, mode):
    x3, x_ds, dy1, dy2 = inputs(n, c, h, w, c + h + n)
    check_dual(x3, x_ds, dy1, dy2, mode, make_bn(c, 1), make_bn(c, 2, momentum=0.2, eps=1e-4, nbt=7))


# one merged, one collapsed and one partial-tile shape with the grid merge
UNUSED_REGIME_SHAPES = [(2, 256, 32, 32), (4, 100, 16, 16), (8, 100, 28, 28)]


@pytest.mark.parametrize("n,c,h,w,mode", [(*s, mode) for s in BN_DUAL_REGIME_SHAPES for mode in ("one", "pair")]
                         + [(*s, "pair_unused") for s in UNUSED_REGIME_SHAPES])
def test_every_launch_regime_matches_eager_torch(n, c, h, w, mode):
    # Both planes of k_bn_stats_dual and the third sum of the DUAL reduce at every regime.  Where C % 8 == 0 the
    # misaligned copy of x_ds takes the scalar statistics, the V = 1 ballot of the transform and the V = 1 dual
    # elementwise kernel (not at the two widest shapes, whose vector runs cover their launch shape).
    x3, x_ds, dy1, dy2 = inputs(n, c, h, w, c + h + n)
    bn, bn_ds = make_bn(c, 1), make_bn(c, 2, momentum=0.2, eps=1e-4, nbt=7)
    check_dual(x3, x_ds, dy1, dy2, mode, bn, bn_ds)
    if c % 8 == 0 and c not in (65536, 4104):
        check_dual(x3, misaligned(x_ds), dy1, dy2, mode, bn, bn_ds)


@pytest.mark.parametrize("mode", ["one", "pair"])
def test_hundred_channels_read_y(mode):
    x3, x_ds, dy1, dy2 = inputs(3, 100, 9, 9, 4)
    check_dual(x3, x_ds, dy1, dy2, mode, make_bn(100, 3), make_bn(100, 4))


@pytest.mark.parametrize("operand", ["x3", "x_ds"])
def test_misaligned_input_takes_the_scalar_kernels(operand):
    x3, x_ds, dy1, dy2 = inputs(8, 64, 16, 16, 5)
    if operand == "x3":
        x3 = misaligned(x3)
    else:
        x_ds = misaligned(x_ds)
    check_dual(x3, x_ds, dy1, dy2, "pair", make_bn(64, 5), make_bn(64, 6))


@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges_match_eager_torch(grad_edges):
    n, c, h, w = 8, 64, 16, 16
    x3, dy, x_ds = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    _, _, _, dy2 = inputs(n, c, h, w, 8)
    if grad_edges:
        dy2 = dy.flip(0).contiguous(memory_format=CL)
    bn, bn_ds = make_bn(c, 8), make_bn(c, 9)
    edge_bn_setup(grad_edges)(bn)
    edge_bn_setup(grad_edges)(bn_ds)
    for mode in ("one", "pair"):
        check_dual(x3.contiguous(memory_format=CL), x_ds.contiguous(memory_format=CL), dy.contiguous(memory_format=CL), dy2,
                   mode, bn, bn_ds)


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters_match_eager_torch(momentum, eps):
    x3, x_ds, dy1, dy2 = inputs(8, 128, 14, 14, 10)
    check_dual(x3, x_ds, dy1, dy2, "pair", make_bn(128, 10, momentum=momentum, eps=eps, nbt=2 ** 40),
               make_bn(128, 11, momentum=1 - momentum, eps=eps * 2, nbt=3))


def check_dual_through_the_c_abi(n, c, h, w):
    """Direct C-ABI calls on a scratch of b200c_bn_dual_scratch_bytes(c) followed by guard bytes: the call leaves the
    whole semaphore region at zero, plane 1's included, writes nothing past the scratch, and both planes' statistics
    are within rounding of float64.  Where C % 8 == 0 the backward runs once on the mask and once on y, with the same
    bits."""
    lib = N.load()
    need = int(lib.b200c_bn_dual_scratch_bytes(c))
    buf = torch.empty(need + (64 << 10), dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    x3, x_ds, dy1, dy2 = inputs(n, c, h, w, 12)
    bn, bn_ds = make_bn(c, 12), make_bn(c, 13)
    m = n * h * w
    y = torch.empty_like(x3)
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device="cuda") if c % 8 == 0 else None
    f = [torch.empty(c, dtype=torch.float32, device="cuda") for _ in range(4)]
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200c_bn_forward_dual(p(x3), p(x_ds), p(y), p(mask), p(bn.weight), p(bn.bias), p(bn.running_mean),
                                      p(bn.running_var), p(bn.num_batches_tracked), p(f[0]), p(f[1]), 0.1, 1e-5,
                                      p(bn_ds.weight), p(bn_ds.bias), p(bn_ds.running_mean), p(bn_ds.running_var),
                                      p(bn_ds.num_batches_tracked), p(f[2]), p(f[3]), 0.1, 1e-5, m, c, p(buf), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    for x, mean, invstd in ((x3, f[0], f[1]), (x_ds, f[2], f[3])):
        check_stats_against_float64(x.permute(0, 2, 3, 1).reshape(m, c), {"mean": mean, "invstd": invstd})
    grads = {}
    for src in ("mask", "y") if mask is not None else ("y",):
        dx, dx_ds = torch.empty_like(x3), torch.empty_like(x3)
        g = [torch.empty(c, dtype=torch.float32, device="cuda") for _ in range(4)]
        N.check(lib.b200c_bn_backward_dual(p(dy1), p(dy2), p(y), p(mask) if src == "mask" else None, p(x3), p(x_ds), p(dx),
                                           p(dx_ds), p(bn.weight), p(f[0]), p(f[1]), p(g[0]), p(g[1]), p(bn_ds.weight), p(f[2]),
                                           p(f[3]), p(g[2]), p(g[3]), m, c, p(buf), s))
        torch.cuda.synchronize()
        check_scratch(buf, need)
        assert same_bits(g[1], g[3])   # Σg is both dbias values
        grads[src] = [dx, dx_ds] + g
    assert all(same_bits(a, b) for a, b in zip(grads["y"], grads.get("mask", grads["y"]))), "mask and y differ"


def test_scratch_stays_in_bounds_and_semaphores_return_to_zero():
    # at 65536 channels plane 1 uses the region's last semaphore
    for n, c, h, w in [(256, 256, 56, 56), (3, 100, 9, 9), (32, 2048, 7, 7), (2, 65536, 32, 32), (64, 3, 32, 32),
                       (8, 4104, 8, 8)]:
        check_dual_through_the_c_abi(n, c, h, w)


def test_above_the_dual_limit_the_downsample_batch_norm_runs_on_torch():
    # 65544 channels: too many for the two planes' semaphores, so the tail is fused alone (4 launches) and its
    # identity is the downsample's batch norm run by torch
    n, c, h, w, c_in = 2, 65544, 2, 2, 8
    assert N.load().b200c_bn_dual_scratch_bytes(c) == 0 < N.load().b200c_bn_scratch_bytes(c)
    g = torch.Generator(device="cuda").manual_seed(14)
    x = (torch.randn(n, h, w, c, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16).permute(0, 3, 1, 2)
    x_id = torch.randn(n, h, w, c_in, device="cuda", generator=g).to(torch.bfloat16).permute(0, 3, 1, 2)
    dy = torch.randn(n, h, w, c, device="cuda", generator=g).to(torch.bfloat16).permute(0, 3, 1, 2)
    torch.manual_seed(14)
    conv = nn.Conv2d(c_in, c, 1, bias=False).cuda().to(torch.bfloat16).to(memory_format=CL)
    base = (make_bn(c, 15), nn.Sequential(conv, make_bn(c, 16, momentum=0.2)))

    def step(fused):
        bn, ds = copy.deepcopy(base)
        xr, x_idr = x.clone().requires_grad_(), x_id.clone().requires_grad_()
        relu = nn.ReLU(inplace=True)
        before = N.launch_count()
        if fused:
            y = fused_norm.bn_add_relu_downsample(bn, relu, xr, ds, x_idr)
        else:
            out = bn(xr)
            out += ds(x_idr)
            y = relu(out)
        y.backward(dy)
        torch.cuda.synchronize()
        tensors = [y, xr.grad, x_idr.grad, ds[0].weight.grad] + [t for b in (bn, ds[1]) for t in
                                                                  (b.weight.grad, b.bias.grad, b.running_mean, b.running_var,
                                                                   b.num_batches_tracked)]
        return tensors, N.launch_count() - before

    with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True):
        want, _ = step(False)
        got, launched = step(True)
    assert launched == 4, launched
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if not same_bits(a, b)]
    assert not bad, f"differs from eager torch: {bad}"


# ---- whole blocks: the dual tail and its fallbacks -----------------------------------------------------------
@pytest.mark.parametrize("case", ["nonstandard_downsample", "hooked_downsample_bn", "hooked_downsample", "hooked_relu"])
def test_other_downsamples_fall_back_with_the_same_bits(case):
    pytest.importorskip("torchvision")
    import test_gpu_fused_resnet as R
    from ant_ray_b200 import train

    base = R.make_model("resnet50").cuda().to(memory_format=CL)
    ds = base.layer2[0].downsample
    seen = []
    if case == "nonstandard_downsample":
        base.layer2[0].downsample = nn.Sequential(ds[0], ds[1], nn.Identity())
    elif case == "hooked_downsample_bn":
        ds[1].register_forward_hook(lambda mod, args, out: None)
    elif case == "hooked_downsample":
        ds.register_forward_pre_hook(lambda mod, args: None)
    else:
        # the block's ReLU module, called after each of its three batch norms; the copies below share the hook
        base.layer2[0].relu.register_forward_hook(lambda mod, args, out: seen.append(mod))
    data = R.batches()
    ref = copy.deepcopy(base)
    want = R.train_steps(ref, data)
    fused = train.prepare_model(copy.deepcopy(base), parallel_strategy=None)
    block, other = fused.layer2[0], fused.layer3[0]
    if case == "hooked_relu":
        # a plain downsample, but the tail also replaces the hooked ReLU's call
        assert fused_norm._downsample_bn(block.downsample) is not None and fused_norm._skips_hooks(block.relu)
    else:
        assert fused_norm._downsample_bn(block.downsample) is None
    assert fused_norm._downsample_bn(other.downsample) is not None
    # the fallback tail is the same 4 launches and the downsample batch norm runs on torch; a hooked ReLU leaves the
    # block's three sites on torch
    sites = R.SITES["resnet50"] - (3 if case == "hooked_relu" else 0)
    got = R.train_steps(fused, data, per_step_launches=4 * sites)
    R.assert_same_training(got, want, fused, ref)
    if case == "hooked_relu":
        calls = [sum(m is relu for m in seen) for relu in (ref.layer2[0].relu, block.relu)]
        assert calls[0] > 0 and calls[1] == calls[0], calls
