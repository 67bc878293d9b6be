"""The fused ResNet stem, maxpool(relu(bn(x))) with nn.MaxPool2d(3, 2, 1), against eager torch's own modules and
autograd, bit for bit: the pooled output, dx, dweight, dbias, the running statistics and num_batches_tracked.

Eager torch runs the batch norm on its native channels-last kernels, the ReLU in place and max_pool2d on its
channels-last kernels (argmax rows first, the first maximum and the last NaN win; the backward sums each input's
gradient over the windows that selected it in fp32, in (ph, pw) order).  The fused site never writes relu(bn(x));
it makes 4 native launches, as every other fused site.  Shapes: the ResNet stem's and odd ones, one shape per launch
regime of the reducing kernels (gpu_common.BN_REGIME_SHAPES), inputs off the 16-byte grid; through the C-ABI, the
argmax bytes against eager torch's indices, with every operand on and off the grid."""
import copy
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, same_bits
from test_gpu_fused_norm import (CONST, ONE_NAN, ZERO, check_scratch, check_stats_against_float64, edge_bn_setup, edge_site_inputs,
                                 make_bn, misaligned, scratch_with_guard)

pytestmark = pytest.mark.gpu
CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pooled_shape(n, c, h, w):
    return n, c, (h - 1) // 2 + 1, (w - 1) // 2 + 1


def run(bn, x, dpool, fused, pool=None):
    x = x.clone().requires_grad_() if x.data_ptr() % 16 == 0 else x.detach().requires_grad_()
    relu = nn.ReLU(inplace=True)
    pool = pool or nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
    if fused:
        before = N.launch_count()
        y = fused_norm.bn_relu_maxpool(bn, relu, pool, x)
        assert type(y.grad_fn).__name__ == "_FusedBatchNormPoolBackward" or not fused_norm._pool_fusable(pool)
        y.backward(dpool)
        torch.cuda.synchronize()
        launches = N.launch_count() - before
    else:
        y = pool(relu(bn(x)))
        y.backward(dpool)
        launches = None
    return {"y": y.detach(), "dx": x.grad, "dweight": bn.weight.grad, "dbias": bn.bias.grad, "running_mean": bn.running_mean,
            "running_var": bn.running_var, "num_batches_tracked": bn.num_batches_tracked}, launches


def check_stem(x, dpool, bn, launches=4, pool=None):
    want, _ = run(copy.deepcopy(bn), x, dpool, False, pool)
    got, launched = run(copy.deepcopy(bn), x, dpool, True, pool)
    assert launched == launches, f"{launched} native launches, expected {launches}"
    bad = [k for k in want if not same_bits(got[k], want[k])]
    assert not bad, f"differs from eager torch: {bad}"
    return want, got


def gauss_inputs(n, c, h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(n, h, w, c, device="cuda", generator=g) * 2 + 0.3).to(torch.bfloat16).permute(0, 3, 1, 2)
    _, _, oh, ow = pooled_shape(n, c, h, w)
    dpool = torch.randn(n, oh, ow, c, device="cuda", generator=g).to(torch.bfloat16).permute(0, 3, 1, 2)
    return x, dpool


STEM_SHAPES = [(256, 64, 112, 112), (32, 64, 112, 112), (4, 64, 113, 113), (2, 64, 3, 3), (8, 64, 1, 1), (3, 100, 9, 9),
               (2, 8, 2, 2), (1, 64, 1, 7)]


@pytest.mark.parametrize("n,c,h,w", STEM_SHAPES)
def test_stem_is_bit_identical_to_eager_torch(n, c, h, w):
    x, dpool = gauss_inputs(n, c, h, w, n + c + h)
    check_stem(x, dpool, make_bn(c, 3))


@pytest.mark.parametrize("n,c,h,w", list(BN_REGIME_SHAPES))
def test_every_launch_regime_matches_eager_torch(n, c, h, w):
    # the statistics kernel and the pooled-gradient reduce (kGradPool) at every launch regime; where C % 8 == 0 the
    # misaligned copy takes the scalar statistics, pooling and elementwise kernels at the same launch shape
    x, dpool = gauss_inputs(n, c, h, w, n + c + h)
    check_stem(x, dpool, make_bn(c, 3))
    if c % 8 == 0:
        check_stem(misaligned(x), dpool, make_bn(c, 3))


def test_misaligned_input_takes_the_scalar_kernels():
    x, dpool = gauss_inputs(4, 64, 20, 20, 5)
    check_stem(misaligned(x), dpool, make_bn(64, 4))


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters_match_eager_torch(momentum, eps):
    x, dpool = gauss_inputs(8, 100, 28, 28, 6)
    check_stem(x, dpool, make_bn(100, 5, momentum=momentum, eps=eps, nbt=2 ** 40))


@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges_match_eager_torch(grad_edges):
    n, c, h, w = 8, 64, 16, 16
    x, _, _ = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    _, dpool = gauss_inputs(n, c, h, w, 9)
    if grad_edges:
        # -0.0, NaN, Inf and near-max gradients; summed over up to four windows per input
        from gpu_common import edge_values
        pat = edge_values(torch.bfloat16).cuda()
        g = torch.Generator(device="cuda").manual_seed(11)
        d = dpool.permute(0, 2, 3, 1).clone()
        idx = torch.randint(0, pat.numel(), d[..., :32].shape, device="cuda", generator=g)
        d[..., :32] = pat[idx]
        d[..., 32:40] = -0.0
        dpool = d.permute(0, 3, 1, 2)
    setup = edge_bn_setup(grad_edges)
    bn = make_bn(c, 8)
    setup(bn)
    with torch.no_grad():
        bn.bias[CONST] = 0.5     # a constant channel: every window a tie of one positive value
        bn.bias[ZERO] = -0.5     # a zero channel after the ReLU: every window's maximum is 0
    want, got = check_stem(x, dpool, bn)
    if not grad_edges:
        assert torch.isnan(got["y"][:, ONE_NAN]).all()   # the channel's NaN statistics: a NaN in every window
        assert (got["y"][:, ZERO] == 0).all()


def test_four_window_gradients_sum_in_torch_order():
    # input (1, 1) is the maximum of the four windows (0, 0), (0, 1), (1, 0), (1, 1); their gradients 1, 2^-30, -1,
    # 2^-30 summed in that order give 2^-30, in any other pairing 0 or 2^-29
    n, c, h, w = 2, 16, 6, 6
    x, dpool = gauss_inputs(n, c, h, w, 12)
    x = x.permute(0, 2, 3, 1).clone()
    x[:, :, :, :] = -1.0
    x[:, 1, 1, :] = 3.0
    x[:, 4, 4, :] = 2.0
    x[0, 0, 0, 0] = 0.5
    x = x.permute(0, 3, 1, 2)
    d = dpool.permute(0, 2, 3, 1).clone()
    d[:, 0, 0, :], d[:, 0, 1, :], d[:, 1, 0, :], d[:, 1, 1, :] = 1.0, 2.0 ** -30, -1.0, 2.0 ** -30
    dpool = d.permute(0, 3, 1, 2)
    bn = make_bn(c, 13)
    with torch.no_grad():
        bn.weight.abs_()
    want, got = check_stem(x, dpool, bn)
    # the check above compares with eager torch; this pins why the case matters
    relu_out = torch.relu(nn.functional.batch_norm(x.float(), None, None, bn.weight.float(), bn.bias.float(), True))
    assert (relu_out[:, :, 1, 1] > 0).all()


def off_grid(numel, dtype):
    """A flat buffer of `numel` elements whose data pointer is one element past a 16-byte boundary."""
    return torch.empty(numel + 1, dtype=dtype, device="cuda")[1:]


def expected_argmax(x, bn):
    """Eager torch's window position of each pooled element's maximum, (ih - 2 ph + 1) * 3 + (iw - 2 pw + 1), or
    255 where the maximum is 0: one byte per pooled element in NHWC order."""
    n, c, h, w = x.shape
    with torch.no_grad():
        pooled, idx = nn.functional.max_pool2d(torch.relu(bn(x)), 3, 2, 1, return_indices=True)
    _, _, oh, ow = pooled.shape
    ph = torch.arange(oh, device="cuda").view(1, 1, oh, 1)
    pw = torch.arange(ow, device="cuda").view(1, 1, 1, ow)
    pos = (idx // w - 2 * ph + 1) * 3 + (idx % w - 2 * pw + 1)
    pos = torch.where(pooled == 0, 255, pos)
    assert ((pos >= 0) & (pos <= 8) | (pos == 255)).all()
    return pooled, pos.to(torch.uint8).permute(0, 2, 3, 1).flatten()


def test_through_the_c_abi_scratch_stays_in_bounds_and_semaphores_return_to_zero():
    for n, c, h, w in [(32, 64, 112, 112), (3, 100, 9, 9)]:
        check_stem_through_the_c_abi(n, c, h, w, aligned=True)


@pytest.mark.parametrize("aligned", [True, False], ids=["vector", "scalar"])
@pytest.mark.parametrize("n,c,h,w", [(32, 64, 112, 112), (3, 100, 9, 9)] + [s for s in BN_REGIME_SHAPES if s[1] <= 2048])
def test_through_the_c_abi_at_every_launch_regime_on_and_off_the_grid(n, c, h, w, aligned):
    # Off the grid, x, y and argmax each sit one element past a 16-byte boundary (the fused module cannot misalign y
    # and argmax): k_bn_pool_fwd<1> and the scalar kernels at C % 8 == 0 too.
    check_stem_through_the_c_abi(n, c, h, w, aligned)


def check_stem_through_the_c_abi(n, c, h, w, aligned):
    """b200c_bn_forward_pool / b200c_bn_backward_pool on a scratch with guard bytes: the scratch stays in bounds and
    its semaphores return to zero, the statistics are within rounding of float64, the pooled output and the argmax
    bytes are eager torch's, and g is eager torch's max_pool2d and threshold backward."""
    lib = N.load()
    x, dpool = gauss_inputs(n, c, h, w, 14)
    if not aligned:
        x = misaligned(x)
    bn = make_bn(c, 15)
    buf, need = scratch_with_guard(c)
    _, _, oh, ow = pooled_shape(n, c, h, w)
    numel = n * oh * ow * c
    y = torch.empty(numel, dtype=torch.bfloat16, device="cuda") if aligned else off_grid(numel, torch.bfloat16)
    argmax = torch.empty(numel, dtype=torch.uint8, device="cuda") if aligned else off_grid(numel, torch.uint8)
    g, dx = torch.empty_like(x), torch.empty_like(x)
    mean, invstd, dw, db = (torch.empty(c, dtype=torch.float32, device="cuda") for _ in range(4))
    s = torch.cuda.current_stream().cuda_stream
    N.check(lib.b200c_bn_forward_pool(x.data_ptr(), y.data_ptr(), argmax.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(),
                                      bn.running_mean.data_ptr(), bn.running_var.data_ptr(), bn.num_batches_tracked.data_ptr(),
                                      mean.data_ptr(), invstd.data_ptr(), n, h, w, c, 0.1, 1e-5, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    check_stats_against_float64(x.permute(0, 2, 3, 1).reshape(n * h * w, c), {"mean": mean, "invstd": invstd})
    pooled, want_argmax = expected_argmax(x, make_bn(c, 15))
    assert same_bits(y.view(n, oh, ow, c), pooled.permute(0, 2, 3, 1)), "pooled output"
    assert torch.equal(argmax, want_argmax), f"{int((argmax != want_argmax).sum())}/{numel} argmax bytes differ"
    N.check(lib.b200c_bn_backward_pool(dpool.contiguous(memory_format=CL).data_ptr(), argmax.data_ptr(), x.data_ptr(),
                                       g.data_ptr(), dx.data_ptr(), bn.weight.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
                                       dw.data_ptr(), db.data_ptr(), n, h, w, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    # g is the batch norm's output gradient: what eager torch's max_pool2d and threshold backward give
    xr = x.detach().clone().requires_grad_()
    ref_bn = make_bn(c, 15)
    t = ref_bn(xr)
    t.retain_grad()
    nn.MaxPool2d(3, 2, 1)(torch.relu(t)).backward(dpool)
    assert same_bits(g, t.grad)


def stem_trace_kernels():
    """Prints the CUDA kernel names of one fused resnet50 forward and of its backward (small batch), as JSON."""
    import torchvision
    torch.manual_seed(0)
    model = fused_norm.fuse_resnet(torchvision.models.resnet50(num_classes=10).cuda().to(memory_format=CL)).train()
    x = torch.randn(2, 3, 64, 64, device="cuda").contiguous(memory_format=CL)

    def traced(fn):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        return out, [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    def forward():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return model(x).float().sum()

    forward().backward()   # warm-up
    model.zero_grad(set_to_none=True)   # no accumulation into .grad in the traced backward
    loss, fwd = traced(forward)
    _, bwd = traced(loss.backward)
    print(json.dumps({"forward": fwd, "backward": bwd}))


def test_resnet50_trace_runs_every_batch_norm_and_the_max_pool_natively():
    pytest.importorskip("torchvision")
    # in a process of its own, as test_gpu_fused_norm_bits does: a whole-model profiler session shares no process
    # with other tests' sessions
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_gpu_fused_stem as t; t.stem_trace_kernels()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    got = json.loads(out.stdout.strip().splitlines()[-1])
    names = got["forward"] + got["backward"]
    assert got["forward"] and got["backward"], "the profiler saw no CUDA kernel"
    assert not [k for k in names if "max_pool" in k], "a torch max_pool kernel ran"
    assert not [k for k in names if "batch_norm" in k], "a torch batch-norm kernel ran"
    assert any("k_bn_pool_fwd" in k for k in names), names
    assert any(re.search(r"k_bn_bwd_reduce<\(b200c::bn::GradSrc\)4, false>", k) for k in names)
    assert any("k_bn_stats_dual" in k for k in names) and any("Tail)3>" in k for k in names)
    assert any(re.search(r"k_bn_bwd_elemt<\d, \(b200c::bn::GradSrc\)2, false, true>", k) for k in names)
    # the maxpool output's two gradients: the one add autograd still makes in the backward
    adds = [k for k in got["backward"] if "CUDAFunctor_add" in k]
    assert len(adds) == 1 and "BFloat16" in adds[0], adds


# ---- whole models: the fused stem and its fallbacks -------------------------------------------------------
@pytest.mark.parametrize("case", ["ceil_mode", "hooked_pool", "padding_0", "hooked_relu", "global_hook"])
def test_other_maxpools_fall_back_with_the_same_bits(case):
    pytest.importorskip("torchvision")
    import test_gpu_fused_resnet as R
    from ant_ray_b200 import train

    base = R.make_model("resnet18").cuda().to(memory_format=CL)
    seen = []
    hook = lambda mod, args, out: seen.append(mod)  # noqa: E731
    if case == "ceil_mode":
        base.maxpool = nn.MaxPool2d(3, 2, 1, ceil_mode=True)
    elif case == "padding_0":
        base.maxpool = nn.MaxPool2d(3, 2, 0)
    elif case == "hooked_pool":
        base.maxpool.register_forward_hook(lambda mod, args, out: None)
    elif case == "hooked_relu":
        base.relu.register_forward_hook(hook)   # the stem's ReLU (each BasicBlock has its own); the copies share it
    data = R.batches()
    ref = copy.deepcopy(base)
    fused = train.prepare_model(copy.deepcopy(base), parallel_strategy=None)
    # the stem runs as bn_relu, the same 4 launches per site, or with a hook on its ReLU on torch; with a global hook
    # every site runs on torch
    sites = {"hooked_relu": R.SITES["resnet18"] - 1, "global_hook": 0}.get(case, R.SITES["resnet18"])
    handle = torch.nn.modules.module.register_module_forward_hook(hook) if case == "global_hook" else None
    try:
        if case in ("hooked_relu", "global_hook"):
            # the ResNet max-pool, but the stem site also replaces the ReLU's call, whose hooks would be skipped
            assert fused_norm._pool_fusable(fused.maxpool) and fused_norm._skips_hooks(fused.relu)
        else:
            assert not fused_norm._pool_fusable(fused.maxpool)
        want = R.train_steps(ref, data)
        calls_ref, seen[:] = len(seen), []
        got = R.train_steps(fused, data, per_step_launches=4 * sites)
    finally:
        if handle is not None:
            handle.remove()
    R.assert_same_training(got, want, fused, ref)
    if case in ("hooked_relu", "global_hook"):
        assert calls_ref > 0 and len(seen) == calls_ref, (len(seen), calls_ref)


def test_fused_stem_trains_bit_identically_at_odd_input_sizes():
    torchvision = pytest.importorskip("torchvision")
    import test_gpu_fused_resnet as R
    from ant_ray_b200 import train

    base = R.make_model("resnet50").cuda().to(memory_format=CL)
    g = torch.Generator(device="cuda").manual_seed(21)
    data = [(torch.randn(4, 3, 99, 99, device="cuda", generator=g).contiguous(memory_format=CL),
             torch.randint(0, 10, (4,), device="cuda", generator=g)) for _ in range(3)]
    ref = copy.deepcopy(base)
    want = R.train_steps(ref, data)
    fused = train.prepare_model(copy.deepcopy(base), parallel_strategy=None)
    assert fused_norm._pool_fusable(fused.maxpool)
    got = R.train_steps(fused, data, per_step_launches=4 * R.SITES["resnet50"])
    R.assert_same_training(got, want, fused, ref)
