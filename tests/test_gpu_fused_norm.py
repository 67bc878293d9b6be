"""The fused batch-norm sites (fused_norm.py, norm_kernels.cuh) against eager torch, bit for bit.

For every distinct batch-norm shape of ResNet-50, at batch 256 and 32, and for an odd shape (batch 3, 100 channels:
a single-row grid, a partial channel tile and the scalar elementwise path): `BatchNorm2d` -> ReLU and
`BatchNorm2d` -> `+= identity` -> ReLU on bf16 channels-last inputs, forward and backward.  The output, the
running statistics, num_batches_tracked and the gradients of the input, the identity, the weight and the bias must
have the same bits as eager torch's.  Sites that must not run fused (eval mode, fp32, NCHW, a hook on the ReLU, a
full backward hook on the batch norm, a global module hook) fall back without a native launch, and call each hook as
often as eager torch does.

Beyond those shapes: one site per launch regime of the reducing kernels (gpu_common.BN_REGIME_SHAPES), operands
whose data pointer is off the 16-byte grid (scalar elementwise kernels), an output gradient in NCHW layout, C = 1
in both layouts (NCHW strides stay on torch), value edges (NaN, +-Inf, constant and zero channels, subnormals, values
near the bf16 maximum, cancellation, the sign of zero, NaN gradients at masked positions), the momentum / eps /
num_batches_tracked range, and the scratch buffer's invariants through direct C-ABI calls."""
import copy
import math

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values, bits_of, bn_launch_config, edge_values, same_bits

pytestmark = pytest.mark.gpu

CL = torch.channels_last
# (C, H, W) of the 53 batch norms of torchvision's resnet50 at 224 x 224
RESNET50_BN_SHAPES = [(64, 112, 112), (64, 56, 56), (256, 56, 56), (128, 56, 56), (128, 28, 28), (512, 28, 28),
                      (256, 28, 28), (256, 14, 14), (1024, 14, 14), (512, 14, 14), (512, 7, 7), (2048, 7, 7)]
CASES = [(n, c, h, w) for c, h, w in RESNET50_BN_SHAPES for n in (256, 32)] + [(3, 100, 9, 9)] + list(BN_REGIME_SHAPES)


def make_bn(c, seed, momentum=0.1, eps=1e-5, nbt=5):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm2d(c, eps=eps, momentum=momentum)
    with torch.no_grad():
        bn.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
        bn.bias.copy_(0.2 * torch.randn(c, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(c, generator=g))
        bn.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
        bn.num_batches_tracked.fill_(nbt)
    return bn.cuda()


def misaligned(t):
    """A channels-last copy of `t` whose data pointer is 2 mod 16, which sends a site to the scalar kernels."""
    n, c, h, w = t.shape
    v = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    assert v.is_contiguous(memory_format=CL) and v.data_ptr() % 16 == 2
    return v


def run(bn, x, identity, dy, fused, misalign=()):
    x = (misaligned(x) if "x" in misalign else x.clone()).requires_grad_()
    if identity is not None:
        identity = (misaligned(identity) if "identity" in misalign else identity.clone()).requires_grad_()
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
    # semaphores of a later wide site share (one buffer per stream); every site must still merge correctly.  Local,
    # dual, stem, activation and residual sites interleave on the stream: the buffer grows at the first dual site,
    # which needs more than the sites before it; a narrow merged activation site follows a wide local site; a wide dual
    # site (plane 1 on semaphores 512 .. 1023) and a wide stochastic-depth site, whose backward reduce keeps its own copy
    # of the grid merge, are followed by narrow local sites; and a dual site's plane 1 counts on semaphores a wider
    # local site used before it.  After every site the semaphores are all back at zero.
    import test_gpu_fused_act as act
    import test_gpu_fused_res as res
    from test_gpu_fused_dual import check_dual, inputs as dual_inputs
    from test_gpu_fused_stem import check_stem, gauss_inputs

    fused_norm._scratch.clear()
    sites = [("local", (256, 16, 56, 56)), ("stem", (8, 16, 56, 56)), ("dual", (32, 512, 28, 28)), ("local", (256, 2048, 7, 7)),
             ("silu", (256, 16, 56, 56)), ("local", (256, 32, 56, 56)), ("dual", (2, 16384, 32, 32)), ("drop", (2, 16384, 32, 32)),
             ("local", (256, 16, 56, 56)), ("local", (3, 100, 9, 9)), ("add", (32, 24, 56, 56)), ("local", (256, 2048, 7, 7)),
             ("dual", (32, 1024, 14, 14)), ("hardswish", (64, 100, 28, 28)), ("stem", (3, 100, 9, 9)), ("local", (256, 32, 56, 56))]
    sizes = []
    for kind, (n, c, h, w) in sites:
        if kind == "local":
            for residual in (False, True):
                check_site(n, c, h, w, residual)
        elif kind == "dual":
            x3, x_ds, dy1, dy2 = dual_inputs(n, c, h, w, c + n)
            check_dual(x3, x_ds, dy1, dy2, "pair", make_bn(c, 1), make_bn(c, 2))
        elif kind == "stem":
            check_stem(*gauss_inputs(n, c, h, w, c + n), make_bn(c, 3))
        elif kind in act.ACTS:
            act.check_gauss_site(kind, n, c, h, w)
        else:
            res.check_gauss_site(kind, n, c, h, w)
        torch.cuda.synchronize()
        assert len(fused_norm._scratch) == 1
        size, _, buf = next(iter(fused_norm._scratch.values()))
        assert (buf[:SEMAPHORE_BYTES] == 0).all(), f"a {kind} site at {(n, c, h, w)} left a semaphore set"
        sizes.append(size)
    assert sizes[2] > sizes[1] == sizes[0], sizes


def test_one_value_per_channel_raises_as_torch_does():
    bn = make_bn(64, 0)
    x = torch.randn(1, 64, 1, 1, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    before = N.launch_count()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        fused_norm.bn_relu(bn, nn.ReLU(), x)
    assert N.launch_count() == before


def check_site(n, c, h, w, residual, inputs=None, bn_setup=None, misalign=(), dy_nchw=False, x_nchw=False, launches=4,
               **bn_args):
    """Run one site eagerly and fused on the same inputs and compare every result bit for bit (NaN matching NaN).
    `inputs` (x, dy, identity) replaces the seeded Gaussian activations, `bn_setup(bn)` edits the batch norm
    before it is copied, `misalign` names the operands moved off the 16-byte grid, `dy_nchw` / `x_nchw` give dy / x
    NCHW strides, and `launches` is the native launch count the site must make.  Returns (eager, fused) results."""
    seed = n * 100003 + c * 101 + h + residual
    g = torch.Generator(device="cuda").manual_seed(seed)

    def act(scale, shift):
        # NHWC strides, stride(1) == 1 included: for C = 1, `.contiguous(memory_format=CL)` keeps NCHW strides
        t = (torch.randn(n, c, h, w, device="cuda", generator=g) * scale + shift).to(torch.bfloat16)
        nhwc = torch.empty(n, h, w, c, dtype=t.dtype, device=t.device).permute(0, 3, 1, 2).copy_(t)
        assert nhwc.stride(1) == 1 and nhwc.is_contiguous(memory_format=CL)
        return nhwc

    if inputs is None:
        x, dy = act(2.0, 0.5), act(1.0, 0.0)
        identity = act(1.0, -0.2) if residual else None
    else:
        x, dy, identity = inputs
        identity = identity if residual else None
    if x_nchw:
        x = torch.empty(x.shape, dtype=x.dtype, device=x.device).copy_(x)   # default strides, even where C == 1
        assert x.stride(1) == h * w
    if dy_nchw:
        dy = torch.empty(dy.shape, dtype=dy.dtype, device=dy.device).copy_(dy)
    elif "dy" in misalign:
        dy = misaligned(dy)
    ref_bn = make_bn(c, seed, **bn_args)
    if bn_setup is not None:
        bn_setup(ref_bn)
    fused_bn = copy.deepcopy(ref_bn)
    assert torch._C._select_batch_norm_backend(x, ref_bn.weight, ref_bn.bias, ref_bn.running_mean, ref_bn.running_var, True,
                                               ref_bn.eps) == torch._C._BatchNormBackend.Native
    want = run(ref_bn, x, identity, dy, fused=False, misalign=misalign)
    before = N.launch_count()
    got = run(fused_bn, x, identity, dy, fused=True, misalign=misalign)
    torch.cuda.synchronize()
    launched = N.launch_count() - before
    bad = []
    for k in want:
        if want[k] is None or got[k] is None:
            ok = want[k] is None and got[k] is None
        else:
            try:
                assert_same_values(got[k], want[k], k)
                ok = True
            except AssertionError as e:
                ok = False
                print(e)
        if not ok:
            bad.append(k)
    assert not bad, f"differs from eager torch: {bad}"
    assert launched == launches, f"{launched} native launches, expected {launches}"
    if launches:
        assert got["y"].is_contiguous(memory_format=CL) and got["dx"].is_contiguous(memory_format=CL)
    return want, got


@pytest.mark.parametrize("operand", ["x", "identity", "dy"])
def test_misaligned_operand_takes_the_scalar_kernels(operand):
    # C % 8 == 0, but one operand sits one element past a 16-byte boundary: the elementwise kernels run scalar
    for n, c, h, w in [(8, 64, 16, 16), (4, 256, 7, 7)]:
        check_site(n, c, h, w, True, misalign=(operand,))
        if operand != "identity":
            check_site(n, c, h, w, False, misalign=(operand,))


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("n,c,h,w", [(8, 64, 16, 16), (3, 100, 9, 9), (64, 1, 32, 32)])
def test_nchw_output_gradient(n, c, h, w, residual):
    # Eager torch picks its backward-reduce kernel from the layout of the gradient that reaches the batch norm: the
    # ReLU's threshold_backward output, which is channels-last here because the ReLU's output is.  The fused
    # backward converts dy to channels-last and must give the same bits.
    check_site(n, c, h, w, residual, dy_nchw=True)


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_one_channel_in_both_layouts(layout, residual):
    # With C = 1 NCHW strides pass the channels-last contiguity check, but torch runs its NCHW statistics kernel
    # on them (stride(1) != 1), so such a site stays on torch.  NHWC strides (stride(1) == 1) run fused.
    check_site(64, 1, 32, 32, residual, x_nchw=layout == "nchw", launches=0 if layout == "nchw" else 4)


# channels of the value-edge site (8, 64, 16, 16): M = 2048 rows, a merged grid of 2 x 8 blocks
CONST, ZERO, ONE_NAN, POS_INF, NEG_INF, NEAR_MAX, POS_NEAR_MAX, SUBNORMAL, CANCEL, DC, NEG_ZERO, UNDERFLOW = range(12)
NONFINITE = {ONE_NAN, POS_INF, NEG_INF, NEAR_MAX, POS_NEAR_MAX}
BF16_MAX, BF16_SUB = torch.finfo(torch.bfloat16).max, 2.0 ** -133


def edge_site_inputs(n, c, h, w, seed, grad_edges):
    g = torch.Generator(device="cuda").manual_seed(seed)
    m = n * h * w

    def gauss(scale=1.0, shift=0.0):
        return torch.randn(m, c, device="cuda", generator=g) * scale + shift

    def drawn(cols):   # edge values of bf16 mixed half and half with Gaussian values
        pat = edge_values(torch.bfloat16).float().cuda()
        e = pat[torch.randint(0, pat.numel(), (m, cols), device="cuda", generator=g)]
        return torch.where(torch.rand(m, cols, device="cuda", generator=g) < 0.5, e, torch.randn(m, cols, device="cuda", generator=g))

    x, dy, identity = gauss(2.0, 0.5), gauss(), gauss(1.0, -0.2)
    if grad_edges:
        identity[:, 0:16], dy[:, 16:32] = drawn(16), drawn(16)
        identity[:, 32:48], dy[:, 32:48] = drawn(16), drawn(16)
        dy[:10, c - 2:] = float("nan")   # bn_setup: channel c - 2 has y == 0 in nearly every row, channel c - 1 y > 0
    else:
        sign = torch.where(torch.rand(m, device="cuda", generator=g) < 0.5, -1.0, 1.0)
        x[:, CONST] = 0.75
        x[:, ZERO] = 0.0
        x[777, ONE_NAN] = float("nan")
        x[5, POS_INF] = float("inf")
        x[1500, NEG_INF] = float("-inf")
        x[:, NEAR_MAX] = sign * BF16_MAX * (0.9 + 0.1 * torch.rand(m, device="cuda", generator=g))
        x[:, POS_NEAR_MAX] = BF16_MAX * (0.5 + 0.5 * torch.rand(m, device="cuda", generator=g))
        x[:, SUBNORMAL] = torch.randint(-127, 128, (m,), device="cuda", generator=g).float() * BF16_SUB
        x[:, CANCEL] = 1000 + 4 * torch.randn(m, device="cuda", generator=g)
        x[:, DC] = 65536 + 256 * torch.randn(m, device="cuda", generator=g)
        x[:, NEG_ZERO] = 0.75                            # t = -w * 0 + (-0.0) = -0.0 exactly (bn_setup)
        identity[:, NEG_ZERO] = torch.where(sign < 0, -0.0, 0.0)
    cl = lambda t: t.to(torch.bfloat16).view(n, h, w, c).permute(0, 3, 1, 2)
    return cl(x), cl(dy), cl(identity)


def edge_bn_setup(grad_edges):
    def setup(bn):
        with torch.no_grad():
            if grad_edges:
                bn.bias[-2], bn.bias[-1] = -10.0, 10.0
            else:
                bn.weight[NEG_ZERO], bn.bias[NEG_ZERO] = -1.5, -0.0
                bn.weight[UNDERFLOW], bn.bias[UNDERFLOW] = 2.0 ** -140, -0.0   # bf16(t) is +-0 or a subnormal
    return setup


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges_match_eager_torch(grad_edges, residual):
    n, c, h, w = 8, 64, 16, 16
    inputs = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    want, got = check_site(n, c, h, w, residual, inputs=inputs, bn_setup=edge_bn_setup(grad_edges))
    if not grad_edges:
        # a channel's NaN or Inf stays in that channel, through the grid merge included
        finite = [k for k in range(c) if k not in NONFINITE]
        for k in ("y", "dx", "d_identity"):
            if got[k] is not None:
                assert torch.isfinite(got[k][:, finite].float()).all(), k
        for k in ("running_mean", "running_var", "dweight", "dbias"):
            assert torch.isfinite(got[k][finite]).all(), k
        assert torch.isnan(got["y"][:, ONE_NAN]).all()
        # where the batch norm's output is exactly -0.0, eager torch's ReLU on the GPU writes +0.0 (its clamp_min
        # is a max(v, 0) that returns +0.0), as does the fused transform (compared above)
        assert (bits_of(want["y"][:, NEG_ZERO]) == 0).all()


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters_match_eager_torch(momentum, eps, residual):
    # num_batches_tracked starts past 2^32, so a 32-bit increment would show
    check_site(8, 100, 28, 28, residual, momentum=momentum, eps=eps, nbt=2 ** 40)


# ---- the scratch buffer, through direct C-ABI calls ---------------------------------------------------
GUARD = 64 << 10
SEMAPHORE_BYTES = 16384


def scratch_with_guard(c):
    need = int(N.load().b200c_bn_scratch_bytes(c))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    return buf, need


def site_inputs(m, c, seed):
    # well-conditioned channels with distinct means and spreads: |mean| <= 5, 0.5 <= std <= 2
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.arange(c, device="cuda")
    mu, sd = (k % 11 - 5).float(), 0.5 + (k % 7).float() / 4
    x = (torch.randn(m, c, device="cuda", generator=g) * sd + mu).to(torch.bfloat16)
    dy = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    bn = make_bn(c, seed)
    return x, dy, bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var


def torch_site(x, dy, w, b, rm, rv, eps=1e-5, momentum=0.1, dy2=None, relu=True):
    """torch's functional chain for one site of m rows: native_batch_norm, relu (unless `relu` is False), then
    threshold_backward of the output gradient, bf16(dy + dy2) where the output has two consumers, and
    native_batch_norm_backward.  "g" is the batch norm's output gradient."""
    m, c = x.shape
    x4, dy4 = x.view(m, c, 1, 1), dy.view(m, c, 1, 1)   # NCHW strides with stride(1) == 1: torch's channels-last kernels
    if dy2 is not None:
        dy4 = dy4 + dy2.view(m, c, 1, 1)
    rm, rv = rm.clone(), rv.clone()
    out, mean, invstd = torch.native_batch_norm(x4, w, b, rm, rv, True, momentum, eps)
    y = torch.relu(out) if relu else out
    grad = torch.ops.aten.threshold_backward(dy4, y, 0) if relu else dy4
    dx, dw, db = torch.ops.aten.native_batch_norm_backward(grad, x4, w, rm, rv, mean, invstd, True, eps, [True, True, True])
    return {"y": y.view(m, c), "mean": mean, "invstd": invstd, "running_mean": rm, "running_var": rv, "dx": dx.view(m, c),
            "dweight": dw, "dbias": db, "g": grad.view(m, c)}


def native_site(x, dy, w, b, rm, rv, scratch, stream, eps=1e-5, momentum=0.1):
    """Allocates on the current stream, then enqueues the forward and backward calls on `stream`."""
    lib = N.load()
    m, c = x.shape
    rm, rv = rm.clone(), rv.clone()
    y, dx = torch.empty_like(x), torch.empty_like(x)
    mean, invstd, dw, db = (torch.empty(c, dtype=torch.float32, device="cuda") for _ in range(4))
    nbt = torch.zeros((), dtype=torch.int64, device="cuda")

    def launch():
        s = stream.cuda_stream
        N.check(lib.b200c_bn_forward(x.data_ptr(), None, y.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                                     nbt.data_ptr(), mean.data_ptr(), invstd.data_ptr(), m, c, momentum, eps, scratch.data_ptr(), s))
        N.check(lib.b200c_bn_backward(dy.data_ptr(), y.data_ptr(), x.data_ptr(), None, dx.data_ptr(), w.data_ptr(), mean.data_ptr(),
                                      invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, scratch.data_ptr(), s))

    return launch, {"y": y, "mean": mean, "invstd": invstd, "running_mean": rm, "running_var": rv, "dx": dx, "dweight": dw,
                    "dbias": db}


def check_scratch(buf, need):
    assert (buf[need:] == 0xA5).all(), "a call wrote past b200c_bn_scratch_bytes(c)"
    assert (buf[:SEMAPHORE_BYTES] == 0).all(), "a call left a semaphore set"


def check_stats_against_float64(x, got):
    # Welford in fp32 along one thread's rows, then merge trees over the block and the grid: a path of at most
    # k = rows per thread + 2 log2(M) roundings.  Bound the error by 4 k u |x|max for the mean and 8 k u E[x^2] for
    # the biased variance (u = 2^-24), far below the spacing of the channels' means and variances.
    m, c = x.shape
    cfg = bn_launch_config(m, c)
    k = -(-m // (cfg.block_y * cfg.grid_y)) + 2 * math.log2(m)
    u = 2.0 ** -24
    step = max(1, (1 << 24) // m)
    for j in range(0, c, step):   # in slices of channels: a float64 copy of a 131072-channel site would take 2 GiB
        x64 = x[:, j:j + step].double()
        mean64, var64 = x64.mean(0), x64.var(0, unbiased=False)
        var_got = 1 / got["invstd"][j:j + step].double() ** 2 - 1e-5
        assert ((got["mean"][j:j + step].double() - mean64).abs() <= 4 * k * u * x64.abs().amax(0)).all()
        assert ((var_got - var64).abs() <= 8 * k * u * (x64 ** 2).mean(0)).all()


def check_native_site(m, c, seed):
    """One ReLU site through b200c_bn_forward / b200c_bn_backward (y read, no mask) on a scratch with guard bytes,
    against torch bit for bit.  Returns (x, native results)."""
    x, dy, w, b, rm, rv = site_inputs(m, c, seed)
    want = torch_site(x, dy, w, b, rm, rv)
    buf, need = scratch_with_guard(c)
    launch, got = native_site(x, dy, w, b, rm, rv, buf, torch.cuda.current_stream())
    launch()
    torch.cuda.synchronize()
    check_scratch(buf, need)
    for k in got:
        assert same_bits(got[k], want[k]), k
    return x, got


@pytest.mark.parametrize("m,c", [(65536, 16), (32768, 100), (32768, 2048), (2048, 131072)])
def test_scratch_stays_in_bounds_and_semaphores_return_to_zero(m, c):
    assert bn_launch_config(m, c).grid_y == (8 if c == 131072 else 128)
    check_stats_against_float64(*check_native_site(m, c, c))


def test_two_streams_with_their_own_scratch():
    sites = [site_inputs(32768, 100, 1), site_inputs(32768, 2048, 2)]
    wants = [torch_site(*s) for s in sites]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    bufs = [scratch_with_guard(s[0].shape[1]) for s in sites]
    runs = [native_site(*s, buf, st) for s, (buf, _), st in zip(sites, bufs, streams)]
    torch.cuda.synchronize()
    for _ in range(3):   # interleaved enqueues, so the two sites' kernels overlap on the device
        for launch, _ in runs:
            launch()
    torch.cuda.synchronize()
    for (_, got), want, (buf, need) in zip(runs, wants, bufs):
        check_scratch(buf, need)
        for k in ("y", "mean", "invstd", "dx", "dweight", "dbias"):
            assert same_bits(got[k], want[k]), k


@pytest.mark.parametrize("case", ["eval", "fp32", "nchw", "relu_hook", "bn_backward_hook", "global_hook"])
def test_ineligible_sites_fall_back_to_torch(case):
    n, c, h, w = 8, 64, 14, 14
    g = torch.Generator(device="cuda").manual_seed(3)
    dtype = torch.float32 if case == "fp32" else torch.bfloat16
    fmt = torch.contiguous_format if case == "nchw" else CL
    x = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
    identity = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
    dy = torch.randn(n, c, h, w, device="cuda", generator=g).to(dtype).contiguous(memory_format=fmt)
    ref_bn = make_bn(c, 1)
    fused_bn = copy.deepcopy(ref_bn)
    if case == "eval":
        ref_bn.eval()
        fused_bn.eval()
    ref_relu, fused_relu = nn.ReLU(), nn.ReLU()
    calls = {"fused": 0, "ref": 0}
    side = "fused"

    def hook(*args):
        calls[side] += 1

    # hooks on each side's own modules (the global one sees both): training sites with a hook run torch's modules,
    # which call it as often as eager torch does
    handles = []
    if case == "relu_hook":
        handles = [r.register_forward_hook(hook) for r in (ref_relu, fused_relu)]
    elif case == "bn_backward_hook":
        handles = [b.register_full_backward_hook(hook) for b in (ref_bn, fused_bn)]
    elif case == "global_hook":
        handles = [torch.nn.modules.module.register_module_forward_hook(hook)]
    hooked = bool(handles)

    def site(bn, relu, t):
        # torch forbids `+= identity` on the output of a module with a full backward hook: that case takes the ReLU site
        return fused_norm.bn_relu(bn, relu, t) if case == "bn_backward_hook" else fused_norm.bn_add_relu(bn, relu, t, identity)

    xf, xr = x.clone().requires_grad_(hooked), x.clone().requires_grad_(hooked)
    try:
        before = N.launch_count()
        got = site(fused_bn, fused_relu, xf)
        if hooked:
            got.backward(dy)
        torch.cuda.synchronize()
        assert N.launch_count() == before, "an ineligible site ran the fused kernels"
        side = "ref"
        out = ref_bn(xr)
        if case != "bn_backward_hook":
            out += identity
        want = ref_relu(out)
        if hooked:
            want.backward(dy)
    finally:
        for handle in handles:
            handle.remove()
    assert same_bits(got, want)
    assert same_bits(fused_bn.running_mean, ref_bn.running_mean) and same_bits(fused_bn.running_var, ref_bn.running_var)
    if hooked:
        assert calls["ref"] > 0 and calls["fused"] == calls["ref"], calls
        for a, b in ((xf.grad, xr.grad), (fused_bn.weight.grad, ref_bn.weight.grad), (fused_bn.bias.grad, ref_bn.bias.grad)):
            assert same_bits(a, b)
