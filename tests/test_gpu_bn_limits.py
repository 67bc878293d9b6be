"""The largest sites the batch-norm C-ABI admits (M * C <= 2^31 - 1), against torch's functional chain, bit for bit.

The kernels index rows with `int`: the statistics' and backward reduce's walks (`m * stride + c`, and the backward
reduce's `address_base += address_increment`, which steps past the last row), the elementwise kernels' `m * stride +
c0` and the mask's byte index.  The sites, at (M, C) = (33554431, 64), 2^31 - 64 elements and the longest walk (4096
iterations of a 128-row grid), and at (16383, 131072), the most channels:
- local ReLU sites through b200c_bn_forward_mask / b200c_bn_backward_mask, with g written, at both shapes;
- SiLU sites through b200c_bn_forward_act / b200c_bn_backward_act (k_act_bwd_reduce's own walk), at both shapes;
- stochastic depth then `+ identity` through b200c_bn_forward_res / b200c_bn_backward_res (k_res_bwd_reduce's own
  walk, and the noise read at row / rows_per_sample): 18631 samples of 1801 rows at the first shape, one row per
  sample at the second;
- eval sites at the first shape: b200c_bn_infer with an identity (fp32 parameters), and b200c_bn_infer_act (Hardswish)
  and b200c_bn_infer_res with an identity (bf16 parameters).
Every output is filled with all-ones bits (a NaN) before its call, so an element no thread writes shows.

Each tensor is 4 GiB.  Comparisons stay on the device (torch.equal of int16 views, the mask byte by byte in slices),
and the work runs in phases that free what they no longer need.  Each test prints its peak allocation.  On an NVIDIA
H100 80GB HBM3 (700 W power limit) they peaked at 30.3 and 30.5 GiB for the ReLU sites, 30.0 and 30.2 GiB for the
SiLU sites, 30.1 and 30.2 GiB for the stochastic-depth sites, and 18.0 GiB for each eval test.  The tests skip, saying
so, where the GPU has less than NEED free."""
import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from test_gpu_bn_act_res_abi import row_noise
from test_gpu_fused_norm import GUARD, check_scratch, check_stats_against_float64, make_bn

pytestmark = pytest.mark.gpu

GiB = 1 << 30
NEED = 34 * GiB
SITES = [(33554431, 64), (16383, 131072)]
CHUNK = 1 << 27   # elements per slice when filling and when checking the mask


def seeded(m, c, seed, scale, shift):
    """bf16 Gaussian values written slice by slice, so no fp32 copy of the whole tensor exists."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.empty(m, c, dtype=torch.bfloat16, device="cuda")
    rows = max(1, CHUNK // c)
    for i in range(0, m, rows):
        j = min(m, i + rows)
        t[i:j] = torch.randn(j - i, c, device="cuda", generator=g) * scale + shift
    return t


def nan_filled(*shape, dtype=torch.bfloat16):
    t = torch.empty(*shape, dtype=dtype, device="cuda")
    t.view(torch.int16 if dtype == torch.bfloat16 else torch.int32 if dtype == torch.float32 else torch.uint8).fill_(
        -1 if dtype != torch.uint8 else 255)
    return t


def same(a, b, what):
    assert a.dtype == b.dtype and a.shape == b.shape, what
    w = {2: torch.int16, 4: torch.int32, 8: torch.int64, 1: torch.uint8}[a.element_size()]
    assert torch.equal(a.reshape(-1).view(w), b.reshape(-1).view(w)), f"{what} differs from torch"


def check_mask(mask, y):
    """Bit a % 8 of byte a / 8 is !(y[a] <= 0), for every element a of y."""
    flat = y.view(-1)
    weights = (1 << torch.arange(8, device="cuda", dtype=torch.int32)).view(1, 8)
    for i in range(0, flat.numel(), CHUNK):
        bits = ~(flat[i:i + CHUNK].float() <= 0)
        want = (bits.view(-1, 8).to(torch.int32) * weights).sum(1).to(torch.uint8)
        assert torch.equal(mask[i // 8:(i + CHUNK) // 8], want), f"mask bytes {i // 8}.. differ"


def scratch(c):
    need = int(N.load().b200c_bn_scratch_bytes(c))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    return buf, need


@pytest.fixture
def room():
    free = torch.cuda.mem_get_info()[0]
    if free < NEED:
        pytest.skip(f"needs {NEED / GiB:.0f} GiB of free GPU memory, {free / GiB:.1f} GiB free")
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    print(f"peak memory {torch.cuda.max_memory_allocated() / GiB:.2f} GiB")


@pytest.mark.parametrize("m,c", SITES)
def test_largest_relu_site_matches_torch(room, m, c):
    assert m * c <= 2 ** 31 - 1 and m * c > 2 ** 31 - 2 ** 18
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 3)
    w, b = bn.weight.detach(), bn.bias.detach()
    x = seeded(m, c, 1, 2.0, 0.5)
    buf, need = scratch(c)

    # forward: the native site, then torch's, compared and freed
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    mean, invstd = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    y, mask = nan_filled(m, c), nan_filled(m * c // 8, dtype=torch.uint8)
    N.check(lib.b200c_bn_forward_mask(x.data_ptr(), None, y.data_ptr(), mask.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(),
                                      rv.data_ptr(), nbt.data_ptr(), mean.data_ptr(), invstd.data_ptr(), m, c, 0.1, 1e-5,
                                      buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    assert int(nbt) == int(bn.num_batches_tracked) + 1
    check_stats_against_float64(x, {"mean": mean, "invstd": invstd})
    rm_t, rv_t = bn.running_mean.clone(), bn.running_var.clone()
    x4 = x.view(m, c, 1, 1)   # NCHW strides with stride(1) == 1: torch's channels-last kernels
    y_t, mean_t, invstd_t = torch.native_batch_norm(x4, w, b, rm_t, rv_t, True, 0.1, 1e-5)
    torch.relu_(y_t)
    for got, want, what in ((mean, mean_t, "save_mean"), (invstd, invstd_t, "save_invstd"), (rm, rm_t, "running_mean"),
                            (rv, rv_t, "running_var"), (y, y_t.view(m, c), "y")):
        same(got, want, what)
    check_mask(mask, y)
    del y_t

    # backward: torch's g first (it needs y, which is then freed), the native call, torch's dx
    dy = seeded(m, c, 2, 1.0, 0.0)
    g_t = torch.ops.aten.threshold_backward(dy.view(m, c, 1, 1), y.view(m, c, 1, 1), 0)
    del y
    g, dx = nan_filled(m, c), nan_filled(m, c)
    dw, db = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    N.check(lib.b200c_bn_backward_mask(dy.data_ptr(), None, mask.data_ptr(), x.data_ptr(), g.data_ptr(), dx.data_ptr(), w.data_ptr(),
                                       mean.data_ptr(), invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    same(g, g_t.view(m, c), "g")
    del g, dy
    dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(g_t, x4, w, rm_t, rv_t, mean_t, invstd_t, True, 1e-5,
                                                                 [True, True, True])
    same(dx, dx_t.view(m, c), "dx")
    same(dw, dw_t, "dweight")
    same(db, db_t, "dbias")


def test_largest_eval_site_with_identity_matches_torch(room):
    m, c = SITES[0]
    lib = N.load()
    bn = make_bn(c, 4)
    w, b, rm, rv = bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var
    x, identity = seeded(m, c, 5, 2.0, 0.5), seeded(m, c, 6, 1.0, -0.2)
    y = nan_filled(m, c)
    N.check(lib.b200c_bn_infer(x.data_ptr(), identity.data_ptr(), y.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(),
                               rv.data_ptr(), 0, 1e-5, m, c, torch.cuda.current_stream().cuda_stream))
    with torch.no_grad():   # eager torch's eval-mode module on NCHW strides with stride(1) == 1
        want = bn.eval()(x.view(m, c, 1, 1))
        want += identity.view(m, c, 1, 1)
        torch.relu_(want)
    same(y, want.view(m, c), "y")


@pytest.mark.parametrize("m,c", SITES)
def test_largest_silu_site_matches_torch(room, m, c):
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 7)
    w, b = bn.weight.detach(), bn.bias.detach()
    x = seeded(m, c, 8, 3.0, 0.5)
    buf, need = scratch(c)

    # forward: the native site, then torch's batch norm and SiLU; t stays for the activation's backward
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    mean, invstd = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    y = nan_filled(m, c)
    N.check(lib.b200c_bn_forward_act(x.data_ptr(), y.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(),
                                     mean.data_ptr(), invstd.data_ptr(), N.ACT_SILU, m, c, 0.1, 1e-5, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    assert int(nbt) == int(bn.num_batches_tracked) + 1
    check_stats_against_float64(x, {"mean": mean, "invstd": invstd})
    rm_t, rv_t = bn.running_mean.clone(), bn.running_var.clone()
    x4 = x.view(m, c, 1, 1)   # NCHW strides with stride(1) == 1: torch's channels-last kernels
    t, mean_t, invstd_t = torch.native_batch_norm(x4, w, b, rm_t, rv_t, True, 0.1, 1e-5)
    for got, want, what in ((mean, mean_t, "save_mean"), (invstd, invstd_t, "save_invstd"), (rm, rm_t, "running_mean"),
                            (rv, rv_t, "running_var"), (y, F.silu(t).view(m, c), "y")):
        same(got, want, what)
    del y

    # backward: torch's g first (it needs t, which is then freed), the native call, torch's dx
    dy = seeded(m, c, 9, 1.0, 0.0)
    g_t = torch.ops.aten.silu_backward(dy.view(m, c, 1, 1), t)
    del t
    g, dx = nan_filled(m, c), nan_filled(m, c)
    dw, db = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    N.check(lib.b200c_bn_backward_act(dy.data_ptr(), x.data_ptr(), g.data_ptr(), dx.data_ptr(), w.data_ptr(), b.data_ptr(), mean.data_ptr(),
                                      invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), N.ACT_SILU, m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    same(g, g_t.view(m, c), "g")
    del g, dy
    dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(g_t, x4, w, rm_t, rv_t, mean_t, invstd_t, True, 1e-5,
                                                                 [True, True, True])
    same(dx, dx_t.view(m, c), "dx")
    same(dw, dw_t, "dweight")
    same(db, db_t, "dbias")


@pytest.mark.parametrize("m,c,rows_per_sample", [(*SITES[0], 1801), (*SITES[1], 1)])
def test_largest_drop_add_site_matches_torch(room, m, c, rows_per_sample):
    assert m % rows_per_sample == 0
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 10)
    w, b = bn.weight.detach(), bn.bias.detach()
    x, identity = seeded(m, c, 11, 2.0, 0.5), seeded(m, c, 12, 1.0, -0.2)
    noise = row_noise(m // rows_per_sample, torch.Generator(device="cuda").manual_seed(13))
    noise_rows = noise.repeat_interleave(rows_per_sample).view(m, 1, 1, 1)   # the noise of each row
    buf, need = scratch(c)

    # forward: the native site, then torch's batch norm, bf16 mul by the noise and bf16 add of the identity, in place
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    mean, invstd = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    y = nan_filled(m, c)
    N.check(lib.b200c_bn_forward_res(x.data_ptr(), identity.data_ptr(), noise.data_ptr(), rows_per_sample, y.data_ptr(), w.data_ptr(),
                                     b.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), mean.data_ptr(), invstd.data_ptr(), m, c,
                                     0.1, 1e-5, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    assert int(nbt) == int(bn.num_batches_tracked) + 1
    check_stats_against_float64(x, {"mean": mean, "invstd": invstd})
    rm_t, rv_t = bn.running_mean.clone(), bn.running_var.clone()
    x4 = x.view(m, c, 1, 1)
    y_t, mean_t, invstd_t = torch.native_batch_norm(x4, w, b, rm_t, rv_t, True, 0.1, 1e-5)
    y_t.mul_(noise_rows).add_(identity.view(m, c, 1, 1))
    for got, want, what in ((mean, mean_t, "save_mean"), (invstd, invstd_t, "save_invstd"), (rm, rm_t, "running_mean"),
                            (rv, rv_t, "running_var"), (y, y_t.view(m, c), "y")):
        same(got, want, what)
    del y, y_t, identity

    # backward: g = bf16(dy * noise) by torch, the native call, torch's dx
    dy = seeded(m, c, 14, 1.0, 0.0)
    g_t = dy.view(m, c, 1, 1) * noise_rows
    g, dx = nan_filled(m, c), nan_filled(m, c)
    dw, db = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    N.check(lib.b200c_bn_backward_res(dy.data_ptr(), noise.data_ptr(), rows_per_sample, x.data_ptr(), g.data_ptr(), dx.data_ptr(),
                                      w.data_ptr(), mean.data_ptr(), invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    same(g, g_t.view(m, c), "g")
    del g, dy
    dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(g_t, x4, w, rm_t, rv_t, mean_t, invstd_t, True, 1e-5,
                                                                 [True, True, True])
    same(dx, dx_t.view(m, c), "dx")
    same(dw, dw_t, "dweight")
    same(db, db_t, "dbias")


def test_largest_eval_act_and_res_sites_match_torch(room):
    m, c = SITES[0]
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 15).eval().to(torch.bfloat16)   # bf16 parameters and running statistics
    params = (bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(), 1, bn.eps)
    x = seeded(m, c, 16, 2.0, 0.5)
    x4 = x.view(m, c, 1, 1)

    y = nan_filled(m, c)
    N.check(lib.b200c_bn_infer_act(x.data_ptr(), y.data_ptr(), *params, N.ACT_HARDSWISH, m, c, s))
    with torch.no_grad():   # eager torch's eval-mode module, then Hardswish
        want = F.hardswish(bn(x4), inplace=True)
    same(y, want.view(m, c), "y of Hardswish")
    del want

    identity = seeded(m, c, 17, 1.0, -0.2)
    y.view(torch.int16).fill_(-1)
    N.check(lib.b200c_bn_infer_res(x.data_ptr(), identity.data_ptr(), y.data_ptr(), *params, m, c, s))
    with torch.no_grad():
        want = bn(x4)
        want += identity.view(m, c, 1, 1)
    same(y, want.view(m, c), "y of the residual add")
