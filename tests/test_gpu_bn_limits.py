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
  and b200c_bn_infer_res with an identity (bf16 parameters);
- concatenation sites (b200c_bn_forward_cat / b200c_bn_backward_cat / b200c_bn_infer_cat) at both shapes: segments of
  (8, 16, 40) channels at the first, 64 segments of 2048 at the second;
- slice sites (b200c_bn_forward_slice / b200c_bn_backward_slice / b200c_bn_infer_slice): the whole [33554431][64]
  output (ldy = lddy = 64, m * ldy = 2^31 - 64), and at (16383, 131072) the slice at c0 = 8 of rows of ldy = lddy =
  131080 channels, which ends at the row's last channel (m * ldy = 2^31 - 8), with a pattern in the channels before it.
The shuffle sites (b200c_bn_forward_shuffle / b200c_bn_backward_shuffle) admit n * 2B * hw up to 2^31 - 1 and index
y, dy and x1 with size_t, the masks by rows of ceil(B / 8) bytes.  Both forms run at (n, B, h, w) = (8192, 65535, 1,
2): the most channels with B odd (2048 channel tiles, the last partial; 8192-byte mask rows with one padding bit; the
dual scratch at its largest); and at (377812, 58, 7, 7): 18512788 rows, whose 32-row tiles cross sample boundaries up
to the top of the index range.  The one-batch-norm form runs at B = 1, h * w = 49 and n = (2^31 - 1) // 98: the
longest backward-reduce walk (block (1, 512), 128 rows of blocks, about 16,000 rows per thread) and one mask byte with
7 padding bits per row.  x1 is the first half of each sample of the block input, y's planes are compared with torch's
batch norm and ReLU and with x1, each mask with its bit rule, and the saved statistics with float64 sums taken over
slices of rows.
Every output is filled with all-ones bits (a NaN) before its call, so an element no thread writes shows.

The squeeze-and-excitation calls admit n * c * hw up to 2^31 - 1, where torch splits its own reduction (so no torch
bits exist for the sums).  They run at (n, c, hw) = (2, 128, 8388607), (85, 3, 8388607) and (1, 2, 2^30 - 1), where
se_reduce_config gives a 132-SM H100 8192, 2048 and 16384 blocks per output (vec 4, 1 and 2), and at (16383, 131072,
1), one row per sample.  Their inputs are integers whose sums are exact in any order (sum |x| and sum |dy x| at most
2^24 per output): pooled must be bf16(fp32(S) * factor) and ds bf16(S) for the float64 row sums S; y and dx are
elementwise and are compared with torch's ops at full size.

Each tensor is 4 GiB.  Comparisons stay on the device (torch.equal of int16 views, the mask byte by byte in slices),
and the work runs in phases that free what they no longer need.  Each test prints its peak allocation.  On an NVIDIA
H100 80GB HBM3 (700 W power limit) they peaked at 30.3 and 30.5 GiB for the ReLU sites, 30.0 and 30.2 GiB for the
SiLU sites, 30.1 and 30.2 GiB for the stochastic-depth sites, 18.0 GiB for each eval test, 30.0 and 30.2 GiB for the
concatenation sites, 26.0 and 26.2 GiB for the slice sites, 17.2 and 24.5 GiB for the 65535-channel shuffle sites
(one and two batch norms), 17.1 and 24.3 GiB for the 58-channel ones, 18.0 GiB for the one-channel one, and 14.0,
14.0, 14.0 and 24.0 GiB for the squeeze-and-excitation sites.  The tests skip, saying
so, where the GPU has less than NEED free."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from gpu_common import BnLaunch, bn_launch_config
from test_fused_se_cpu import se_reduce_config
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


def check_shuffle_mask(mask, y):
    """The shuffle sites' mask of one batch norm whose output rows are y [m][B]: bit c % 8 of byte r * ceil(B / 8) +
    c / 8 is !(y[r, c] <= 0), and the bits of each row's padding channels are 0."""
    m, c = y.shape
    mb = -(-c // 8)
    assert mask.shape == (m * mb,), "mask length"
    weights = (1 << torch.arange(8, device="cuda", dtype=torch.int32)).view(1, 1, 8)
    rows = max(1, CHUNK // (8 * mb))
    for i in range(0, m, rows):
        j = min(m, i + rows)
        bits = torch.zeros(j - i, 8 * mb, dtype=torch.int32, device="cuda")
        bits[:, :c] = ~(y[i:j].float() <= 0)
        want = (bits.view(j - i, mb, 8) * weights).sum(2).to(torch.uint8)
        assert torch.equal(mask.view(m, mb)[i:j], want), f"mask rows {i}.. differ"


def scratch(c, dual=False):
    need = int(N.load().b200c_bn_dual_scratch_bytes(c) if dual else N.load().b200c_bn_scratch_bytes(c))
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


# ---- concatenation sites ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m,chans", [(SITES[0][0], (8, 16, 40)), (SITES[1][0], (2048,) * 64)], ids=["3_segments", "64_segments"])
def test_largest_cat_site_matches_torch(room, m, chans):
    c = sum(chans)
    assert (m, c) in SITES
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 20)
    w, b = bn.weight.detach(), bn.bias.detach()
    segs = [seeded(m, k, 21 + i, 2.0, 0.5) for i, k in enumerate(chans)]
    table = ((ctypes.c_void_p * len(segs))(*(t.data_ptr() for t in segs)), (ctypes.c_int * len(chans))(*chans), len(chans))
    buf, need = scratch(c)

    # forward: the native site, then torch's batch norm and ReLU on the concatenation, compared and freed
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    mean, invstd = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    y, mask = nan_filled(m, c), nan_filled(m * c // 8, dtype=torch.uint8)
    N.check(lib.b200c_bn_forward_cat(*table, y.data_ptr(), mask.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(), rv.data_ptr(),
                                     nbt.data_ptr(), mean.data_ptr(), invstd.data_ptr(), m, c, 0.1, 1e-5, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    assert int(nbt) == int(bn.num_batches_tracked) + 1
    x = torch.cat(segs, 1)
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
    dy = seeded(m, c, 22, 1.0, 0.0)
    g_t = torch.ops.aten.threshold_backward(dy.view(m, c, 1, 1), y.view(m, c, 1, 1), 0)
    del y
    dx = nan_filled(m, c)
    dw, db = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    N.check(lib.b200c_bn_backward_cat(dy.data_ptr(), mask.data_ptr(), *table, dx.data_ptr(), w.data_ptr(), mean.data_ptr(),
                                      invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    del dy, mask
    dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(g_t, x4, w, rm_t, rv_t, mean_t, invstd_t, True, 1e-5,
                                                                 [True, True, True])
    same(dx, dx_t.view(m, c), "dx")   # every segment's gradient is its channels of dx
    same(dw, dw_t, "dweight")
    same(db, db_t, "dbias")
    del dx, dx_t, g_t

    # eval: fp32 parameters, eager torch's eval-mode module and ReLU
    y = nan_filled(m, c)
    N.check(lib.b200c_bn_infer_cat(*table, y.data_ptr(), w.data_ptr(), b.data_ptr(), bn.running_mean.data_ptr(),
                                   bn.running_var.data_ptr(), 0, 1e-5, m, c, s))
    with torch.no_grad():
        want = torch.relu_(bn.eval()(x4))
    same(y, want.view(m, c), "eval y")


# ---- slice sites --------------------------------------------------------------------------------------------------
OUT_PATTERN = 0x3F5A   # a bf16 outside the slice, which no call writes


@pytest.mark.parametrize("m,c,ldy,c0", [(*SITES[0], 64, 0), (*SITES[1], 131080, 8)], ids=["whole_output", "last_slice"])
def test_largest_slice_site_matches_torch(room, m, c, ldy, c0):
    # y is out[:, c0:c0 + c] of an [m][ldy] output and ends at the row's last channel; dy has the same row stride
    assert c0 + c == ldy and 2 ** 31 - 64 <= m * ldy <= 2 ** 31 - 1
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    bn = make_bn(c, 40)
    w, b = bn.weight.detach(), bn.bias.detach()
    x = seeded(m, c, 41, 2.0, 0.5)
    buf, need = scratch(c)

    # forward: the native site into a patterned output, then torch's batch norm and ReLU, compared and freed
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    mean, invstd = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    out, mask = torch.empty(m, ldy, dtype=torch.bfloat16, device="cuda"), nan_filled(m * c // 8, dtype=torch.uint8)
    out.view(torch.int16).fill_(OUT_PATTERN)
    N.check(lib.b200c_bn_forward_slice(x.data_ptr(), out.data_ptr() + 2 * c0, ldy, mask.data_ptr(), w.data_ptr(), b.data_ptr(),
                                       rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), mean.data_ptr(), invstd.data_ptr(), m, c, 0.1, 1e-5,
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
                            (rv, rv_t, "running_var"), (out[:, c0:], y_t.view(m, c), "y")):
        same(got, want, what)
    assert bool((out[:, :c0].view(torch.int16) == OUT_PATTERN).all()), "a write outside the slice"
    check_mask(mask, y_t.view(m, c))
    del out

    # backward: the native call from dy's slice, then torch's g (which needs y, then freed) and dx
    dy = seeded(m, ldy, 42, 1.0, 0.0)
    dx = nan_filled(m, c)
    dw, db = nan_filled(c, dtype=torch.float32), nan_filled(c, dtype=torch.float32)
    N.check(lib.b200c_bn_backward_slice(dy.data_ptr() + 2 * c0, ldy, mask.data_ptr(), x.data_ptr(), dx.data_ptr(), w.data_ptr(),
                                        mean.data_ptr(), invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    g_t = torch.ops.aten.threshold_backward(dy[:, c0:], y_t.view(m, c), 0).reshape(m, c, 1, 1)
    del dy, y_t, mask
    dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(g_t, x4, w, rm_t, rv_t, mean_t, invstd_t, True, 1e-5,
                                                                 [True, True, True])
    same(dx, dx_t.view(m, c), "dx")
    same(dw, dw_t, "dweight")
    same(db, db_t, "dbias")
    del dx, dx_t, g_t

    # eval: fp32 parameters into a fresh pattern, eager torch's eval-mode module and ReLU
    out = torch.empty(m, ldy, dtype=torch.bfloat16, device="cuda")
    out.view(torch.int16).fill_(OUT_PATTERN)
    N.check(lib.b200c_bn_infer_slice(x.data_ptr(), out.data_ptr() + 2 * c0, ldy, w.data_ptr(), b.data_ptr(), bn.running_mean.data_ptr(),
                                     bn.running_var.data_ptr(), 0, 1e-5, m, c, s))
    with torch.no_grad():
        want = torch.relu_(bn.eval()(x4))
    same(out[:, c0:], want.view(m, c), "eval y")
    assert bool((out[:, :c0].view(torch.int16) == OUT_PATTERN).all()), "an eval write outside the slice"


# ---- shuffle sites ------------------------------------------------------------------------------------------------
# (n, B, h, w, two batch norms): the most channels with B odd (2048 channel tiles, the last partial, 8192-byte mask rows
# with one padding bit, the dual scratch at its largest); 18512788 rows of 58 channels, whose 32-row tiles cross
# sample boundaries up to the top of the index range; and B = 1, the longest backward-reduce walk (block (1, 512), 128
# rows of blocks) with one mask byte of 7 padding bits per row.  h * w > 1 everywhere: with h = w = 1 torch's choice of
# kernel would follow its layout guess.
SHUFFLE_SITES = [(8192, 65535, 1, 2, False), (8192, 65535, 1, 2, True), (377812, 58, 7, 7, False), (377812, 58, 7, 7, True),
                 ((2 ** 31 - 1) // 98, 1, 7, 7, False)]


def check_stats_by_rows(x, mean, invstd):
    """check_stats_against_float64's bounds, with the float64 sums taken over slices of rows: one channel of a billion
    rows has no float64 copy beside the site."""
    m, c = x.shape
    cfg = bn_launch_config(m, c)
    k = -(-m // (cfg.block_y * cfg.grid_y)) + 2 * math.log2(m)
    u = 2.0 ** -24
    rows = max(1, CHUNK // c)
    total, amax = torch.zeros(c, dtype=torch.float64, device="cuda"), torch.zeros(c, dtype=torch.float64, device="cuda")
    for i in range(0, m, rows):
        x64 = x[i:i + rows].double()
        total += x64.sum(0)
        amax = torch.maximum(amax, x64.abs().amax(0))
    mean64 = total / m
    dev, sq = torch.zeros_like(total), torch.zeros_like(total)
    for i in range(0, m, rows):
        x64 = x[i:i + rows].double()
        dev += ((x64 - mean64) ** 2).sum(0)
        sq += (x64 ** 2).sum(0)
    var_got = 1 / invstd.double() ** 2 - 1e-5
    assert bool(((mean.double() - mean64).abs() <= 4 * k * u * amax).all()), "save_mean"
    assert bool(((var_got - dev / m).abs() <= 8 * k * u * sq / m).all()), "save_invstd"


@pytest.mark.parametrize("n,c,h,w,two", SHUFFLE_SITES, ids=["65535_one", "65535_two", "58_one", "58_two", "1_one"])
def test_largest_shuffle_site_matches_torch(room, n, c, h, w, two):
    hw = h * w
    m = n * hw
    assert hw > 1 and 2 ** 31 - 2 ** 15 <= n * 2 * c * hw <= 2 ** 31 - 1
    cfg = bn_launch_config(m, c)
    print(f"backward reduce {cfg}")
    if c == 1:
        assert cfg == BnLaunch(1, 512, 1, 128)
    lib = N.load()
    s = torch.cuda.current_stream().cuda_stream
    nb = 2 if two else 1
    bns = [make_bn(c, 50 + i) for i in range(nb)]
    xs = [seeded(m, c, 52 + i, 1.5, -0.2) for i in range(nb)]   # t, then u: channels-last [m][B] rows
    x = None if two else seeded(n, 2 * c * hw, 54, 2.0, 0.5)    # the block input, whose first half is x1
    buf, need = scratch(c, two)

    # forward: the native site, then torch's batch norms and ReLU, compared plane by plane
    mb = int(lib.b200c_bn_shuffle_mask_bytes(m, c))
    assert mb == m * -(-c // 8)
    y = nan_filled(n * 2 * c * hw)
    st, ref = [], []
    for bn in bns:
        st.append({"mask": nan_filled(mb, dtype=torch.uint8), "rm": bn.running_mean.clone(), "rv": bn.running_var.clone(),
                   "nbt": bn.num_batches_tracked.clone(), "mean": nan_filled(c, dtype=torch.float32),
                   "invstd": nan_filled(c, dtype=torch.float32)})

    def fwd(bn, o):
        return (o["mask"].data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(), o["rm"].data_ptr(), o["rv"].data_ptr(), o["nbt"].data_ptr(),
                o["mean"].data_ptr(), o["invstd"].data_ptr(), 0.1, 1e-5)

    lead = (None, 0, xs[1].data_ptr(), *fwd(bns[1], st[1])) if two else (x.data_ptr(), 2 * c * hw, None, *(None,) * 8, 0.0, 0.0)
    N.check(lib.b200c_bn_forward_shuffle(*lead, xs[0].data_ptr(), *fwd(bns[0], st[0]), y.data_ptr(), n, hw, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    planes = y.view(n, c, 2, hw)   # [..., 1, :] relu(bn_t(t)), [..., 0, :] the lead
    for i, (bn, o) in enumerate(zip(bns, st)):
        assert int(o["nbt"]) == int(bn.num_batches_tracked) + 1
        check_stats_by_rows(xs[i], o["mean"], o["invstd"])
        rm_t, rv_t = bn.running_mean.clone(), bn.running_var.clone()
        y_t, mean_t, invstd_t = torch.native_batch_norm(xs[i].view(m, c, 1, 1), bn.weight.detach(), bn.bias.detach(), rm_t, rv_t,
                                                        True, 0.1, 1e-5)
        torch.relu_(y_t)
        for got, want, what in ((o["mean"], mean_t, "save_mean"), (o["invstd"], invstd_t, "save_invstd"), (o["rm"], rm_t, "running_mean"),
                                (o["rv"], rv_t, "running_var"), (planes[:, :, 1 - i], y_t.view(n, hw, c).permute(0, 2, 1), "y")):
            same(got, want, f"{what} of batch norm {i}")
        check_shuffle_mask(o["mask"], y_t.view(m, c))
        ref.append((y_t.view(m, c), rm_t, rv_t, mean_t, invstd_t))
    if not two:
        same(planes[:, :, 0], x.view(n, 2, c, hw)[:, 0], "y's x1 planes")
    del y, planes, x

    # backward: the native call, then per batch norm torch's g (which needs y, then freed) and dx
    dy = seeded(m, 2 * c, 55, 1.0, 0.0)
    for o in st:
        o.update(dx=nan_filled(m, c), dw=nan_filled(c, dtype=torch.float32), db=nan_filled(c, dtype=torch.float32))

    def bwd(x_, bn, o):
        return (x_.data_ptr(), o["mask"].data_ptr(), o["dx"].data_ptr(), bn.weight.data_ptr(), o["mean"].data_ptr(), o["invstd"].data_ptr(),
                o["dw"].data_ptr(), o["db"].data_ptr())

    u_part = bwd(xs[1], bns[1], st[1]) if two else (None,) * 8
    N.check(lib.b200c_bn_backward_shuffle(dy.data_ptr(), *u_part, *bwd(xs[0], bns[0], st[0]), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    gs = [torch.ops.aten.threshold_backward(dy.view(m, c, 2)[:, :, 1 - i], ref[i][0], 0).reshape(m, c, 1, 1) for i in range(nb)]
    del dy
    for i, (bn, o) in enumerate(zip(bns, st)):
        y_t, rm_t, rv_t, mean_t, invstd_t = ref[i]
        ref[i] = None
        del y_t, o["mask"]
        dx_t, dw_t, db_t = torch.ops.aten.native_batch_norm_backward(gs[i], xs[i].view(m, c, 1, 1), bn.weight.detach(), rm_t, rv_t,
                                                                     mean_t, invstd_t, True, 1e-5, [True, True, True])
        gs[i] = None
        same(o["dx"], dx_t.view(m, c), f"dx of batch norm {i}")
        same(o["dw"], dw_t, f"dweight of batch norm {i}")
        same(o["db"], db_t, f"dbias of batch norm {i}")
        del dx_t


# ---- squeeze-and-excitation sites ---------------------------------------------------------------------------------
SE_SITES = [(2, 128, 8388607), (85, 3, 8388607), (1, 2, 2 ** 30 - 1), (16383, 131072, 1)]
SE_LAUNCH = {(2, 128, 8388607): (4, 8192), (85, 3, 8388607): (1, 2048), (1, 2, 2 ** 30 - 1): (2, 16384),
             (16383, 131072, 1): (4, 1)}   # (vec, blocks per output) at 132 SMs of 2048 threads


def se_ints(n, c, hw, seed, lo, hi, sparse=False):
    """Integer-valued bf16 [n * hw, c] rows in lo .. hi - 1, written slice by slice; with `sparse`, +-1 on the rows
    whose index within the sample is (37 c + 11) mod 128 for channel c and 0 elsewhere, so that no output sums more
    than 2^24 / 2^7 of them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.empty(n * hw, c, dtype=torch.bfloat16, device="cuda")
    rows = max(1, CHUNK // c)
    residue = (torch.arange(c, device="cuda") * 37 + 11) % 128
    for i in range(0, n * hw, rows):
        j = min(n * hw, i + rows)
        if sparse:
            sign = torch.randint(0, 2, (j - i, c), device="cuda", generator=g, dtype=torch.int8) * 2 - 1
            on = (torch.arange(i, j, device="cuda") % hw % 128).view(-1, 1) == residue
            t[i:j] = torch.where(on, sign, 0)
        else:
            t[i:j] = torch.randint(lo, hi, (j - i, c), device="cuda", generator=g, dtype=torch.int8)
    return t


def row_sums(a, n, c, hw, b=None):
    """The float64 sums over each sample's rows of a, or of the bf16 product a * b, and of their magnitudes, in slices:
    two [n, c]."""
    out = torch.zeros(n, c, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(out)
    a3, b3 = a.view(n, hw, c), None if b is None else b.view(n, hw, c)
    per, rows = max(1, CHUNK // (hw * c)), max(1, CHUNK // c)
    for i in range(0, n, per):
        for r in range(0, hw, rows):
            t = a3[i:i + per, r:r + rows]
            if b3 is not None:
                t = t * b3[i:i + per, r:r + rows]
            t = t.double()
            out[i:i + per] += t.sum(1)
            mag[i:i + per] += t.abs_().sum(1)
    return out, mag


@pytest.mark.parametrize("n,c,hw", SE_SITES)
def test_largest_se_site_sums_exactly(room, n, c, hw):
    assert 2 ** 31 - 2 ** 24 < n * c * hw <= 2 ** 31 - 1
    lib = N.load()
    st = torch.cuda.current_stream().cuda_stream
    props = torch.cuda.get_device_properties(torch.cuda.current_device())
    launch = se_reduce_config(n, c, hw, 0, props.multi_processor_count, props.max_threads_per_multi_processor)
    print(f"launch {launch}")
    if (props.multi_processor_count, props.max_threads_per_multi_processor) == (132, 2048):
        assert (launch.vec, launch.ctas) == SE_LAUNCH[(n, c, hw)]
    need = int(lib.b200c_se_scratch_bytes(n, c, hw))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    x = se_ints(n, c, hw, 30, -2, 3, sparse=hw > 2 ** 23)
    x3 = x.view(n, hw, c)

    # pool: bf16(fp32(S) * factor), factor = float(n * c) / float(n * c * hw) in fp32 as the launcher computes it
    pooled = nan_filled(n, c)
    N.check(lib.b200c_se_pool(x.data_ptr(), pooled.data_ptr(), n, c, hw, buf.data_ptr(), need, st))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    factor = (torch.tensor(n * c, dtype=torch.float32) / torch.tensor(n * c * hw, dtype=torch.float32)).item()
    if hw == 1:
        assert factor == 1.0
        want = x.view(n, c)   # one row: S is x itself (and pooled has x's 2^31 - 2^17 elements, too many for float64 sums)
    else:
        sums, abs_sums = row_sums(x, n, c, hw)
        assert float(abs_sums.max()) <= 2 ** 24   # every partial sum, in any order, is an integer fp32 holds
        want = (sums.float() * factor).to(torch.bfloat16)
    same(pooled, want, "pooled")
    del pooled

    # scale: torch's s * x at full size
    s = seeded(n, c, 31, 0.25, 0.5)   # n * c reaches 2^31 - 2^17 at one row per sample: written slice by slice
    y = nan_filled(n * hw, c)
    N.check(lib.b200c_se_scale(x.data_ptr(), s.data_ptr(), y.data_ptr(), n, c, hw, st))
    same(y, (x3 * s.view(n, 1, c)).view(n * hw, c), "y")
    del y

    # backward reduce: bf16(S) of the products, or with one row the product itself
    dy = se_ints(n, c, hw, 32, -1, 2)
    ds = nan_filled(n, c)
    N.check(lib.b200c_se_backward_reduce(dy.data_ptr(), x.data_ptr(), ds.data_ptr(), n, c, hw, buf.data_ptr(), need, st))
    torch.cuda.synchronize()
    check_scratch(buf, need)
    if hw == 1:
        want = (dy * x).view(n, c)
    else:
        sums, abs_sums = row_sums(dy, n, c, hw, x)
        assert float(abs_sums.max()) <= 2 ** 24
        want = sums.float().to(torch.bfloat16)
    same(ds, want, "ds")
    del x, x3, ds, want

    # backward elementwise: torch's dy * s, then + gp / hw
    gp = seeded(n, c, 33, 0.5, 0.0)
    dx = nan_filled(n * hw, c)
    N.check(lib.b200c_se_backward_elemt(dy.data_ptr(), s.data_ptr(), gp.data_ptr(), dx.data_ptr(), n, c, hw, st))
    dx_t = dy.view(n, hw, c) * s.view(n, 1, c)
    dx_t.add_(gp.view(n, 1, c) / hw)
    same(dx, dx_t.view(n * hw, c), "dx")
