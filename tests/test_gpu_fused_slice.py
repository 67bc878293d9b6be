"""The slice batch-norm sites (fused_norm.bn_relu_concat, norm_slice.cuh) against eager torch's
`torch.cat([F.relu(bn(x_b)) for each site] + ready tensors, 1)`, bit for bit (a NaN matches a NaN): y and its strides,
the running statistics, num_batches_tracked, dweight, dbias, and the gradient of every x_b and ready tensor with its
strides.

Shapes: every Inception module of inception_v3 at 299 x 299 and googlenet at 224 x 224, at batch 32 and 256, and the
launch regimes of gpu_common.BN_REGIME_SHAPES as the first, a middle and the last slice.  Value edges and the
momentum / eps range of test_gpu_fused_norm, an NCHW output gradient, retain_graph with two backwards, x without grad,
eval under no_grad and inference_mode with fp32 and bf16 parameters, the fallbacks (the module ops and torch.cat, no
slice call; among them operands for which torch.cat writes a contiguous output), direct C-ABI calls with guard bytes past the scratch and a pattern outside the slice, two streams, and
the largest m * ldy below 2^31.  `trace_cases` is the traced code of test_gpu_zz_trace_slice.py, which checks that
every `b200c::bn_slice` kernel is launched by the case test_fused_slice_cpu.KERNELS gives it."""
import copy
import json

import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values, same_bits
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn

pytestmark = pytest.mark.gpu
CL = torch.channels_last
R = "ready"

# (H = W, branch channels in output order; ("ready", C) a max-pool branch) of every distinct Inception module
INCEPTION_V3 = [(35, (64, 64, 96, 32)), (35, (64, 64, 96, 64)), (17, (384, 96, (R, 288))), (17, (192, 192, 192, 192)),
                (8, (320, 192, (R, 768))), (8, (320, 384, 384, 384, 384, 192))]
GOOGLENET = [(28, (64, 128, 32, 32)), (28, (128, 192, 96, 64)), (14, (192, 208, 48, 64)), (14, (160, 224, 64, 64)),
             (14, (128, 256, 64, 64)), (14, (112, 288, 64, 64)), (14, (256, 320, 128, 128)), (7, (256, 320, 128, 128)),
             (7, (384, 384, 128, 128))]


class Spy:
    """fused_norm's library handle, recording every slice call."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        if name.endswith("_slice"):
            self.calls.append(name)
        return getattr(self.lib, name)


@pytest.fixture
def spy(monkeypatch):
    s = Spy(N.load())
    monkeypatch.setattr(fused_norm, "_lib", s)
    return s


def gauss(n, c, h, w, g, scale=2.0, shift=0.5):
    return (torch.randn(n, c, h, w, device="cuda", generator=g) * scale + shift).to(torch.bfloat16).contiguous(memory_format=CL)


def make_case(n, h, branches, seed=0, momentum=0.1, eps=1e-3, nbt=5):
    """Inputs of a module: per branch ("site", x, bn) or ("ready", t)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for i, b in enumerate(branches):
        if isinstance(b, tuple):
            out.append((R, gauss(n, b[1], h, h, g)))
        else:
            out.append(("site", gauss(n, b, h, h, g), make_bn(b, seed + i, momentum, eps, nbt)))
    return out


def run(case, dys, fused, x_grad=True):
    """One forward (fused: bn_relu_concat; else eager torch) and a backward per dy (retain_graph between them)."""
    grads, branches, leaves, bns = {}, [], [], []
    for i, b in enumerate(case):
        t = (off_grid(b[1]) if b[1].data_ptr() % 16 else b[1].detach().clone()).requires_grad_(x_grad or b[0] == R)
        leaves.append(t)
        t = t.view_as(t) if t.requires_grad else t   # a non-leaf: its hook sees the gradient as autograd hands it over
        if t.requires_grad:
            t.register_hook(lambda g, i=i: grads.setdefault(f"grad{i}", []).append((g.stride(), g.clone())))
        if b[0] == R:
            branches.append(t)
        else:
            bn = copy.deepcopy(b[2])
            bns.append(bn)
            branches.append((bn, t))
    if fused:
        y = fused_norm.bn_relu_concat(branches)
    else:
        y = torch.cat([F.relu(b[0](b[1]), inplace=True) if isinstance(b, tuple) else b for b in branches], 1)
    for k, dy in enumerate(dys):
        y.backward(dy, retain_graph=k + 1 < len(dys))
    out = {"y": y.detach(), "y_stride": y.stride()}
    for i, bn in enumerate(bns):
        out.update({f"running_mean{i}": bn.running_mean, f"running_var{i}": bn.running_var, f"nbt{i}": bn.num_batches_tracked,
                    f"dweight{i}": bn.weight.grad, f"dbias{i}": bn.bias.grad})
    for k, v in grads.items():
        for j, (stride, g) in enumerate(v):
            out[f"{k}_{j}"], out[f"{k}_{j}_stride"] = g, stride
    for i, t in enumerate(leaves):
        out[f"leaf{i}"] = t.grad
    return out


def check(case, dys, spy, fused_calls=True, x_grad=True):
    want = run(case, dys, False, x_grad)
    spy.calls.clear()
    got = run(case, dys, True, x_grad)
    sites = sum(b[0] == "site" for b in case)
    expect = ["b200c_bn_forward_slice"] * sites + ["b200c_bn_backward_slice"] * sites * len(dys) if fused_calls else []
    assert spy.calls == expect, spy.calls
    assert got.keys() == want.keys()
    for k in want:
        if k.endswith("stride"):
            assert got[k] == want[k], k
        elif want[k] is None:
            assert got[k] is None, k
        else:
            assert_same_values(got[k], want[k], k)
    return want, got


def total(branches):
    return sum(b[1] if isinstance(b, tuple) else b for b in branches)


def check_shape(n, h, branches, spy, seed=0, **kw):
    case = make_case(n, h, branches, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    dy = torch.randn(n, total(branches), h, h, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    return check(case, [dy], spy, **kw)


@pytest.mark.parametrize("n", [32, 256])
@pytest.mark.parametrize("model", ["inception_v3", "googlenet"])
def test_every_inception_module(model, n, spy):
    for h, branches in INCEPTION_V3 if model == "inception_v3" else GOOGLENET:
        check_shape(n, h, branches, spy)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("n,c,h,w", list(BN_REGIME_SHAPES))
def test_launch_regimes_as_slices(n, c, h, w, where, spy):
    others = [16, 24]
    branches = {"first": [c] + others, "middle": [16, c, 24], "last": others + [c]}[where]
    g = torch.Generator(device="cuda").manual_seed(2)
    case = [("site", gauss(n, b, h, w, g), make_bn(b, i)) for i, b in enumerate(branches)]
    dy = torch.randn(n, sum(branches), h, w, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    # C % 8 != 0 cannot be a slice: the module runs its ops and torch.cat
    check(case, [dy], spy, fused_calls=c % 8 == 0)


@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges(grad_edges, spy):
    n, c, h, w = 8, 64, 16, 16
    x, dy_edge, _ = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    g = torch.Generator(device="cuda").manual_seed(9)
    bn = make_bn(c, 9)
    edge_bn_setup(grad_edges)(bn)
    case = [("site", gauss(n, 16, h, w, g), make_bn(16, 1)), ("site", x.contiguous(memory_format=CL), bn),
            (R, gauss(n, 24, h, w, g))]
    dy = torch.cat([torch.randn(n, 16, h, w, device="cuda", generator=g).to(torch.bfloat16), dy_edge,
                    torch.randn(n, 24, h, w, device="cuda", generator=g).to(torch.bfloat16)], 1).contiguous(memory_format=CL)
    check(case, [dy], spy)


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters(momentum, eps, spy):
    case = make_case(8, 17, (64, 32, (R, 40), 96), 3)
    for b in case:
        if b[0] == "site":
            b[2].momentum, b[2].eps = momentum, eps
            b[2].num_batches_tracked.fill_(2 ** 40)
    dy = torch.randn(8, 232, 17, 17, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    check(case, [dy], spy)


def test_nchw_output_gradient(spy):
    case = make_case(8, 8, (320, 192, (R, 768)), 4)
    check(case, [torch.randn(8, 1280, 8, 8, device="cuda").to(torch.bfloat16)], spy)


def test_output_gradient_off_the_grid(spy):
    case = make_case(4, 7, (64, 32), 4)
    dy = torch.randn(4 * 96 * 49 + 1, device="cuda").to(torch.bfloat16)[1:].view(4, 7, 7, 96).permute(0, 3, 1, 2)
    assert dy.is_contiguous(memory_format=CL) and dy.data_ptr() % 16 == 2
    check(case, [dy], spy)


def test_retain_graph_with_two_backwards(spy):
    case = make_case(8, 14, (64, (R, 32), 96), 5)
    g = torch.Generator(device="cuda").manual_seed(5)
    dys = [torch.randn(8, 192, 14, 14, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL) for _ in range(2)]
    check(case, dys, spy)


def test_x_without_grad(spy):
    case = make_case(8, 14, (64, 96), 6)
    check(case, [torch.randn(8, 160, 14, 14, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)], spy, x_grad=False)


def test_max_pool_branch_gradient_keeps_eager_layout(spy):
    # InceptionB's ready branch: F.max_pool2d of the module input, whose backward picks its kernel by dy's layout
    g = torch.Generator(device="cuda").manual_seed(7)
    src = gauss(8, 288, 35, 35, g)
    case = [("site", gauss(8, 384, 17, 17, g), make_bn(384, 1)), ("site", gauss(8, 96, 17, 17, g), make_bn(96, 2))]
    for dy_layout in (CL, torch.contiguous_format):
        results = []
        for fused in (False, True):
            s = src.detach().clone().requires_grad_()
            branches = [(copy.deepcopy(b[2]), b[1]) for b in case] + [F.max_pool2d(s, kernel_size=3, stride=2)]
            y = fused_norm.bn_relu_concat(branches) if fused else torch.cat(
                [F.relu(b[0](b[1]), inplace=True) if isinstance(b, tuple) else b for b in branches], 1)
            y.backward(torch.ones_like(y).contiguous(memory_format=dy_layout) * 0.5)
            results.append((y.detach(), s.grad, s.grad.stride()))
        assert_same_values(results[1][0], results[0][0], "y")
        assert_same_values(results[1][1], results[0][1], "pool input grad")
        assert results[1][2] == results[0][2]


@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
@pytest.mark.parametrize("param_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_eval(mode, param_dtype, spy):
    g = torch.Generator(device="cuda").manual_seed(8)
    xs = [gauss(16, c, 8, 8, g) for c in (320, 384, 384)]
    ready = gauss(16, 768, 8, 8, g)
    bns = [make_bn(x.shape[1], i).to(param_dtype).eval() for i, x in enumerate(xs)]
    ctx = torch.no_grad if mode == "no_grad" else torch.inference_mode
    with ctx():
        want = torch.cat([F.relu(bn(x), inplace=True) for bn, x in zip(bns[:2], xs[:2])] + [ready, F.relu(bns[2](xs[2]))], 1)
        spy.calls.clear()
        got = fused_norm.bn_relu_concat([(bns[0], xs[0]), (bns[1], xs[1]), ready, (bns[2], xs[2])])
    assert spy.calls == ["b200c_bn_infer_slice"] * 3
    assert_same_values(got, want, "y")
    assert got.stride() == want.stride()


def off_grid(t):
    """A channels-last copy of `t` whose data pointer is 2 mod 16."""
    n, c, h, w = t.shape
    v = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    return v


@pytest.mark.parametrize("fallback", ["odd_channels", "off_grid", "fp32", "nchw", "mixed_modes", "cat_contiguous"])
def test_fallbacks_keep_eager_bits_without_a_slice_call(fallback, spy):
    case = make_case(4, 7, (64, 12 if fallback == "odd_channels" else 16, (R, 32), 32), 10)
    if fallback == "off_grid":
        case[1] = ("site", off_grid(case[1][1]), case[1][2])
    elif fallback == "fp32":
        case = [(b[0], b[1].float().contiguous(memory_format=CL), *b[2:]) for b in case]
    elif fallback == "nchw":
        case = [(b[0], b[1].contiguous(), *b[2:]) for b in case]
    elif fallback == "mixed_modes":
        case[0][2].eval()
    elif fallback == "cat_contiguous":
        # N = 1, W = 1: channels-last operands whose views (run's hooks) also fit the contiguous order, so torch.cat
        # writes a contiguous output, which is not rows of channels
        g = torch.Generator(device="cuda").manual_seed(10)
        case = [(b[0], gauss(1, b[1].shape[1], 196, 1, g), *b[2:]) for b in case]
        dy = torch.randn(1, 144, 196, 1, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
        check(case, [dy], spy, fused_calls=False)
        return
    c = sum(b[1].shape[1] for b in case)
    dy = torch.randn(4, c, 7, 7, device="cuda").to(case[0][1].dtype).contiguous(memory_format=CL)
    check(case, [dy], spy, fused_calls=False)


# ---- direct C-ABI calls: guard bytes past the scratch, semaphores left at zero, the rest of the output kept -------
GUARD = 64 << 10
SEMAPHORE_BYTES = 16384
PATTERN = 0x3F5A   # a bf16 that no call writes


def guarded_scratch(lib, c):
    need = int(lib.b200c_bn_scratch_bytes(c))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    return buf, need


def assert_scratch_kept(buf, need):
    torch.cuda.synchronize()
    assert (buf[need:] == 0xA5).all() and (buf[:SEMAPHORE_BYTES] == 0).all()


def slice_site_through_the_c_abi(lib, x, bn, out, c0, dy, dx, stream, buf):
    """One training site into out[:, c0:c0 + C] and its backward from dy[:, c0:c0 + C], through the C-ABI."""
    n, c, h, w = x.shape
    m = n * h * w
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device="cuda")
    stats = torch.empty(2 * c, device="cuda")
    dw, db = torch.full((c,), float("nan"), device="cuda"), torch.full((c,), float("nan"), device="cuda")
    rm, rv, nbt = bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()
    N.check(lib.b200c_bn_forward_slice(x.data_ptr(), out.data_ptr() + 2 * c0, out.shape[1], mask.data_ptr(), bn.weight.data_ptr(),
                                       bn.bias.data_ptr(), rm.data_ptr(), rv.data_ptr(), nbt.data_ptr(), stats.data_ptr(),
                                       stats.data_ptr() + 4 * c, m, c, bn.momentum, bn.eps, buf.data_ptr(), stream))
    N.check(lib.b200c_bn_backward_slice(dy.data_ptr() + 2 * c0, dy.shape[1], mask.data_ptr(), x.data_ptr(), dx.data_ptr(),
                                        bn.weight.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * c, dw.data_ptr(), db.data_ptr(), m,
                                        c, buf.data_ptr(), stream))
    return {"running_mean": rm, "running_var": rv, "nbt": nbt, "dweight": dw, "dbias": db}


def eager_site(x, bn, dy):
    x = x.detach().clone().requires_grad_()
    bn = copy.deepcopy(bn)
    y = F.relu(bn(x))
    y.backward(dy)
    return y.detach(), x.grad, {"running_mean": bn.running_mean, "running_var": bn.running_var, "nbt": bn.num_batches_tracked,
                                "dweight": bn.weight.grad, "dbias": bn.bias.grad}


@pytest.mark.parametrize("n,c,h,ldy,c0", [(2, 64, 32, 128, 0), (2, 64, 32, 128, 64), (32, 384, 8, 1280, 512),
                                          (2, 128, 3, 200, 40), (256, 32, 35, 288, 256)])
def test_c_abi_calls_keep_to_their_slice_and_scratch(n, c, h, ldy, c0):
    lib = N.load()
    g = torch.Generator(device="cuda").manual_seed(11)
    x = gauss(n, c, h, h, g)
    bn = make_bn(c, 11)
    out = torch.empty((n, ldy, h, h), dtype=torch.bfloat16, device="cuda").contiguous(memory_format=CL)
    out.view(torch.int16).fill_(PATTERN)
    dy_full = torch.randn(n, ldy, h, h, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    dy_before = dy_full.clone()
    dx = torch.full_like(x, float("nan"))
    buf, need = guarded_scratch(lib, c)
    before = N.launch_count()
    got = slice_site_through_the_c_abi(lib, x, bn, out, c0, dy_full, dx, torch.cuda.current_stream().cuda_stream, buf)
    assert_scratch_kept(buf, need)
    assert N.launch_count() - before == 4
    y_want, dx_want, want = eager_site(x, bn, dy_full[:, c0:c0 + c])
    assert_same_values(out[:, c0:c0 + c], y_want, "y")
    assert_same_values(dx, dx_want, "dx")
    for k in want:
        assert_same_values(got[k], want[k], k)
    outside = torch.cat([out[:, :c0], out[:, c0 + c:]], 1)
    assert (outside.view(torch.int16) == PATTERN).all(), "a write outside the slice"
    assert torch.equal(dy_full.view(torch.int16), dy_before.view(torch.int16))
    # eval, fp32 and bf16 parameters, into the same slice of a fresh pattern
    for dtype in (torch.float32, torch.bfloat16):
        ebn = copy.deepcopy(bn).to(dtype).eval()
        out.view(torch.int16).fill_(PATTERN)
        N.check(lib.b200c_bn_infer_slice(x.data_ptr(), out.data_ptr() + 2 * c0, ldy, ebn.weight.data_ptr(), ebn.bias.data_ptr(),
                                         ebn.running_mean.data_ptr(), ebn.running_var.data_ptr(), int(dtype == torch.bfloat16), ebn.eps,
                                         n * h * h, c, torch.cuda.current_stream().cuda_stream))
        with torch.no_grad():
            assert_same_values(out[:, c0:c0 + c], F.relu(ebn(x)), f"eval {dtype}")
        outside = torch.cat([out[:, :c0], out[:, c0 + c:]], 1)
        assert (outside.view(torch.int16) == PATTERN).all(), "an eval write outside the slice"


def test_two_streams_write_two_slices_of_one_output():
    lib = N.load()
    g = torch.Generator(device="cuda").manual_seed(12)
    n, h = 64, 17
    xs = [gauss(n, c, h, h, g) for c in (192, 384)]
    bns = [make_bn(x.shape[1], 20 + i) for i, x in enumerate(xs)]
    out = torch.empty((n, 576, h, h), dtype=torch.bfloat16, device="cuda").contiguous(memory_format=CL)
    out.view(torch.int16).fill_(PATTERN)
    dy = torch.randn(n, 576, h, h, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    dxs = [torch.full_like(x, float("nan")) for x in xs]
    streams = [torch.cuda.Stream() for _ in xs]
    bufs = [guarded_scratch(lib, x.shape[1]) for x in xs]
    torch.cuda.synchronize()
    got = []
    for i, (x, bn, st, (buf, _)) in enumerate(zip(xs, bns, streams, bufs)):
        with torch.cuda.stream(st):
            got.append(slice_site_through_the_c_abi(lib, x, bn, out, 192 * i, dy, dxs[i], st.cuda_stream, buf))
    for buf, need in bufs:
        assert_scratch_kept(buf, need)
    for i, (x, bn) in enumerate(zip(xs, bns)):
        y_want, dx_want, want = eager_site(x, bn, dy[:, 192 * i:192 * i + x.shape[1]])
        assert_same_values(out[:, 192 * i:192 * i + x.shape[1]], y_want, f"y{i}")
        assert_same_values(dxs[i], dx_want, f"dx{i}")
        for k in want:
            assert_same_values(got[i][k], want[k], f"{k}{i}")


def test_largest_m_times_ldy_below_2_31(spy):
    # m * ldy = 2^31 - 128: 16777215 rows of a 64-channel site and a 64-channel ready branch.  The values are compared
    # on the device (gpu_common.same_bits; the inputs hold no NaN), as test_gpu_bn_limits compares its largest sites.
    m = (2 ** 31 - 1) // 128
    case = make_case(1, 1, (64, (R, 64)), 13)
    g = torch.Generator(device="cuda").manual_seed(13)
    case = [("site", gauss(m, 64, 1, 1, g), case[0][2]), (R, gauss(m, 64, 1, 1, g))]
    dy = torch.randn(m, 128, 1, 1, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    want = run(case, [dy], False)
    spy.calls.clear()
    got = run(case, [dy], True)
    assert spy.calls == ["b200c_bn_forward_slice", "b200c_bn_backward_slice"], spy.calls
    assert got.keys() == want.keys()
    for k in want:
        assert got[k] == want[k] if k.endswith("stride") else same_bits(got[k], want[k]), k


def trace_cases():
    """Runs every case of KERNELS once under torch.profiler and prints {case: [b200c::bn_slice kernels]} as JSON."""
    from torch.profiler import ProfilerActivity, profile

    case = make_case(8, 14, (64, (R, 32), 96), 14)

    def train():
        branches = [(copy.deepcopy(b[2]), b[1].detach().clone().requires_grad_()) if b[0] == "site" else b[1] for b in case]
        fused_norm.bn_relu_concat(branches).sum().backward()

    def evaluate(dtype):
        with torch.no_grad():
            fused_norm.bn_relu_concat([(copy.deepcopy(b[2]).to(dtype).eval(), b[1]) if b[0] == "site" else b[1] for b in case])

    # as test_gpu_fused_cat.trace_cases: each case runs in three sessions, whose records are united
    cases = {}
    for name, fn in (("train", train), ("eval_fp32", lambda: evaluate(torch.float32)), ("eval_bf16", lambda: evaluate(torch.bfloat16))):
        names = set()
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names |= {e.name[e.name.index("b200c::bn_slice::"):].split("(")[0] for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_slice::" in e.name}
        cases[name] = sorted(names)
    print(json.dumps(cases))
