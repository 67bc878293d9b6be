"""VGG's stage-end sites (fused_norm.bn_relu_maxpool with nn.MaxPool2d(2, 2), norm_pool2.cuh) against eager torch's
`pool(relu(bn(x)))`, bit for bit (a NaN matches a NaN): y and its strides, the running statistics, num_batches_tracked,
dx, dweight and dbias.

Shapes: every pool site of vgg11_bn .. vgg19_bn at 224 x 224 (the four models share them) at batch 32 and 256; the
launch regimes of gpu_common.BN_REGIME_SHAPES; C = 100 and a misaligned x (the one-channel kernels); odd 7 x 7 and
15 x 9 inputs, whose last row and column take no window.  Value edges of x and dy, ties inside a window, all-negative
windows, NaN, -0.0 and +-Inf; a momentum / eps range; channels-last, NCHW and expanded output gradients; retain_graph;
x without grad; eval under no_grad and inference_mode with fp32 and bf16 parameters; direct C-ABI calls with
NaN-filled outputs and guard bytes past a scratch of exactly the library's size, whose semaphores end at zero; two
streams; and n * c * h * w just below 2^31.  `trace_cases` is the traced code of test_gpu_zz_trace_vgg.py, which
checks that every `b200c::bn_pool2` kernel is launched by the case test_fused_vgg_cpu.KERNELS gives it."""
import copy
import json

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, BN_SEMAPHORES, assert_same_values, bits_of, edge_values
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn, misaligned

pytestmark = pytest.mark.gpu
CL = torch.channels_last

# (C, H) of the five pool sites of every VGG-BN model at 224 x 224
VGG_SITES = [(64, 224), (128, 112), (256, 56), (512, 28), (512, 14)]


class Spy:
    """fused_norm's library handle, recording every pool2 call."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        if name.endswith("_pool2"):
            self.calls.append(name)
        return getattr(self.lib, name)


@pytest.fixture
def spy(monkeypatch):
    s = Spy(N.load())
    monkeypatch.setattr(fused_norm, "_lib", s)
    return s


def gauss(shape, g, scale=2.0, shift=0.5, fmt=CL):
    """bf16 values of `shape`, channels-last with a channel stride of 1 (as a convolution writes it), or NCHW."""
    n, c, h, w = shape
    if fmt == CL:
        return torch.randn(n, h, w, c, dtype=torch.bfloat16, device="cuda", generator=g).permute(0, 3, 1, 2) * scale + shift
    return (torch.randn(*shape, dtype=torch.bfloat16, device="cuda", generator=g) * scale + shift).contiguous()


def make_case(n, c, h, w, seed=0, momentum=0.1, eps=1e-5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return {"x": gauss((n, c, h, w), g), "bn": make_bn(c, seed, momentum, eps)}


def output_grad(x, seed=1, fmt=CL):
    n, c, h, w = x.shape
    return gauss((n, c, h // 2, w // 2), torch.Generator(device="cuda").manual_seed(seed), 1.0, 0.0, fmt)


def run(case, dys, fused, x_grad=True):
    """One forward (fused: bn_relu_maxpool; else eager torch) and a backward per dy (retain_graph between them)."""
    bn = copy.deepcopy(case["bn"])
    # a misaligned case keeps its x off the 16-byte grid (a clone would land on it)
    x = (misaligned(case["x"]) if case.get("misalign") else case["x"].detach().clone()).requires_grad_(x_grad)
    relu, pool = nn.ReLU(inplace=True), nn.MaxPool2d(2, 2)
    y = fused_norm.bn_relu_maxpool(bn, relu, pool, x) if fused else pool(relu(bn(x)))
    res = {"y": y.detach().clone(), "stride": y.stride(), "rm": bn.running_mean, "rv": bn.running_var, "nbt": bn.num_batches_tracked}
    for i, dy in enumerate(dys):
        y.backward(dy, retain_graph=i + 1 < len(dys))
        res.update({f"dx{i}": None if x.grad is None else x.grad.clone(), f"dw{i}": bn.weight.grad.clone(),
                    f"db{i}": bn.bias.grad.clone()})
        x.grad = bn.weight.grad = bn.bias.grad = None
    return res


def compare(want, got):
    assert got["stride"] == want["stride"]
    for k in want:
        if k != "stride":
            if want[k] is None:
                assert got[k] is None, k
            else:
                assert_same_values(got[k], want[k], k)


def check(case, dys, spy, x_grad=True, fused_calls=True):
    want = run(case, dys, False, x_grad)
    spy.calls.clear()
    got = run(case, dys, True, x_grad)
    expect = ["b200c_bn_forward_pool2"] + ["b200c_bn_backward_pool2"] * len(dys)
    assert spy.calls == (expect if fused_calls else []), spy.calls
    compare(want, got)
    return want, got


def scratch_semaphores_zero():
    for _, _, buf in fused_norm._scratch.values():
        assert not buf[:BN_SEMAPHORES * 4].any()


@pytest.mark.parametrize("n", [32, 256])
def test_every_pool_site_of_vgg(n, spy):
    for i, (c, h) in enumerate(VGG_SITES):
        case = make_case(n, c, h, h, seed=i)
        check(case, [output_grad(case["x"])], spy)
        del case
    scratch_semaphores_zero()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("n,c,h,w", [s for s in BN_REGIME_SHAPES if min(s[2:]) >= 2])
def test_launch_regimes(n, c, h, w, spy):
    case = make_case(n, c, h, w, seed=c)
    check(case, [output_grad(case["x"])], spy)
    scratch_semaphores_zero()
    del case
    torch.cuda.empty_cache()


@pytest.mark.parametrize("c", [100, 64])
def test_one_channel_kernels(c, spy):
    """C = 100 (C % 8 != 0) and a misaligned x both run the kernels of one channel per thread."""
    case = make_case(8, c, 28, 28, seed=2)
    case["misalign"] = c == 64
    check(case, [output_grad(case["x"])], spy)


@pytest.mark.parametrize("h,w", [(7, 7), (15, 9), (2, 2), (3, 2)])
def test_odd_spatial_sizes(h, w, spy):
    for c in (64, 100):
        case = make_case(4, c, h, w, seed=h * w)
        want, got = check(case, [output_grad(case["x"])], spy)
        if h % 2:
            assert (bits_of(got["dx0"][:, :, h - 1]) != 0).any()   # the row outside every window still has dx
        assert got["y"].shape == (4, c, h // 2, w // 2)


@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges(grad_edges, spy):
    n, c, h, w = 8, 64, 16, 16
    x, _, _ = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    case = make_case(n, c, h, w, seed=3)
    case["x"] = x.contiguous(memory_format=CL)
    edge_bn_setup(grad_edges)(case["bn"])
    g = torch.Generator(device="cuda").manual_seed(4)
    dy = torch.randn(n, h // 2, w // 2, c, device="cuda", generator=g)
    if grad_edges:
        pat = edge_values(torch.bfloat16).float().cuda()
        dy[..., 16:48] = pat[torch.randint(0, pat.numel(), dy[..., 16:48].shape, device="cuda", generator=g)]
        dy[:2, ..., c - 2:] = float("nan")
    check(case, [dy.to(torch.bfloat16).permute(0, 3, 1, 2)], spy)


def test_ties_negative_windows_nan_inf_and_negative_zero_gradient(spy):
    """Channels of x constant over each window (every element ties), windows all below the mean (the ReLU stops every
    gradient), NaN and +-Inf at one position of a window, and a dy of -0.0 everywhere: the single window's gradient
    passes as it is, so dx and the sums see -0.0."""
    n, c, h, w = 4, 64, 8, 8
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(n, h, w, c, device="cuda", generator=g)
    x[..., 0:8] = x[:, ::2, ::2, 0:8].repeat_interleave(2, 1).repeat_interleave(2, 2)   # ties in every window
    x[..., 8:16] = -50.0   # all-negative windows
    x[0, 1, 1, 16] = float("nan")
    x[1, 2, 3, 17] = float("nan")
    x[1, 3, 3, 17] = float("nan")   # two NaNs in one window: the last wins
    x[2, 4, 4, 18] = float("inf")
    x[3, 5, 4, 19] = float("-inf")
    case = make_case(n, c, h, w, seed=5)
    case["x"] = x.to(torch.bfloat16).permute(0, 3, 1, 2)
    for dy in (torch.full((n, h // 2, w // 2, c), -0.0, device="cuda"),
               torch.where(torch.rand(n, h // 2, w // 2, c, device="cuda", generator=g) < 0.5, -0.0, 1.0)):
        dy[0, 0, 0, 20] = float("nan")
        dy[0, 1, 0, 21] = float("inf")
        check(case, [dy.to(torch.bfloat16).permute(0, 3, 1, 2)], spy)


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-5), (0.3, 1e-3), (0.1, 0.5)])
def test_hyperparameters(momentum, eps, spy):
    case = make_case(16, 128, 14, 14, seed=6, momentum=momentum, eps=eps)
    check(case, [output_grad(case["x"])], spy)


@pytest.mark.parametrize("layout", ["channels_last", "nchw", "expanded"])
def test_output_gradient_layouts(layout, spy):
    for c in (100, 64):
        case = make_case(8, c, 14, 14, seed=7)
        dy = output_grad(case["x"], fmt=torch.contiguous_format if layout == "nchw" else CL)
        if layout == "expanded":
            dy = torch.ones((), dtype=torch.bfloat16, device="cuda").expand(dy.shape)
        check(case, [dy], spy)


def test_retain_graph_with_two_backwards(spy):
    case = make_case(8, 64, 14, 14, seed=8)
    check(case, [output_grad(case["x"], 1), output_grad(case["x"], 2, torch.contiguous_format)], spy)


def test_x_without_grad(spy):
    case = make_case(8, 64, 14, 14, seed=9)
    want, got = check(case, [output_grad(case["x"])], spy, x_grad=False)
    assert got["dx0"] is None


@pytest.mark.parametrize("param_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
def test_eval(mode, param_dtype, spy):
    for c, h, w in ((64, 14, 14), (100, 7, 9), (8, 2, 2)):
        case = make_case(8, c, h, w, seed=10)
        bn = copy.deepcopy(case["bn"]).to(param_dtype).eval()
        relu, pool = nn.ReLU(inplace=True), nn.MaxPool2d(2, 2)
        with torch.no_grad() if mode == "no_grad" else torch.inference_mode():
            want = pool(relu(bn(case["x"])))
            spy.calls.clear()
            got = fused_norm.bn_relu_maxpool(bn, relu, pool, case["x"])
        assert spy.calls == ["b200c_bn_infer_pool2"], spy.calls
        assert got.stride() == want.stride()
        assert_same_values(got, want, "y")


def test_other_pools_and_hooks_keep_eager_bits_without_a_pool2_call(spy):
    for pool in (nn.MaxPool2d(2, 2, ceil_mode=True), nn.MaxPool2d(3, 2), nn.MaxPool2d(2, 1)):
        case = make_case(4, 64, 9, 9, seed=11)
        want = pool(nn.ReLU()(copy.deepcopy(case["bn"])(case["x"])))
        spy.calls.clear()
        got = fused_norm.bn_relu_maxpool(copy.deepcopy(case["bn"]), nn.ReLU(), pool, case["x"])
        assert spy.calls == []
        assert_same_values(got, want, "y")
    case = make_case(4, 64, 8, 8, seed=12)
    case["bn"].register_forward_hook(lambda *a: None)
    check(case, [output_grad(case["x"])], spy, fused_calls=False)


# ---- the C-ABI directly ----
GUARD = 64 << 10


def abi_site(lib, case, dy, stream, buf):
    """One forward and one backward through the C-ABI, every output NaN-filled (argmax 0x5A) first."""
    x = case["x"]
    n, c, h, w = x.shape
    bn = copy.deepcopy(case["bn"])
    y = torch.full((n, h // 2, w // 2, c), float("nan"), dtype=torch.bfloat16, device="cuda").permute(0, 3, 1, 2)
    argmax = torch.full((y.numel(),), 0x5A, dtype=torch.uint8, device="cuda")
    stats = torch.full((2 * c,), float("nan"), device="cuda")
    s = stats.data_ptr()
    N.check(lib.b200c_bn_forward_pool2(x.data_ptr(), y.data_ptr(), argmax.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(),
                                       bn.running_mean.data_ptr(), bn.running_var.data_ptr(), bn.num_batches_tracked.data_ptr(), s,
                                       s + 4 * c, n, h, w, c, bn.momentum, bn.eps, buf.data_ptr(), stream))
    dx = torch.full_like(x, float("nan")).contiguous(memory_format=CL)
    dw, db = (torch.full((c,), float("nan"), device="cuda") for _ in range(2))
    N.check(lib.b200c_bn_backward_pool2(dy.data_ptr(), argmax.data_ptr(), x.data_ptr(), dx.data_ptr(), bn.weight.data_ptr(), s,
                                        s + 4 * c, dw.data_ptr(), db.data_ptr(), n, h, w, c, buf.data_ptr(), stream))
    return {"y": y, "rm": bn.running_mean, "rv": bn.running_var, "nbt": bn.num_batches_tracked, "dx0": dx, "dw0": dw, "db0": db}


@pytest.mark.parametrize("n,c,h,w", [(64, 3, 32, 32), (8, 64, 28, 28), (4, 100, 15, 9), (2, 2048, 5, 5), (64, 17, 32, 32)])
def test_c_abi_calls_keep_to_their_scratch(n, c, h, w):
    lib = N.load()
    case = make_case(n, c, h, w, seed=13)
    dy = output_grad(case["x"])
    need = lib.b200c_bn_scratch_bytes(c)
    buf = torch.zeros(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[need:] = 0xA5
    before = lib.b200c_launch_count()
    got = abi_site(lib, case, dy, torch.cuda.current_stream().cuda_stream, buf)
    torch.cuda.synchronize()
    assert lib.b200c_launch_count() == before + 4
    want = run(case, [dy], False)
    for k in got:
        assert_same_values(got[k], want[k], k)
    assert (buf[need:] == 0xA5).all()
    assert not buf[:BN_SEMAPHORES * 4].any()


def test_two_streams():
    cases = [make_case(16, c, 28, 28, seed=14 + c) for c in (64, 100)]
    dys = [output_grad(c["x"]) for c in cases]
    wants = [run(c, [dy], False) for c, dy in zip(cases, dys)]
    streams = [torch.cuda.Stream() for _ in cases]
    torch.cuda.synchronize()
    gots = []
    for case, dy, s in zip(cases, dys, streams):
        with torch.cuda.stream(s):
            gots.append(run(case, [dy], True))
    torch.cuda.synchronize()
    for want, got in zip(wants, gots):
        compare(want, got)


def test_largest_nchw_below_2_31(spy):
    c, h = 64, 2
    w = (2 ** 31 - 1) // (c * h)
    case = make_case(1, c, h, w, seed=15)
    assert case["x"].numel() < 2 ** 31 <= case["x"].numel() + c * h
    check(case, [output_grad(case["x"])], spy)
    del case
    torch.cuda.empty_cache()


def trace_cases():
    """Runs every case of KERNELS once under torch.profiler and prints {case: [b200c::bn_pool2 kernels]} as JSON."""
    from torch.profiler import ProfilerActivity, profile

    def train(c, misalign):
        case = make_case(8, c, 14, 14, seed=16)
        case["misalign"] = misalign
        run(case, [output_grad(case["x"])], True)

    def evaluate(c, dtype):
        case = make_case(8, c, 14, 14, seed=17)
        bn = copy.deepcopy(case["bn"]).to(dtype).eval()
        with torch.no_grad():
            fused_norm.bn_relu_maxpool(bn, nn.ReLU(), nn.MaxPool2d(2, 2), case["x"])

    # as test_gpu_fused_cat.trace_cases: each case runs in three sessions, whose records are united
    out = {}
    for name, fn in (("train_vec", lambda: train(64, False)), ("train_scalar", lambda: train(64, True)),
                     ("eval_vec_fp32", lambda: evaluate(64, torch.float32)), ("eval_scalar_fp32", lambda: evaluate(100, torch.float32)),
                     ("eval_vec_bf16", lambda: evaluate(64, torch.bfloat16)), ("eval_scalar_bf16", lambda: evaluate(100, torch.bfloat16))):
        names = set()
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names |= {e.name[e.name.index("b200c::bn_pool2::"):].split("(")[0] for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_pool2::" in e.name}
        out[name] = sorted(names)
    print(json.dumps(out))
