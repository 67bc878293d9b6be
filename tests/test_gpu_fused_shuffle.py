"""The ShuffleNetV2 block-end sites (fused_norm.bn_relu_shuffle, norm_shuffle.cuh) against eager torch's
`channel_shuffle(torch.cat((x1 or F.relu(bn_u(u)), F.relu(bn_t(t))), 1), 2)`, bit for bit (a NaN matches a NaN): y and
its strides, the running statistics, num_batches_tracked, dweight, dbias, dt, du, and x1's gradient with its strides.

Shapes: every block end of shufflenet_v2_x0_5 .. x2_0 at 224 x 224, both forms, at batch 32 and 256; the launch regimes
of gpu_common.BN_REGIME_SHAPES as branch widths (B % 8 == 0 and not).  Value edges and a momentum / eps range; a
channels-last, an NCHW, an off-grid and an expanded output gradient; retain_graph with two backwards; x without grad;
eval under no_grad and inference_mode with fp32 and bf16 parameters; the fallbacks (no shuffle call, eager bits and
strides); direct C-ABI calls with NaN-filled outputs and guard bytes past the scratch, whose semaphores end at zero;
two streams; and the largest n * 2B * h * w below 2^31.  `trace_cases` is the traced code of
test_gpu_zz_trace_shuffle.py, which checks that every `b200c::bn_shuffle` kernel is launched by the case
test_fused_shuffle_cpu.KERNELS gives it."""
import copy
import json

import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, BN_SEMAPHORES, assert_same_values
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn

torchvision = pytest.importorskip("torchvision")
from torchvision.models.shufflenetv2 import channel_shuffle  # noqa: E402

pytestmark = pytest.mark.gpu
CL = torch.channels_last

# branch widths B of each stage of shufflenet_v2_x0_5, x1_0, x1_5, x2_0, and the stages' sizes at 224 x 224
WIDTHS = {"x0_5": (24, 48, 96), "x1_0": (58, 116, 232), "x1_5": (88, 176, 352), "x2_0": (122, 244, 488)}
SIZES = (28, 14, 7)


class Spy:
    """fused_norm's library handle, recording every shuffle call."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        if name.endswith("_shuffle"):
            self.calls.append(name)
        return getattr(self.lib, name)


@pytest.fixture
def spy(monkeypatch):
    s = Spy(N.load())
    monkeypatch.setattr(fused_norm, "_lib", s)
    return s


def gauss(shape, g, scale=2.0, shift=0.5, fmt=CL):
    """bf16 values of `shape`; channels-last with a channel stride of 1 even for one channel (as a convolution writes
    it, and as torch's channels-last batch-norm kernels take it), or contiguous NCHW."""
    if fmt == CL:
        n, c, h, w = shape
        return torch.randn(n, h, w, c, dtype=torch.bfloat16, device="cuda", generator=g).permute(0, 3, 1, 2) * scale + shift
    return (torch.randn(*shape, dtype=torch.bfloat16, device="cuda", generator=g) * scale + shift).contiguous(memory_format=fmt)


def make_case(n, c, h, w, two, seed=0, momentum=0.1, eps=1e-5, nbt=5):
    """A block end's inputs: x (one form: NCHW [n, 2c, h, w], whose first half is x1) or u, t, and the batch norms."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    first = gauss((n, c, h, w), g) if two else gauss((n, 2 * c, h, w), g, fmt=torch.contiguous_format)
    return {"first": first, "t": gauss((n, c, h, w), g, 1.5, -0.2), "bn_t": make_bn(c, seed, momentum, eps, nbt),
            "bn_u": make_bn(c, seed + 1, momentum, eps, nbt) if two else None, "two": two}


def output_grad(case, seed=1, fmt=CL):
    n, c, h, w = case["t"].shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    return gauss((n, 2 * c, h, w), g, 1.0, 0.0, fmt)


def run(case, dys, fused, x_grad=True):
    """One forward (fused: bn_relu_shuffle; else eager torch) and a backward per dy (retain_graph between them)."""
    grads = {}
    bn_t = copy.deepcopy(case["bn_t"])
    # hooks on the leaves themselves: a view_as would restride a one-channel tensor, whose batch norm torch then runs on
    # its NCHW kernels
    t = case["t"].detach().clone().requires_grad_()
    tv = t
    tv.register_hook(lambda g: grads.setdefault("t", []).append((g.stride(), g.clone())))
    first = case["first"].detach().clone().requires_grad_(x_grad or case["two"])
    bn_u = None
    if case["two"]:
        bn_u = copy.deepcopy(case["bn_u"])
        a = first
        a.register_hook(lambda g: grads.setdefault("u", []).append((g.stride(), g.clone())))
    else:
        a = first.chunk(2, 1)[0]
        if a.requires_grad:
            a.register_hook(lambda g: grads.setdefault("x1", []).append((g.stride(), g.clone())))
    if fused:
        y = fused_norm.bn_relu_shuffle((bn_u, a, ()) if case["two"] else a, (bn_t, tv, ()))
    else:
        lead = F.relu(bn_u(a), inplace=True) if case["two"] else a
        y = channel_shuffle(torch.cat((lead, F.relu(bn_t(tv), inplace=True)), 1), 2)
    for k, dy in enumerate(dys):
        y.backward(dy.to(y.dtype), retain_graph=k + 1 < len(dys))
    out = {"y": y.detach(), "y_stride": y.stride(), "leaf_t": t.grad, "leaf_first": first.grad}
    for name, bn in (("t", bn_t), ("u", bn_u)):
        if bn is not None:
            out.update({f"running_mean_{name}": bn.running_mean, f"running_var_{name}": bn.running_var,
                        f"nbt_{name}": bn.num_batches_tracked, f"dweight_{name}": bn.weight.grad, f"dbias_{name}": bn.bias.grad})
    for k, v in grads.items():
        for j, (stride, g) in enumerate(v):
            out[f"grad_{k}_{j}"], out[f"grad_{k}_{j}_stride"] = g, stride
    return out


def compare(want, got):
    assert got.keys() == want.keys()
    for k in want:
        if k.endswith("stride"):
            assert got[k] == want[k], k
        elif want[k] is None:
            assert got[k] is None, k
        else:
            assert_same_values(got[k], want[k], k)


def check(case, dys, spy, fused_calls=True, x_grad=True):
    want = run(case, dys, False, x_grad)
    spy.calls.clear()
    got = run(case, dys, True, x_grad)
    expect = ["b200c_bn_forward_shuffle"] + ["b200c_bn_backward_shuffle"] * len(dys)
    assert spy.calls == (expect if fused_calls else []), spy.calls
    compare(want, got)
    return want, got


def scratch_semaphores_zero():
    for _, _, buf in fused_norm._scratch.values():
        assert not buf[:BN_SEMAPHORES * 4].any()


@pytest.mark.parametrize("n", [32, 256])
@pytest.mark.parametrize("width", list(WIDTHS))
def test_every_block_end_of_every_width(width, n, spy):
    for stage, (c, h) in enumerate(zip(WIDTHS[width], SIZES)):
        for two in (True, False):
            case = make_case(n, c, h, h, two, seed=stage)
            check(case, [output_grad(case)], spy)
    scratch_semaphores_zero()


@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
@pytest.mark.parametrize("n,c,h,w", [s for s in BN_REGIME_SHAPES if s[1] <= 65536])
def test_launch_regimes_as_branch_widths(n, c, h, w, two, spy):
    case = make_case(n, c, h, w, two, seed=c)
    check(case, [output_grad(case)], spy)
    scratch_semaphores_zero()


@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges(grad_edges, two, spy):
    n, c, h, w = 8, 64, 16, 16
    x, dy, other = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    case = make_case(n, c, h, w, two, seed=3)
    case["t"] = x.contiguous(memory_format=CL)
    if two:
        case["first"] = x.flip(1).contiguous(memory_format=CL)
    setup = edge_bn_setup(grad_edges)
    setup(case["bn_t"])
    if two:
        setup(case["bn_u"])
    # channel 2k of the output's gradient is the first operand's, 2k + 1 relu(bn_t(t))'s
    check(case, [torch.stack((other, dy), 2).reshape(n, 2 * c, h, w).contiguous(memory_format=CL)], spy)


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-5), (0.3, 1e-3), (0.1, 0.5)])
def test_hyperparameters(momentum, eps, spy):
    for two in (False, True):
        case = make_case(16, 58, 14, 14, two, seed=4, momentum=momentum, eps=eps)
        check(case, [output_grad(case)], spy)


def off_grid(t):
    """A channels-last copy of `t` whose data pointer is 2 mod 16."""
    n, c, h, w = t.shape
    v = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    assert v.is_contiguous(memory_format=CL) and v.data_ptr() % 16 == 2
    return v


@pytest.mark.parametrize("layout", ["nchw", "off_grid", "expanded"])
def test_output_gradient_layouts(layout, spy):
    for two in (False, True):
        for c in (58, 64):
            case = make_case(8, c, 14, 14, two, seed=5)
            dy = output_grad(case, fmt=torch.contiguous_format if layout == "nchw" else CL)
            if layout == "off_grid":
                dy = off_grid(dy)
            elif layout == "expanded":
                dy = torch.ones((), dtype=torch.bfloat16, device="cuda").expand(dy.shape)
            check(case, [dy], spy)


def test_retain_graph_with_two_backwards(spy):
    for two in (False, True):
        case = make_case(8, 58, 14, 14, two, seed=6)
        check(case, [output_grad(case, 1), output_grad(case, 2, torch.contiguous_format)], spy)


def test_x_without_grad(spy):
    case = make_case(8, 58, 14, 14, False, seed=7)
    want, got = check(case, [output_grad(case)], spy, x_grad=False)
    assert got["leaf_first"] is None and not any(k.startswith("grad_x1") for k in got)


@pytest.mark.parametrize("param_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
def test_eval(mode, param_dtype, spy):
    for two in (False, True):
        for c in (58, 64, 1):
            case = make_case(8, c, 14, 14, two, seed=8)
            bn_t = copy.deepcopy(case["bn_t"]).to(param_dtype).eval()
            bn_u = copy.deepcopy(case["bn_u"]).to(param_dtype).eval() if two else None
            ctx = torch.no_grad() if mode == "no_grad" else torch.inference_mode()
            with ctx:
                a = case["first"] if two else case["first"].chunk(2, 1)[0]
                want = channel_shuffle(torch.cat((F.relu(bn_u(a)) if two else a, F.relu(bn_t(case["t"]))), 1), 2)
                spy.calls.clear()
                got = fused_norm.bn_relu_shuffle((bn_u, a, ()) if two else a, (bn_t, case["t"], ()))
            assert spy.calls == ["b200c_bn_infer_shuffle"], (two, c, spy.calls)
            assert got.stride() == want.stride()
            assert_same_values(got, want, "y")


def fallback_case(kind):
    two = kind in ("u_nchw", "mixed")
    case = make_case(8, 58, 14, 14, two, seed=9)
    if kind == "x_channels_last":
        case["first"] = case["first"].contiguous(memory_format=CL)
    elif kind == "t_nchw":
        case["t"] = case["t"].contiguous()
    elif kind == "u_nchw":
        case["first"] = case["first"].contiguous()
    elif kind == "t_fp32":
        case["t"] = case["t"].float()
    elif kind == "hooked_bn":
        case["bn_t"].register_forward_hook(lambda *a: None)
    elif kind == "mixed":
        case["bn_u"].eval()
    return case


@pytest.mark.parametrize("kind", ["x_channels_last", "t_nchw", "u_nchw", "t_fp32", "hooked_bn", "mixed"])
def test_fallbacks_keep_eager_bits_without_a_shuffle_call(kind, spy):
    case = fallback_case(kind)
    check(case, [output_grad(case)], spy, fused_calls=False)


# ---- the C-ABI directly ----
GUARD = 64 << 10


def guarded_scratch(lib, c, two):
    need = lib.b200c_bn_dual_scratch_bytes(c) if two else lib.b200c_bn_scratch_bytes(c)
    buf = torch.zeros(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[need:] = 0xA5
    return buf, need


def nan_like(t, dtype=None):
    return torch.full_like(t, float("nan"), dtype=dtype)


def abi_site(lib, case, dy, stream, buf):
    """One forward and one backward through the C-ABI, every output NaN-filled first; returns y, the statistics, the
    gradients and each batch norm's running statistics."""
    t, first, two = case["t"], case["first"], case["two"]
    n, c, h, w = t.shape
    m = n * h * w
    bns = [copy.deepcopy(case["bn_t"])] + ([copy.deepcopy(case["bn_u"])] if two else [])
    y = torch.full((n, 2 * c, h, w), float("nan"), dtype=torch.bfloat16, device="cuda")
    masks = [torch.full((lib.b200c_bn_shuffle_mask_bytes(m, c),), 0x5A, dtype=torch.uint8, device="cuda") for _ in bns]
    stats = [torch.full((2 * c,), float("nan"), device="cuda") for _ in bns]

    def params(bn, mask, st):
        return (mask.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                bn.num_batches_tracked.data_ptr(), st.data_ptr(), st.data_ptr() + 4 * c, bn.momentum, bn.eps)

    lead = (None, 0, first.data_ptr(), *params(bns[1], masks[1], stats[1])) if two else \
        (first.data_ptr(), first.stride(0), None, *(None,) * 8, 0.0, 0.0)
    scratch = buf.data_ptr()
    N.check(lib.b200c_bn_forward_shuffle(*lead, t.data_ptr(), *params(bns[0], masks[0], stats[0]), y.data_ptr(), n, h * w, c,
                                         scratch, stream))
    outs = []
    for bn, x in zip(bns, [t, first]):
        outs.append((nan_like(x).contiguous(memory_format=CL), nan_like(bn.weight), nan_like(bn.bias)))

    def bwd(bn, mask, st, x, o):
        return (x.data_ptr(), mask.data_ptr(), o[0].data_ptr(), bn.weight.data_ptr(), st.data_ptr(), st.data_ptr() + 4 * c,
                o[1].data_ptr(), o[2].data_ptr())

    u_part = bwd(bns[1], masks[1], stats[1], first, outs[1]) if two else (None,) * 8
    tp = bwd(bns[0], masks[0], stats[0], t, outs[0])
    N.check(lib.b200c_bn_backward_shuffle(dy.data_ptr(), *u_part, tp[0], tp[1], tp[2], *tp[3:], m, c, scratch, stream))
    res = {"y": y}
    for i, bn in enumerate(bns):
        res.update({f"rm{i}": bn.running_mean, f"rv{i}": bn.running_var, f"nbt{i}": bn.num_batches_tracked, f"dx{i}": outs[i][0],
                    f"dw{i}": outs[i][1], f"db{i}": outs[i][2]})
    return res


def eager_site(case, dy):
    t = case["t"].detach().clone().requires_grad_()
    bns = [copy.deepcopy(case["bn_t"])] + ([copy.deepcopy(case["bn_u"])] if case["two"] else [])
    if case["two"]:
        u = case["first"].detach().clone().requires_grad_()
        lead = F.relu(bns[1](u))
    else:
        lead = case["first"].chunk(2, 1)[0]
    y = channel_shuffle(torch.cat((lead, F.relu(bns[0](t))), 1), 2)
    y.backward(dy)
    res = {"y": y.detach()}
    for i, (bn, x) in enumerate(zip(bns, [t] + ([u] if case["two"] else []))):
        res.update({f"rm{i}": bn.running_mean, f"rv{i}": bn.running_var, f"nbt{i}": bn.num_batches_tracked, f"dx{i}": x.grad,
                    f"dw{i}": bn.weight.grad, f"db{i}": bn.bias.grad})
    return res


@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
@pytest.mark.parametrize("n,c,h", [(64, 3, 32), (8, 58, 28), (2, 64, 1), (4, 100, 16), (64, 17, 32)])
def test_c_abi_calls_keep_to_their_scratch(n, c, h, two):
    lib = N.load()
    case = make_case(n, c, h, h, two, seed=10)
    dy = output_grad(case)
    buf, need = guarded_scratch(lib, c, two)
    got = abi_site(lib, case, dy, torch.cuda.current_stream().cuda_stream, buf)
    torch.cuda.synchronize()
    want = eager_site(case, dy)
    for k in want:
        assert_same_values(got[k], want[k], k)
    assert (buf[need:] == 0xA5).all()
    assert not buf[:BN_SEMAPHORES * 4].any()


def test_two_streams():
    cases = [make_case(16, 58, 28, 28, two, seed=11 + two) for two in (False, True)]
    dys = [output_grad(c) for c in cases]
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


@pytest.mark.parametrize("two,c,w", [(False, 58, (2 ** 31 - 1) // 116), (True, 64, (2 ** 31 - 1) // 128)])
def test_largest_n_2b_hw_below_2_31(two, c, w, spy):
    case = make_case(1, c, 1, w, two, seed=12)
    assert 2 * case["t"].numel() < 2 ** 31 <= 2 * (case["t"].numel() + c)
    check(case, [output_grad(case)], spy)
    del case
    torch.cuda.empty_cache()


def trace_cases():
    """Runs every case of KERNELS once under torch.profiler and prints {case: [b200c::bn_shuffle kernels]} as JSON."""
    from torch.profiler import ProfilerActivity, profile

    cases = {two: make_case(8, 58, 14, 14, two, seed=13) for two in (False, True)}

    def train(two):
        run(cases[two], [output_grad(cases[two])], True)

    def evaluate(two, dtype):
        case = cases[two]
        bn_t = copy.deepcopy(case["bn_t"]).to(dtype).eval()
        with torch.no_grad():
            if two:
                fused_norm.bn_relu_shuffle((copy.deepcopy(case["bn_u"]).to(dtype).eval(), case["first"], ()), (bn_t, case["t"], ()))
            else:
                fused_norm.bn_relu_shuffle(case["first"].chunk(2, 1)[0], (bn_t, case["t"], ()))

    # as test_gpu_fused_cat.trace_cases: each case runs in three sessions, whose records are united
    out = {}
    for name, fn in (("train_one", lambda: train(False)), ("train_two", lambda: train(True)),
                     ("eval_one_fp32", lambda: evaluate(False, torch.float32)), ("eval_two_fp32", lambda: evaluate(True, torch.float32)),
                     ("eval_one_bf16", lambda: evaluate(False, torch.bfloat16)), ("eval_two_bf16", lambda: evaluate(True, torch.bfloat16))):
        names = set()
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names |= {e.name[e.name.index("b200c::bn_shuffle::"):].split("(")[0] for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_shuffle::" in e.name}
        out[name] = sorted(names)
    print(json.dumps(out))
