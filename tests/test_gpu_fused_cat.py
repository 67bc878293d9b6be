"""The concatenation batch-norm site (fused_norm.bn_relu_cat, norm_cat.cuh) against eager torch's
`relu(bn(torch.cat(segs, 1)))`, bit for bit (a NaN matches a NaN): y, the running statistics, num_batches_tracked,
dweight, dbias and every segment's gradient with its strides.

Shapes: every concatenation site of densenet121/161/169/201 at batch 32 and 224 x 224, densenet121's at batch 256,
1, 2, 49 and 64 segments, and the launch regimes of gpu_common.BN_REGIME_SHAPES realised as segment splits.  Value edges
and the momentum / eps range of test_gpu_fused_norm, an NCHW output gradient, eval under no_grad and inference_mode
with fp32 and bf16 parameters, the fallbacks (a segment of C_s % 8 != 0, a segment off the 16-byte grid, 65
segments: torch.cat and bn_relu, no concatenation call), direct C-ABI calls with guard bytes past the scratch, and the
memory the site saves.  `trace_cases` is the traced code of test_gpu_zz_trace_dense.py, which checks that every
`b200c::bn_cat` kernel is launched by the case test_fused_cat_cpu.KERNELS gives it."""
import copy
import ctypes
import json

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from gpu_common import BN_REGIME_SHAPES, assert_same_values
from test_gpu_fused_norm import edge_bn_setup, edge_site_inputs, make_bn

pytestmark = pytest.mark.gpu
CL = torch.channels_last


# (growth, initial features, block sizes) of torchvision's DenseNets
DENSENETS = {"densenet121": (32, 64, (6, 12, 24, 16)), "densenet161": (48, 96, (6, 12, 36, 24)),
             "densenet169": (32, 64, (6, 12, 32, 32)), "densenet201": (32, 64, (6, 12, 48, 32))}


def dense_sites(arch, size=224):
    """(segment channels, H, W) of every concatenation batch norm of `arch`: each dense layer's norm1, each transition's
    norm and norm5, in the order the forward runs them."""
    k, c, blocks = DENSENETS[arch]
    hw, sites = size // 4, []
    for b, layers in enumerate(blocks):
        segs = [c]
        for _ in range(layers):
            sites.append((tuple(segs), hw, hw))
            segs.append(k)
        sites.append((tuple(segs), hw, hw))   # the transition's norm, or norm5
        c = sum(segs) // 2
        if b < len(blocks) - 1:
            hw //= 2
    return sites


def segments(n, chans, h, w, seed, scale=2.0, shift=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [(torch.randn(n, c, h, w, device="cuda", generator=g) * scale + shift).to(torch.bfloat16).contiguous(memory_format=CL)
            for c in chans]


class Spy:
    """fused_norm's library handle, recording every concatenation call."""

    def __init__(self, lib):
        self.lib, self.calls = lib, []

    def __getattr__(self, name):
        if name.endswith("_cat"):
            self.calls.append(name)
        return getattr(self.lib, name)


@pytest.fixture
def spy(monkeypatch):
    s = Spy(N.load())
    monkeypatch.setattr(fused_norm, "_lib", s)
    return s


def run(bn, segs, dy, fused):
    segs = [(off_grid(s) if s.data_ptr() % 16 else s.detach().clone()).requires_grad_() for s in segs]
    relu = nn.ReLU(inplace=True)
    y = fused_norm.bn_relu_cat(bn, relu, segs) if fused else relu(bn(torch.cat(segs, 1)))
    y.backward(dy)
    out = {"y": y.detach(), "running_mean": bn.running_mean, "running_var": bn.running_var,
           "num_batches_tracked": bn.num_batches_tracked, "dweight": bn.weight.grad, "dbias": bn.bias.grad}
    for i, s in enumerate(segs):
        out[f"grad{i}"] = s.grad
        out[f"stride{i}"] = s.grad.stride()
    return out


def check(segs, dy, spy, bn_setup=None, momentum=0.1, eps=1e-5, nbt=5, fused_calls=True, seed=0):
    c = sum(s.shape[1] for s in segs)
    bn = make_bn(c, seed, momentum, eps, nbt)
    if bn_setup:
        bn_setup(bn)
    want = run(copy.deepcopy(bn), segs, dy, False)
    spy.calls.clear()
    got = run(copy.deepcopy(bn), segs, dy, True)
    expect = ["b200c_bn_forward_cat", "b200c_bn_backward_cat"] if fused_calls else []
    assert spy.calls == expect, spy.calls
    assert got.keys() == want.keys()
    for k in want:
        if k.startswith("stride"):
            assert got[k] == want[k], k
        else:
            assert_same_values(got[k], want[k], k)
    return want, got


def check_shape(n, chans, h, w, spy, seed=0, **kw):
    segs = segments(n, chans, h, w, seed)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    dy = torch.randn(n, sum(chans), h, w, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    return check(segs, dy, spy, seed=seed, **kw)


@pytest.mark.parametrize("arch", sorted(DENSENETS))
def test_every_densenet_site_at_batch_32(arch, spy):
    for chans, h, w in sorted(set(dense_sites(arch))):
        check_shape(32, chans, h, w, spy)


def test_densenet121_sites_at_batch_256(spy):
    for chans, h, w in sorted(set(dense_sites("densenet121"))):
        check_shape(256, chans, h, w, spy)


@pytest.mark.parametrize("chans", [(64,), (64, 32), (64,) + (32,) * 48, (64,) + (32,) * 63], ids=["1", "2", "49", "64"])
def test_segment_counts(chans, spy):
    check_shape(4, chans, 7, 7, spy)


def regime_split(c):
    """C (a multiple of 8) as segments: up to 4 of 8-multiples, uneven, or C alone where C is 8."""
    if c == 8:
        return (8,)
    a = max(8, c // 8 // 3 * 8)
    rest = c - a
    b = max(8, rest // 16 * 8) if rest > 8 else rest
    return tuple(x for x in (a, b, rest - b) if x)


@pytest.mark.parametrize("n,c,h,w", list(BN_REGIME_SHAPES))
def test_launch_regimes_as_segment_splits(n, c, h, w, spy):
    if c % 8:
        # no split takes these channels: the site concatenates and runs bn_relu
        check_shape(n, (c,), h, w, spy, fused_calls=False)
    else:
        chans = regime_split(c)
        assert sum(chans) == c and all(x % 8 == 0 for x in chans)
        check_shape(n, chans, h, w, spy)


@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges(grad_edges, spy):
    n, c, h, w = 8, 64, 16, 16
    x, dy, _ = edge_site_inputs(n, c, h, w, 7 + grad_edges, grad_edges)
    segs = [t.contiguous(memory_format=CL) for t in torch.split(x, [16, 24, 24], 1)]
    check(segs, dy.contiguous(memory_format=CL), spy, bn_setup=edge_bn_setup(grad_edges))


@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters(momentum, eps, spy):
    segs = segments(8, (64, 32, 32), 28, 28, 3)
    dy = torch.randn(8, 128, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    check(segs, dy, spy, momentum=momentum, eps=eps, nbt=2 ** 40)


def test_nchw_output_gradient(spy):
    segs = segments(8, (64, 32), 14, 14, 4)
    check(segs, torch.randn(8, 96, 14, 14, device="cuda").to(torch.bfloat16), spy)


def off_grid(t):
    """A channels-last copy of `t` whose data pointer is 2 mod 16."""
    n, c, h, w = t.shape
    v = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    v.copy_(t)
    assert v.is_contiguous(memory_format=CL) and v.data_ptr() % 16 == 2
    return v


@pytest.mark.parametrize("case", ["odd_channels", "off_grid", "65_segments"])
def test_fallbacks_keep_eager_bits_without_a_concatenation_call(case, spy):
    n, h, w = 4, 7, 7
    if case == "odd_channels":
        segs = segments(n, (64, 12, 32), h, w, 5)
    elif case == "off_grid":
        segs = segments(n, (64, 32), h, w, 5)
        segs[1] = off_grid(segs[1])
    else:
        segs = segments(n, (8,) * 65, h, w, 5)
    dy = torch.randn(n, sum(s.shape[1] for s in segs), h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    check(segs, dy, spy, fused_calls=False)


@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
@pytest.mark.parametrize("param_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_eval(mode, param_dtype, spy):
    segs = segments(16, (64, 32, 32, 32), 14, 14, 6)
    bn = make_bn(160, 6).to(param_dtype).eval()
    relu = nn.ReLU(inplace=True)
    ctx = torch.no_grad if mode == "no_grad" else torch.inference_mode
    with ctx():
        want = relu(bn(torch.cat(segs, 1)))
        spy.calls.clear()
        got = fused_norm.bn_relu_cat(bn, relu, segs)
    assert spy.calls == ["b200c_bn_infer_cat"]
    assert_same_values(got, want, "y")
    assert got.stride() == want.stride()


def test_functional_relu_site(spy):
    # norm5 with DenseNet's F.relu: relu None
    segs = segments(8, (64, 32, 32), 7, 7, 8)
    bn = make_bn(128, 8)
    ref = copy.deepcopy(bn)
    want = torch.relu_(ref(torch.cat(segs, 1)))
    spy.calls.clear()
    got = fused_norm.bn_relu_cat(bn, None, segs)
    assert spy.calls == ["b200c_bn_forward_cat"]
    assert_same_values(got, want, "y")
    assert_same_values(bn.running_var, ref.running_var, "running_var")


# ---- direct C-ABI calls: guard bytes past the scratch, semaphores left at zero ---------------------------
GUARD = 64 << 10
SEMAPHORE_BYTES = 16384


@pytest.mark.parametrize("n,chans,h,w", [(2, (64, 32), 32, 32), (32, (256,) + (32,) * 31, 7, 7), (2, (128, 64), 3, 3)])
def test_c_abi_calls_keep_to_their_scratch(n, chans, h, w):
    lib = N.load()
    c, m = sum(chans), n * h * w
    segs = segments(n, chans, h, w, 9)
    dy = torch.randn(n, c, h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL)
    bn = make_bn(c, 9)
    need = int(lib.b200c_bn_scratch_bytes(c))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    table = ((ctypes.c_void_p * len(segs))(*(s.data_ptr() for s in segs)), (ctypes.c_int * len(segs))(*chans), len(segs))
    y = torch.full((n, c, h, w), float("nan"), dtype=torch.bfloat16, device="cuda").contiguous(memory_format=CL)
    dx = torch.full_like(y, float("nan"))
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device="cuda")
    stats = torch.empty(2 * c, device="cuda")
    dw, db = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    rm, rv = bn.running_mean.clone(), bn.running_var.clone()
    nbt = bn.num_batches_tracked.clone()
    s = torch.cuda.current_stream().cuda_stream
    before = N.launch_count()
    N.check(lib.b200c_bn_forward_cat(*table, y.data_ptr(), mask.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(), rm.data_ptr(),
                                     rv.data_ptr(), nbt.data_ptr(), stats.data_ptr(), stats.data_ptr() + 4 * c, m, c, 0.1, 1e-5,
                                     buf.data_ptr(), s))
    torch.cuda.synchronize()
    assert (buf[need:] == 0xA5).all() and (buf[:SEMAPHORE_BYTES] == 0).all()
    N.check(lib.b200c_bn_backward_cat(dy.data_ptr(), mask.data_ptr(), *table, dx.data_ptr(), bn.weight.data_ptr(), stats.data_ptr(),
                                      stats.data_ptr() + 4 * c, dw.data_ptr(), db.data_ptr(), m, c, buf.data_ptr(), s))
    torch.cuda.synchronize()
    assert (buf[need:] == 0xA5).all() and (buf[:SEMAPHORE_BYTES] == 0).all()
    assert N.launch_count() - before == 4
    want = run(copy.deepcopy(bn), segs, dy, False)
    assert_same_values(y, want["y"], "y")
    assert_same_values(rv, want["running_var"], "running_var")
    assert_same_values(dw, want["dweight"], "dweight")
    c0 = 0
    for i, k in enumerate(chans):
        assert_same_values(dx[:, c0:c0 + k], want[f"grad{i}"], f"grad{i}")
        c0 += k


def test_site_saves_the_concatenation_s_memory():
    # densenet121's last dense layer of block 2 at batch 32: 12 segments over 28 x 28
    n, chans, h, w = 32, (128,) + (32,) * 11, 28, 28
    cat_bytes = n * sum(chans) * h * w * 2
    segs = [s.requires_grad_() for s in segments(n, chans, h, w, 10)]
    peaks = {}
    for fused in (False, True):
        bn = make_bn(sum(chans), 10)
        relu = nn.ReLU(inplace=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        y = fused_norm.bn_relu_cat(bn, relu, segs) if fused else relu(bn(torch.cat(segs, 1)))
        y.sum().backward()
        torch.cuda.synchronize()
        peaks[fused] = torch.cuda.max_memory_allocated() - base
        del y
        for s in segs:
            s.grad = None
    assert peaks[False] - peaks[True] >= cat_bytes // 2, (peaks, cat_bytes)


def trace_cases():
    """Runs every case of KERNELS once under torch.profiler and prints {case: [b200c::bn_cat kernels]} as JSON."""
    from torch.profiler import ProfilerActivity, profile

    segs = segments(8, (64, 32, 32), 14, 14, 11)
    cases = {}

    def train():
        s = [t.detach().clone().requires_grad_() for t in segs]
        fused_norm.bn_relu_cat(make_bn(128, 11), nn.ReLU(), s).sum().backward()

    def evaluate(dtype):
        bn = make_bn(128, 11).to(dtype).eval()
        with torch.no_grad():
            fused_norm.bn_relu_cat(bn, nn.ReLU(), segs)

    # A session now and then arrives without its first kernel records (test_gpu_fused_norm_paths.reducing_kernels), and
    # an eval case launches one kernel: each case runs in three sessions, whose records are united, since a case
    # launches the same kernels every time.
    for case, fn in (("train", train), ("eval_fp32", lambda: evaluate(torch.float32)), ("eval_bf16", lambda: evaluate(torch.bfloat16))):
        names = set()
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            names |= {e.name[e.name.index("b200c::bn_cat::"):].split("(")[0] for e in prof.events()
                      if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn_cat::" in e.name}
        cases[case] = sorted(names)
    print(json.dumps(cases))
