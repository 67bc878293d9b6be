"""The ShuffleNetV2 block-end kernels (norm_shuffle.cuh) and the Inception slice kernels (norm_slice.cuh) through the
C-ABI, every operand in an allocation of its own, against eager torch bit for bit and against plain references for
what torch does not compute.

Each operand sits `offset` bytes past a 16-byte boundary between a head and a tail guard of GUARD bytes filled with
PATTERN; outputs are filled with all-ones bits (a NaN; masks 0xA5) before the call.  After every call: every guard
byte is unchanged, every input (t, u, x1 with the gaps between its samples, dy, x) is bitwise unchanged, the scratch's
guard is intact and its semaphores are zero, and b200c_launch_count grew by 2 per training call and 1 per eval call.

Shuffle (b200c_bn_forward_shuffle, b200c_bn_backward_shuffle, b200c_bn_infer_shuffle), both forms, at every shape of
SHUFFLE_SHAPES (test_shuffle_shapes_reach_every_tile_and_launch_regime checks on the CPU which regimes they reach):
- eager `channel_shuffle(torch.cat((x1 or relu(bn_u(u)), relu(bn_t(t))), 1), 2)` bit for bit: y, the running
  statistics, num_batches_tracked, dt, du, dweight and dbias; the stride-1 form's even planes of y against x1's bits;
- each mask against its bit rule (bit c % 8 of byte r * ceil(B / 8) + c / 8 is !(y <= 0), padding bits 0), in exactly
  b200c_bn_shuffle_mask_bytes(m, B) bytes;
- the saved mean and invstd against float64;
- t, u, x1, y, dt and du alone at 2, 6 and 10 bytes past the 16-byte grid, dy at 4 and 12, each mask at 1 and 3 and
  the fp32 outputs at 4: every output keeps the aligned call's bits;
- x1's sample stride at B * hw, 2B * hw and 2B * hw + 3 with NaN between the samples' planes, and x1 holding every
  bf16 bit pattern (NaN payloads, +-0, +-Inf, subnormals), in training and eval;
- a null num_batches_tracked for t and, separately, u, every other output keeping the non-null call's bits;
- eval with fp32 and bf16 parameters, also at m = 1.

Slice (b200c_bn_forward_slice, b200c_bn_backward_slice, b200c_bn_infer_slice) at every BN_REGIME_SHAPES width with
C % 8 == 0 and at two small widths, each in an output of row stride ldy with a pattern outside the slice: the whole
output (ldy == C, c0 = 0), a last slice ending at ldy, middle slices, and dy's row stride lddy == C, lddy > ldy and
lddy < ldy.  Against eager `relu(bn(x))`: y inside the slice, the running statistics, num_batches_tracked, dx, dweight
and dbias bit for bit; the mask against check_mask over the branch's own m * C / 8 bytes; the saved statistics
against float64; the mask at 1 and 3 and the fp32 outputs at 4 bytes off the grid with the aligned call's bits; eval
with fp32 and bf16 parameters."""
import copy

import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import _native as N
from gpu_common import BN_REGIME_SHAPES, bn_launch_config
from test_gpu_bn_limits import check_mask, check_shuffle_mask, same
from test_gpu_fused_norm import GUARD, check_scratch, check_stats_against_float64, make_bn
from test_gpu_fused_shuffle import eager_site as eager_shuffle
from test_gpu_fused_shuffle import make_case, output_grad
from test_gpu_fused_slice import eager_site as eager_slice

torchvision = pytest.importorskip("torchvision")
from torchvision.models.shufflenetv2 import channel_shuffle  # noqa: E402

gpu = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
PATTERN = 0x5C      # every guard byte
OUT_PATTERN = 0x3F5A   # a bf16 outside the slice, which no call writes
TILE = 32           # norm_shuffle.cuh's kTile


# ---- operands between guards --------------------------------------------------------------------------------------
class Arena:
    """One allocation holding one operand of `numel` elements `offset` bytes past a 16-byte boundary, between a head
    and a tail guard of at least GUARD bytes of PATTERN."""

    def __init__(self, numel, dtype, offset=0):
        size = torch.empty((), dtype=dtype).element_size()
        self.buf = torch.full((2 * GUARD + 16 + numel * size,), PATTERN, dtype=torch.uint8, device="cuda")
        self.lo, self.hi = GUARD + offset, GUARD + offset + numel * size
        self.t = self.buf[self.lo:self.hi].view(dtype)
        self.snapshot = None
        assert self.t.data_ptr() % 16 == offset

    def guards_intact(self):
        return bool((self.buf[:self.lo] == PATTERN).all()) and bool((self.buf[self.hi:] == PATTERN).all())


class Operands:
    """The arenas of one call, placed as `place` (name -> byte offset) says."""

    def __init__(self, place=None):
        self.place, self.ins, self.outs = place or {}, {}, {}

    def input(self, name, src, key=None):
        a = Arena(src.numel(), src.dtype, self.place.get(key or name, 0))
        a.t.copy_(src.reshape(-1))
        self.ins[name] = a
        return a.t

    def output(self, name, numel, dtype, key=None, init=None):
        """An output filled with all-ones bits (0xA5 for bytes), or a copy of `init` (an in-out operand)."""
        a = Arena(numel, dtype, self.place.get(key or name, 0))
        if init is not None:
            a.t.copy_(init.reshape(-1))
        elif dtype == torch.uint8:
            a.t.fill_(0xA5)
        else:
            a.t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[a.t.element_size()]).fill_(-1)
        self.outs[name] = a
        return a.t

    def seal(self):
        """Snapshots every input allocation as filled."""
        for a in self.ins.values():
            a.snapshot = a.buf.clone()

    def check(self):
        torch.cuda.synchronize()
        bad = [k for k, a in {**self.ins, **self.outs}.items() if not a.guards_intact()]
        assert not bad, f"a call wrote into the guard bytes of {bad}"
        changed = [k for k, a in self.ins.items() if not torch.equal(a.buf, a.snapshot)]
        assert not changed, f"a call changed its inputs {changed}"


def p(t):
    return t.data_ptr() if t is not None else None


def guarded_scratch(c, two):
    lib = N.load()
    need = int(lib.b200c_bn_dual_scratch_bytes(c) if two else lib.b200c_bn_scratch_bytes(c))
    buf = torch.empty(need + GUARD, dtype=torch.uint8, device="cuda")
    buf[:need].zero_()
    buf[need:].fill_(0xA5)
    return buf, need


def assert_same_outputs(got, want, where):
    assert got.keys() == want.keys(), where
    for k in want:
        if want[k] is None:
            assert got[k] is None, (where, k)
        else:
            same(got[k], want[k], f"{where}: {k}")


# ---- shuffle ------------------------------------------------------------------------------------------------------
# (n, B, hw): m = 2, m < 32, m % 32 != 0, B < 8 and B % 8 != 0, partial channel tiles, tiles over several samples and
# over a boundary with hw > 32, block.x below 32 and above it, several channel tiles, a collapsed and a merged grid
SHUFFLE_SHAPES = [(2, 3, 1), (1, 7, 7), (1, 33, 31), (3, 8, 33), (5, 58, 49), (2, 100, 196), (1400, 1, 49), (64, 32, 49),
                  (3, 257, 7), (2, 2048, 7), (8, 17, 31), (37, 31, 1)]
SHUFFLE_WIDTHS = {1, 3, 7, 8, 17, 31, 32, 33, 58, 100, 257, 2048}
SHUFFLE_HW = {1, 7, 31, 33, 49, 196}


def tiles_samples(m, hw):
    """For each kTile-row tile of [m] rows: (its first sample, its last sample)."""
    return [(r0 // hw, (min(r0 + TILE, m) - 1) // hw) for r0 in range(0, m, TILE)]


def test_shuffle_shapes_reach_every_tile_and_launch_regime():
    seen = set()
    assert {b for _, b, _ in SHUFFLE_SHAPES} == SHUFFLE_WIDTHS and {hw for _, _, hw in SHUFFLE_SHAPES} == SHUFFLE_HW
    for n, c, hw in SHUFFLE_SHAPES:
        m = n * hw
        cfg = bn_launch_config(m, c)
        tiles = tiles_samples(m, hw)
        checks = {"m = 2": m == 2, "m < 32": m < 32, "partial last row tile": m % TILE != 0,
                  "partial channel tile": c % TILE != 0, "B < 8": c < 8, "padding bits": c % 8 != 0,
                  "a tile over three samples": any(b - a >= 2 for a, b in tiles),
                  "a sample boundary in a tile, hw > 32": hw > TILE and any(b > a for a, b in tiles),
                  "collapsed grid": cfg.grid_y == 1, "merged grid": cfg.grid_y >= 8,
                  "block_x < 32": cfg.block_x < 32, "grid_x > 1": cfg.grid_x > 1}
        seen |= {k for k, v in checks.items() if v}
    missing = set(checks) - seen
    assert not missing, missing


class ShuffleSite:
    """make_case's block end of n samples, B channels per branch and h = 1, w = hw, its output gradient, and the
    operands as the C-ABI reads them: t and u as [m][B] rows, x1 as [n][B * hw] planes, dy as [m][2B] rows.  With
    `x1_bits`, x1 holds every bf16 bit pattern in turn."""

    def __init__(self, n, c, hw, two, seed, x1_bits=False):
        self.n, self.c, self.hw, self.m, self.two = n, c, hw, n * hw, two
        self.case = make_case(n, c, 1, hw, two, seed)
        if x1_bits:
            x1 = self.case["first"][:, :c]
            assert x1.numel() >= 1 << 16
            bits = (torch.arange(x1.numel(), device="cuda") % (1 << 16)).to(torch.int16)
            x1.copy_(bits.view(BF16).view(x1.shape))
            assert torch.equal(self.case["first"][:, :c].reshape(-1).view(torch.int16), bits)
        self.dy = output_grad(self.case, seed + 1)
        self.t = self.rows(self.case["t"])
        self.u = self.rows(self.case["first"]) if two else None
        self.x1 = None if two else self.case["first"][:, :c].reshape(n, c * hw)
        self.dy_rows = self.rows(self.dy)
        self.bns = [self.case["bn_t"]] + ([self.case["bn_u"]] if two else [])
        self._want = None

    def rows(self, t):
        return t.permute(0, 2, 3, 1).reshape(self.m, -1)

    def planes(self, y):
        """y (flat NCHW [n][2B][hw]) as [n][B][2][hw]: [..., 0, :] is the lead's, [..., 1, :] relu(bn_t(t))'s."""
        return y.view(self.n, self.c, 2, self.hw)

    def branch_rows(self, y, k):
        """Plane k of every channel of y as [m][B] rows."""
        return self.planes(y)[:, :, k].permute(0, 2, 1).reshape(self.m, self.c)

    def want(self):
        """Eager torch's training results, named as shuffle_train's outputs."""
        if self._want is None:
            w = eager_shuffle(self.case, self.dy)
            self._want = {"y": w["y"].reshape(-1)}
            for i in range(len(self.bns)):
                self._want.update({f"running_mean{i}": w[f"rm{i}"], f"running_var{i}": w[f"rv{i}"], f"nbt{i}": w[f"nbt{i}"],
                                   f"dx{i}": self.rows(w[f"dx{i}"]), f"dweight{i}": w[f"dw{i}"], f"dbias{i}": w[f"db{i}"]})
        return self._want


def x1_operand(ops, site, stride):
    """x1's planes at sample stride `stride` in one NaN-filled input, so a read between them shows in y."""
    n, c, hw = site.n, site.c, site.hw
    a = Arena((n - 1) * stride + c * hw, BF16, ops.place.get("x1", 0))
    a.t.view(torch.int16).fill_(-1)
    a.t.as_strided((n, c * hw), (stride, 1)).copy_(site.x1)
    ops.ins["x1"] = a
    return a.t


def shuffle_train(site, place=None, x1_stride=None, null_nbt=()):
    """b200c_bn_forward_shuffle then b200c_bn_backward_shuffle with every operand in an arena of its own (`place`:
    t, u, x1, y, dt, du, dy, mask_t, mask_u, f32 -> byte offset) and, for the batch norms named in `null_nbt` ("t",
    "u"), a null num_batches_tracked.  Checks the guards, inputs, scratch and launch count; returns the outputs (index 0
    is t's batch norm, 1 u's)."""
    lib, n, c, hw, m, two = N.load(), site.n, site.c, site.hw, site.m, site.two
    s = torch.cuda.current_stream().cuda_stream
    ops = Operands(place)
    t = ops.input("t", site.t)
    u = ops.input("u", site.u) if two else None
    stride = x1_stride or 2 * c * hw
    x1 = None if two else x1_operand(ops, site, stride)
    dy = ops.input("dy", site.dy_rows)
    mb = int(lib.b200c_bn_shuffle_mask_bytes(m, c))
    assert mb == m * -(-c // 8)
    out = {"y": ops.output("y", n * 2 * c * hw, BF16)}
    fwd, bwd = [], []
    for i, bn in enumerate(site.bns):
        name = "tu"[i]
        o = {f"mask{i}": ops.output(f"mask{i}", mb, torch.uint8, f"mask_{name}"),
             f"running_mean{i}": ops.output(f"running_mean{i}", c, F32, "f32", bn.running_mean),
             f"running_var{i}": ops.output(f"running_var{i}", c, F32, "f32", bn.running_var),
             f"nbt{i}": None if name in null_nbt else ops.output(f"nbt{i}", 1, torch.int64, None, bn.num_batches_tracked).view(()),
             f"mean{i}": ops.output(f"mean{i}", c, F32, "f32"), f"invstd{i}": ops.output(f"invstd{i}", c, F32, "f32"),
             f"dx{i}": ops.output(f"dx{i}", m * c, BF16, "d" + name).view(m, c),
             f"dweight{i}": ops.output(f"dweight{i}", c, F32, "f32"), f"dbias{i}": ops.output(f"dbias{i}", c, F32, "f32")}
        out.update(o)
        fwd.append((p(o[f"mask{i}"]), p(bn.weight), p(bn.bias), p(o[f"running_mean{i}"]), p(o[f"running_var{i}"]), p(o[f"nbt{i}"]),
                    p(o[f"mean{i}"]), p(o[f"invstd{i}"]), bn.momentum, bn.eps))
        x = (t, u)[i]
        bwd.append((p(x), p(o[f"mask{i}"]), p(o[f"dx{i}"]), p(bn.weight), p(o[f"mean{i}"]), p(o[f"invstd{i}"]), p(o[f"dweight{i}"]),
                    p(o[f"dbias{i}"])))
    ops.seal()
    buf, need = guarded_scratch(c, two)
    lead = (None, 0, p(u), *fwd[1]) if two else (p(x1), stride, None, *(None,) * 8, 0.0, 0.0)
    before = N.launch_count()
    N.check(lib.b200c_bn_forward_shuffle(*lead, p(t), *fwd[0], p(out["y"]), n, hw, c, p(buf), s))
    assert N.launch_count() - before == 2
    N.check(lib.b200c_bn_backward_shuffle(p(dy), *(bwd[1] if two else (None,) * 8), *bwd[0], m, c, p(buf), s))
    assert N.launch_count() - before == 4
    ops.check()
    check_scratch(buf, need)
    return out


def check_shuffle_against_references(site, got):
    """Everything torch computes against eager torch, the lead's planes of a stride-1 y against x1, the masks against
    their bit rule and the saved statistics against float64."""
    want = site.want()
    y, wy = site.planes(got["y"]), site.planes(want["y"])
    same(y[:, :, 1], wy[:, :, 1], "y's relu(bn_t(t)) planes")
    if site.two:
        same(y[:, :, 0], wy[:, :, 0], "y's relu(bn_u(u)) planes")
    else:
        same(y[:, :, 0], site.x1.view(site.n, site.c, site.hw), "y's x1 planes against x1")
    for k in want:
        if k != "y" and got[k] is not None:
            same(got[k], want[k], k)
    for i, x in enumerate((site.t, site.u)[:len(site.bns)]):
        check_shuffle_mask(got[f"mask{i}"], site.branch_rows(want["y"], 1 - i))
        check_stats_against_float64(x, {"mean": got[f"mean{i}"], "invstd": got[f"invstd{i}"]})


def shuffle_placements(two):
    ops = ("t", "u", "y", "dt", "du") if two else ("t", "x1", "y", "dt")
    v = [{op: off} for op in ops for off in (2, 6, 10)] + [{"dy": off} for off in (4, 12)]
    v += [{mask: off} for mask in (("mask_t", "mask_u") if two else ("mask_t",)) for off in (1, 3)]
    return v + [{"f32": 4}]


@gpu
@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
@pytest.mark.parametrize("n,c,hw", SHUFFLE_SHAPES)
def test_shuffle_training_matches_torch_at_every_placement(n, c, hw, two):
    site = ShuffleSite(n, c, hw, two, seed=n + c + hw)
    aligned = shuffle_train(site)
    check_shuffle_against_references(site, aligned)
    for place in shuffle_placements(two):
        assert_same_outputs(shuffle_train(site, place), aligned, f"{place} against the aligned call")


def shuffle_infer(site, dtype, place=None, x1_stride=None):
    """b200c_bn_infer_shuffle with the batch norms in eval mode with `dtype` parameters, every operand in an arena of
    its own; checks the guards, inputs and launch count.  Returns (y, the eval batch norms)."""
    lib, n, c, hw = N.load(), site.n, site.c, site.hw
    bns = [copy.deepcopy(bn).to(dtype).eval() for bn in site.bns]
    ops = Operands(place)
    t = ops.input("t", site.t)
    u = ops.input("u", site.u) if site.two else None
    stride = x1_stride or 2 * c * hw
    x1 = None if site.two else x1_operand(ops, site, stride)
    y = ops.output("y", n * 2 * c * hw, BF16)
    ops.seal()

    def params(bn):
        return p(bn.weight), p(bn.bias), p(bn.running_mean), p(bn.running_var)

    lead = (None, 0, p(u), *params(bns[1]), bns[1].eps) if site.two else (p(x1), stride, None, *(None,) * 4, 0.0)
    before = N.launch_count()
    N.check(lib.b200c_bn_infer_shuffle(*lead, p(t), *params(bns[0]), bns[0].eps, p(y), int(dtype == BF16), n, hw, c,
                                       torch.cuda.current_stream().cuda_stream))
    assert N.launch_count() - before == 1
    ops.check()
    return y, bns


def check_shuffle_eval(site, y, bns):
    """y against eager torch's eval modules, cat and channel_shuffle, and a stride-1 y's lead planes against x1."""
    with torch.no_grad():
        lead = F.relu(bns[1](site.case["first"])) if site.two else site.case["first"][:, :site.c]
        want = site.planes(channel_shuffle(torch.cat((lead, F.relu(bns[0](site.case["t"]))), 1), 2).reshape(-1))
    got = site.planes(y)
    same(got[:, :, 1], want[:, :, 1], "eval y's relu(bn_t(t)) planes")
    same(got[:, :, 0], want[:, :, 0] if site.two else site.x1.view(site.n, site.c, site.hw), "eval y's lead planes")


@gpu
@pytest.mark.parametrize("dtype", [F32, BF16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
def test_shuffle_eval_matches_torch(two, dtype):
    for n, c, hw in [(1, 1, 1), (1, 58, 1), (1, 33, 1)] + SHUFFLE_SHAPES:
        site = ShuffleSite(n, c, hw, two, seed=7 * n + c + hw)
        y, bns = shuffle_infer(site, dtype)
        check_shuffle_eval(site, y, bns)
        for place in ({"t": 6}, {"u" if two else "x1": 10}, {"y": 2}):
            same(shuffle_infer(site, dtype, place)[0], y, f"eval y at {(n, c, hw)} with {place} against the aligned call")


# x1 holds every bf16 bit pattern (n * B * hw >= 2^16), at three sample strides
X1_SHAPES = [(4, 100, 196), (41, 33, 49)]


@gpu
@pytest.mark.parametrize("n,c,hw", X1_SHAPES)
def test_shuffle_x1_strides_pass_every_bit_pattern_through(n, c, hw):
    site = ShuffleSite(n, c, hw, False, seed=11, x1_bits=True)
    for stride in (c * hw, 2 * c * hw, 2 * c * hw + 3):
        got = shuffle_train(site, x1_stride=stride)
        check_shuffle_against_references(site, got)
        for dtype in (F32, BF16):
            y, bns = shuffle_infer(site, dtype, x1_stride=stride)
            check_shuffle_eval(site, y, bns)


@gpu
@pytest.mark.parametrize("two", [False, True], ids=["one", "two"])
def test_shuffle_null_num_batches_tracked(two):
    site = ShuffleSite(8, 58, 49, two, seed=12)
    full = shuffle_train(site)
    check_shuffle_against_references(site, full)
    for name in ("tu" if two else "t"):
        got = shuffle_train(site, null_nbt=(name,))
        key = f"nbt{'tu'.index(name)}"
        assert got[key] is None
        assert_same_outputs({k: v for k, v in got.items() if k != key}, {k: v for k, v in full.items() if k != key},
                            f"null num_batches_tracked of {name}")


# ---- slice --------------------------------------------------------------------------------------------------------
# (ldy, c0, lddy, dc0) of a C-channel branch: y is out[:, c0:c0 + C] of an [m][ldy] output, dy dy_full[:, dc0:dc0 + C] of
# an [m][lddy] gradient
LAYOUTS = {"whole": lambda c: (c, 0, c, 0),                        # ldy == C, c0 = 0; lddy == C
           "last": lambda c: (c + 16, 16, c, 0),                   # the slice ends at ldy; lddy == C < ldy
           "middle_wider_dy": lambda c: (c + 32, 8, c + 64, 40),   # lddy > ldy
           "first_narrower_dy": lambda c: (2 * c + 8, 0, c + 8, 8)}   # lddy < ldy
SLICE_SHAPES = [s for s in BN_REGIME_SHAPES if s[1] % 8 == 0]
SLICE_CASES = [(s, layout) for i, s in enumerate(SLICE_SHAPES) for layout in (list(LAYOUTS)[i % len(LAYOUTS)],)]
SLICE_CASES += [(s, layout) for s in [(4, 64, 7, 7), (3, 24, 5, 5)] for layout in LAYOUTS]


def slice_train(x, dy_full, bn, ldy, c0, lddy, dc0, place=None):
    """b200c_bn_forward_slice into out[:, c0:c0 + C] (out filled with OUT_PATTERN) and b200c_bn_backward_slice from
    dy_full[:, dc0:dc0 + C], every operand in an arena of its own (`place`: mask, f32 -> byte offset); checks the
    guards, inputs, scratch and launch count.  Returns the outputs, out as [m][ldy]."""
    lib = N.load()
    m, c = x.shape
    s = torch.cuda.current_stream().cuda_stream
    ops = Operands(place)
    xa, dya = ops.input("x", x), ops.input("dy", dy_full)
    out = {"out": ops.output("out", m * ldy, BF16)}
    out["out"].view(torch.int16).fill_(OUT_PATTERN)
    out.update(mask=ops.output("mask", m * c // 8, torch.uint8),
               running_mean=ops.output("running_mean", c, F32, "f32", bn.running_mean),
               running_var=ops.output("running_var", c, F32, "f32", bn.running_var),
               nbt=ops.output("nbt", 1, torch.int64, None, bn.num_batches_tracked).view(()),
               mean=ops.output("mean", c, F32, "f32"), invstd=ops.output("invstd", c, F32, "f32"), dx=ops.output("dx", m * c, BF16).view(m, c),
               dweight=ops.output("dweight", c, F32, "f32"), dbias=ops.output("dbias", c, F32, "f32"))
    ops.seal()
    buf, need = guarded_scratch(c, False)
    o = {k: p(v) for k, v in out.items()}
    before = N.launch_count()
    N.check(lib.b200c_bn_forward_slice(p(xa), o["out"] + 2 * c0, ldy, o["mask"], p(bn.weight), p(bn.bias), o["running_mean"],
                                       o["running_var"], o["nbt"], o["mean"], o["invstd"], m, c, bn.momentum, bn.eps, p(buf), s))
    assert N.launch_count() - before == 2
    N.check(lib.b200c_bn_backward_slice(p(dya) + 2 * dc0, lddy, o["mask"], p(xa), o["dx"], p(bn.weight), o["mean"], o["invstd"],
                                        o["dweight"], o["dbias"], m, c, p(buf), s))
    assert N.launch_count() - before == 4
    ops.check()
    check_scratch(buf, need)
    out["out"] = out["out"].view(m, ldy)
    return out


def check_outside_slice(out, c0, c):
    outside = torch.cat([out[:, :c0], out[:, c0 + c:]], 1)
    assert (outside.view(torch.int16) == OUT_PATTERN).all(), "a write outside the slice"


@gpu
@pytest.mark.parametrize("shape,layout", SLICE_CASES, ids=[f"{n}x{c}x{h}x{w}-{lay}" for (n, c, h, w), lay in SLICE_CASES])
def test_slice_calls_match_torch(shape, layout):
    n, c, h, w = shape
    m = n * h * w
    ldy, c0, lddy, dc0 = LAYOUTS[layout](c)
    g = torch.Generator(device="cuda").manual_seed(m + c)
    x = (torch.randn(m, c, device="cuda", generator=g) * 2.0 + 0.5).to(BF16)
    dy_full = torch.randn(m, lddy, device="cuda", generator=g).to(BF16)
    bn = make_bn(c, c + 1)
    got = slice_train(x, dy_full, bn, ldy, c0, lddy, dc0)

    nchw = lambda t: t.view(n, h, w, c).permute(0, 3, 1, 2)  # noqa: E731
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(m, c)  # noqa: E731
    y_want, dx_want, want = eager_slice(nchw(x), bn, nchw(dy_full[:, dc0:dc0 + c].contiguous()))
    y_rows = rows(y_want)
    same(got["out"][:, c0:c0 + c], y_rows, "y")
    check_outside_slice(got["out"], c0, c)
    check_mask(got["mask"], y_rows)
    check_stats_against_float64(x, got)
    same(got["dx"], rows(dx_want), "dx")
    for k in want:
        same(got[k], want[k], k)
    for place in ({"mask": 1}, {"mask": 3}, {"f32": 4}):
        assert_same_outputs(slice_train(x, dy_full, bn, ldy, c0, lddy, dc0, place), got, f"{place} against the aligned call")

    lib = N.load()
    for dtype in (F32, BF16):
        ebn = copy.deepcopy(bn).to(dtype).eval()
        ops = Operands()
        xa = ops.input("x", x)
        out = ops.output("out", m * ldy, BF16).view(m, ldy)
        out.view(torch.int16).fill_(OUT_PATTERN)
        ops.seal()
        before = N.launch_count()
        N.check(lib.b200c_bn_infer_slice(p(xa), p(out) + 2 * c0, ldy, p(ebn.weight), p(ebn.bias), p(ebn.running_mean),
                                         p(ebn.running_var), int(dtype == BF16), ebn.eps, m, c, torch.cuda.current_stream().cuda_stream))
        assert N.launch_count() - before == 1
        ops.check()
        with torch.no_grad():
            same(out[:, c0:c0 + c], rows(F.relu(ebn(nchw(x)))), f"eval y ({dtype})")
        check_outside_slice(out, c0, c)
