"""Pin the CPU oracle (oracle/) before anything is compared against it.

(a) The reference tests' known-answer values for this path (SURVEY.md section 4 / 8c):
    python/ray/util/collective/tests/single_node_cpu_tests/test_allreduce.py:13-128,
    test_allgather.py:14-38, test_reducescatter.py:14-36, test_broadcast.py:10-86, and the
    CPUCommunicator DAG test's fp16 fills (dag/tests/experimental/test_cpu_communicator_dag.py:105-134).
(b) Outputs of REAL gloo (the library the reference's CPU backend delegates to) on seeded inputs,
    committed as tests/golden/gloo_vectors.pt by tests/golden/make_golden.py.  Integers, min/max,
    data movement and every W=2 case must match bit for bit; W>2 floating-point sums/products may
    differ from gloo in association order only, so they are held to the north-star tolerance
    (1e-5 relative in fp32; half types one rounding step).
(c) The oracle's half-precision conversions against torch's.
(d) The oracle at value edges (tests/gpu_common.py::make_edge_inputs: NaN, +-Inf, +-0, subnormals,
    overflow, rounding ties, integer wrap-around and high words) against a restatement written here:
    Python integers modulo 2^bits, and for floats a rank-order fold with torch CPU ops in fp32 (fp64
    for f64) whose MIN / MAX spell out the `a > b ? a : b` rule.
"""
import os

import pytest
import torch

from gpu_common import FLOAT_DTYPES, INT_DTYPES, _from_bits, _int_range, assert_same_values, bits_of, make_edge_inputs, make_input

from oracle import oracle as O

GOLD = torch.load(os.path.join(os.path.dirname(__file__), "golden", "gloo_vectors.pt"))
OPS = {"sum": O.SUM, "prod": O.PROD, "min": O.MIN, "max": O.MAX}
DT = {str(d): d for d in (torch.int8, torch.uint8, torch.int32, torch.int64, torch.float16, torch.bfloat16, torch.float32, torch.float64)}


# ---- (a) known-answer values of the reference tests -------------------------------------------
@pytest.mark.parametrize("n", [2, 2**5, 2**10, 2**15, 2**20])
def test_allreduce_ones(n):
    out = O.allreduce([torch.ones(n), torch.ones(n)])
    assert (out == 2).all()


def test_allreduce_chain_of_groups():
    x = [torch.ones(10), torch.ones(10)]
    for i in range(5):
        s = O.allreduce(x)
        x = [s.clone(), s.clone()]
        assert (s == 2 ** (i + 1)).all()


@pytest.mark.parametrize("op,val", [(O.PROD, 6), (O.MIN, 2), (O.MAX, 3)])
def test_allreduce_ops_fill(op, val):
    out = O.allreduce([torch.ones(10) * 2, torch.ones(10) * 3], op)
    assert (out == val).all()


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float16, torch.float32, torch.float64])
def test_allreduce_dtypes_fill(dtype):
    assert (O.allreduce([torch.ones(10, dtype=dtype)] * 2) == 2).all()


def test_allgather_reducescatter_broadcast_fill():
    got = O.allgather([torch.ones(5, 5, 5) * (j + 1) for j in range(2)])
    for j in range(2):
        assert (got[j] == j + 1).all()
    rs = O.reducescatter([[torch.ones(10) for _ in range(2)] for _ in range(2)])
    assert all((t == 2).all() for t in rs)
    for src in (0, 1):
        assert (O.broadcast([torch.ones(10) * 2, torch.ones(10) * 3], src) == src + 2).all()


def test_cpu_communicator_fp16_fills():
    # test_cpu_communicator_dag.py:105-134: W=2, value i + idx, shape (10*i,), fp16, exact sum
    for i in range(1, 4):
        ins = [torch.full((10 * i,), float(i + idx), dtype=torch.float16) for idx in range(2)]
        assert (O.allreduce(ins) == 2 * i + 1).all()
    ins = [torch.full((8,), float(v), dtype=torch.float16) for v in (1, 2, 4)]
    assert (O.allreduce(ins, O.AVG) == (ins[0].float() + ins[1].float() + ins[2].float()).div(3).half()).all()


# ---- (b) real gloo on seeded inputs ---------------------------------------------------------------
def _tol(dtype):
    return {torch.float32: 1e-5, torch.float64: 1e-12, torch.float16: 2e-3, torch.bfloat16: 1.6e-2}[dtype]


@pytest.mark.parametrize("world", sorted(GOLD["cases"]))
def test_oracle_matches_gloo(world):
    n = GOLD["n"]
    per_rank = GOLD["cases"][world]
    checked = 0
    for (kind, dts, opn), want0 in per_rank[0].items():
        if kind.startswith("ddp_"):
            continue
        dt = DT[dts]
        if kind in ("allreduce", "reduce"):
            ins = [make_input(dt, n, r, opn) for r in range(world)]
            got = O.allreduce(ins, OPS[opn])
            holder = 0 if kind == "allreduce" else world - 1
            want = per_rank[holder][(kind, dts, opn)]
            exact = (not dt.is_floating_point) or opn in ("min", "max") or world == 2
            if exact:
                assert torch.equal(got, want), f"{kind} {dts} {opn} W={world}"
            else:
                assert torch.allclose(got.double(), want.double(), rtol=_tol(dt), atol=_tol(dt)), f"{kind} {dts} {opn} W={world}"
            if kind == "reduce":  # non-root ranks keep their input (torch_gloo_collective_group.py:170-179)
                assert torch.equal(per_rank[0][(kind, dts, opn)], make_input(dt, n, 0, opn))
        elif kind == "reducescatter":
            lists = [[make_input(dt, n, r * 16 + j) for j in range(world)] for r in range(world)]
            got = O.reducescatter(lists)
            for r in range(world):
                want = per_rank[r][(kind, dts, opn)]
                if not dt.is_floating_point or world == 2:
                    assert torch.equal(got[r], want)
                else:
                    assert torch.allclose(got[r].double(), want.double(), rtol=_tol(dt), atol=_tol(dt))
        elif kind == "allgather":
            got = torch.stack(O.allgather([make_input(dt, n, r) for r in range(world)]))
            for r in range(world):
                assert torch.equal(got, per_rank[r][(kind, dts, opn)])
        elif kind == "broadcast":
            got = O.broadcast([make_input(dt, n, r) for r in range(world)], 1)
            for r in range(world):
                assert torch.equal(got, per_rank[r][(kind, dts, opn)])
        checked += 1
    assert checked >= 50


@pytest.mark.parametrize("world", sorted(GOLD["cases"]))
def test_fused_gradient_mean_vs_torch_hooks(world):
    """The fused reduction computes the same mean as torch's DDP hooks, with one rounding fewer:
    fp32 wire vs default hook (div_(W) then SUM) within 1e-5; bf16 wire vs bf16_compress_hook
    (which also ROUNDS THE SUM in bf16 at every gloo step) within bf16 resolution."""
    ins = [make_input(torch.float32, 1000, r) for r in range(world)]
    want = GOLD["cases"][world][0][("ddp_default_hook", "torch.float32", "")]
    got = O.allreduce_scaled(ins, None, 1.0 / world)
    assert torch.allclose(got, want, rtol=1e-5, atol=1e-6)
    want16 = GOLD["cases"][world][0][("ddp_bf16_compress_hook", "torch.float32", "")]
    got16 = O.allreduce_scaled(ins, torch.bfloat16, 1.0 / world)
    assert torch.allclose(got16, want16, rtol=2e-2, atol=2e-2)
    # and the fused result is at least as close to the exact mean as the compress hook's
    exact = torch.stack(ins).double().mean(0)
    assert (got16.double() - exact).abs().mean() <= (want16.double() - exact).abs().mean() * 1.05


# ---- (c) conversions ------------------------------------------------------------------------------
def test_half_conversions_match_torch():
    lib = O.lib()
    g = torch.Generator().manual_seed(0)
    vals = torch.cat([torch.randn(4000, generator=g) * s for s in (1e-8, 1e-5, 1e-3, 1.0, 1e3, 7e4, 1e38)] +
                     [torch.tensor([0.0, -0.0, float("inf"), -float("inf"), 65504.0, 65520.0, 65519.9, 5.96e-8, 2.98e-8, 2.9802322e-8])])
    for v in vals.tolist():
        t = torch.tensor(v, dtype=torch.float32)
        assert lib.oracle_float_to_bf16(v) == (t.bfloat16().view(torch.int16).item() & 0xFFFF), v
        assert lib.oracle_float_to_f16(v) == (t.half().view(torch.int16).item() & 0xFFFF), v
    for bits in list(range(0, 65536, 7)) + [0x7C00, 0xFC00, 0x0001, 0x03FF, 0x0400]:
        h = torch.tensor(bits - 65536 if bits >= 32768 else bits, dtype=torch.int16)
        f16, bf = h.view(torch.float16).float().item(), h.view(torch.bfloat16).float().item()
        got16, gotbf = lib.oracle_f16_to_float(bits), lib.oracle_bf16_to_float(bits)
        assert (got16 == f16) or (got16 != got16 and f16 != f16)
        assert (gotbf == bf) or (gotbf != gotbf and bf != bf)


def test_integer_wraparound_and_avg():
    a = torch.tensor([127, -128, 100], dtype=torch.int8)
    b = torch.tensor([1, -1, 100], dtype=torch.int8)
    assert O.allreduce([a, b]).tolist() == [-128, 127, -56]
    assert O.allreduce([a, b], O.PROD).tolist() == [127, -128, 16]
    assert O.allreduce([torch.tensor([7, -7], dtype=torch.int32)] * 3, O.AVG).tolist() == [7, -7]
    assert O.allreduce([torch.tensor([1.0]), torch.tensor([2.0]), torch.tensor([4.0])], O.AVG).item() == pytest.approx(7 / 3, rel=1e-6)


# ---- (d) value edges ------------------------------------------------------------------------------
EDGE_N = 2 * 31 + 2 * 31 * 31 + 101   # the fixed blocks of the longest pattern (f32, 31 values) and a random tail


def _ints_of(t):
    bits, lo, _ = _int_range(t.dtype)
    return [(v - lo) % 2 ** bits + lo for v in bits_of(t).tolist()]


def _restate_int(ins, op):
    bits, lo, _ = _int_range(ins[0].dtype)
    cols = list(zip(*[_ints_of(t) for t in ins]))
    wrap = lambda v: (v - lo) % 2 ** bits + lo  # noqa: E731
    out = []
    for col in cols:
        acc = col[0]
        for x in col[1:]:
            if op in (O.SUM, O.AVG):
                acc = wrap(acc + x)
            elif op == O.PROD:
                acc = wrap(acc * x)
            elif op == O.MAX:
                acc = acc if acc > x else x
            else:
                acc = acc if acc < x else x
        if op == O.AVG:  # the wrapped sum, divided with truncation toward zero
            acc = abs(acc) // len(cols[0]) * (1 if acc >= 0 else -1)
        out.append(acc)
    return _from_bits(out, ins[0].dtype)


def _restate_float(ins, op, wire=None, scale=None):
    dt = ins[0].dtype
    acc_t = torch.float64 if dt == torch.float64 else torch.float32
    xs = [t.to(acc_t) if wire is None else t.to(wire).to(acc_t) for t in ins]
    acc = xs[0]
    for x in xs[1:]:
        if op in (O.SUM, O.AVG):
            acc = acc + x
        elif op == O.PROD:
            acc = acc * x
        elif op == O.MAX:
            acc = torch.where(acc > x, acc, x)
        else:
            acc = torch.where(acc < x, acc, x)
    if op == O.AVG and dt == torch.float64:
        acc = acc / len(ins)
    elif op == O.AVG or scale is not None:
        acc = acc * torch.tensor(1.0 / len(ins) if scale is None else scale, dtype=torch.float32)
    if wire is not None:
        acc = acc.to(wire).to(acc_t)
    return acc.to(dt)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("dtype", INT_DTYPES + FLOAT_DTYPES, ids=str)
def test_oracle_at_value_edges(dtype, world):
    ins = make_edge_inputs(dtype, EDGE_N, world, seed=world)
    for name, op in (("sum", O.SUM), ("prod", O.PROD), ("max", O.MAX), ("min", O.MIN), ("avg", O.AVG)):
        want = _restate_int(ins, op) if not dtype.is_floating_point else _restate_float(ins, op)
        assert_same_values(O.allreduce(ins, op), want, f"{dtype} {name} W={world}")


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_oracle_fused_mean_at_value_edges(world):
    """Wire rounding of every contribution, fp32 sum, the scale, then ONE rounding to the wire."""
    ins = make_edge_inputs(torch.float32, EDGE_N, world, seed=100 + world)
    for wire in (None, torch.bfloat16, torch.float16):
        assert_same_values(O.allreduce_scaled(ins, wire, 1.0 / world), _restate_float(ins, O.SUM, wire, 1.0 / world),
                           f"fused mean wire={wire} W={world}")
    for dt in (torch.bfloat16, torch.float16):
        ins = make_edge_inputs(dt, EDGE_N, world, seed=200 + world)
        assert_same_values(O.allreduce_scaled(ins, None, 1.0 / 3), _restate_float(ins, O.SUM, None, 1.0 / 3), f"{dt} scaled W={world}")


def test_oracle_edge_table():
    """Single cases that decide the documented semantics (include/b200coll.h, b200c_redop_t)."""
    nan, inf = float("nan"), float("inf")
    f = lambda *v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    assert O.allreduce([f(nan), f(1.0)], O.MAX).item() == 1.0                   # a NaN in the fold is replaced ...
    assert O.allreduce([f(1.0), f(nan)], O.MAX).isnan().all()                  # ... a NaN at the next rank is taken
    assert bits_of(O.allreduce([f(0.0), f(-0.0)], O.MAX)).item() == bits_of(f(-0.0)).item()
    assert bits_of(O.allreduce([f(-0.0), f(0.0)], O.MAX)).item() == 0
    assert bits_of(O.allreduce([f(-0.0), f(-0.0)])).item() == bits_of(f(-0.0)).item()   # no +0 start value
    assert O.allreduce([f(inf), f(-inf)]).isnan().all()
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32)  # noqa: E731
    assert O.allreduce([i32(2**31 - 1), i32(1)], O.AVG).item() == -(2**30)     # wrapped sum, truncating divide
    assert O.allreduce([i32(-3), i32(0)], O.AVG).item() == -1
    # fused mean, f16 wire, W = 2, scale 0.5: the contribution overflows before the scale, the sum does not
    got = O.allreduce_scaled([f(70000.0, 60000.0, 1e-8, 3e-5), f(0.0, 60000.0, 0.0, 3e-5)], torch.float16, 0.5)
    assert got[0].item() == inf and got[1].item() == 60000.0 and got[2].item() == 0.0
    assert got[3].item() == torch.tensor(3e-5).half().float().item()
    u64 = torch.tensor([-1], dtype=torch.int64).view(torch.uint64)              # 2^64 - 1
    two = torch.tensor([2], dtype=torch.int64).view(torch.uint64)
    assert bits_of(O.allreduce([u64, two], O.AVG)).item() == 0                  # (2^64 - 1 + 2) mod 2^64 = 1, / 2 = 0
    assert bits_of(O.allreduce([u64, u64], O.AVG)).item() == 2**63 - 1         # unsigned: (2^64 - 2) / 2
