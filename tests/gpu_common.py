"""Shared helpers for the GPU parity tests: seeded inputs, dtype tables and the batch-norm launch shapes."""
from typing import NamedTuple

import torch

from ant_ray_b200 import _native as N

INT_DTYPES = [torch.int8, torch.uint8, torch.int32, torch.int64, torch.uint32, torch.uint64]
FLOAT_DTYPES = [torch.float16, torch.bfloat16, torch.float32, torch.float64]
NATIVE = {torch.int8: N.INT8, torch.uint8: N.UINT8, torch.int32: N.INT32, torch.int64: N.INT64,
          torch.uint32: N.UINT32, torch.uint64: N.UINT64,
          torch.float16: N.FLOAT16, torch.bfloat16: N.BFLOAT16, torch.float32: N.FLOAT32, torch.float64: N.FLOAT64}


def make_input(dtype, n, rank, op="sum"):
    """SURVEY.md 8(d): rank r draws from manual_seed(1234 + r); N(0,1) floats, bounded ints."""
    g = torch.Generator().manual_seed(1234 + rank)
    if dtype.is_floating_point:
        x = torch.randn(n, generator=g, dtype=torch.float32)
        if op == "prod":
            x = 1.0 + 0.1 * x  # keep W-fold products finite in half precision
        return x.to(dtype)
    info = torch.iinfo(dtype)
    lo, hi = max(info.min, -(2**15)), min(info.max, 2**15)
    if op == "prod":
        lo, hi = max(info.min, -3), min(info.max, 4)
    return torch.randint(lo, hi, (n,), generator=g, dtype=torch.int64).to(dtype)


def same_bits(a, b):
    """Whether two tensors (or two Nones) have the same dtype, shape and element bits, whatever their layout."""
    if a is None or b is None:
        return a is None and b is None
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits_of(a), bits_of(b))


def assert_equal_bits(a: torch.Tensor, b: torch.Tensor, what=""):
    """Bit-exact comparison (NaN-safe: compares the raw bytes)."""
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: {a.dtype}{tuple(a.shape)} vs {b.dtype}{tuple(b.shape)}"
    if not torch.equal(a.view(torch.uint8), b.view(torch.uint8)):
        diff = (a.double() - b.double()).abs()
        idx = int(diff.argmax())
        raise AssertionError(f"{what}: {int((diff > 0).sum())}/{a.numel()} elements differ; worst at {idx}: "
                             f"{a.flatten()[idx].item()} vs {b.flatten()[idx].item()}")


# ---- value edges ----------------------------------------------------------------------------------
_SIGNED = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def bits_of(t: torch.Tensor) -> torch.Tensor:
    """The raw bits of every element, as the signed integer type of the same width."""
    return t.contiguous().view(_SIGNED[t.element_size()])


def _from_bits(words, dtype):
    """Tensor of `dtype` whose elements have the given bit patterns (Python ints, taken mod 2^bits)."""
    bits = 8 * torch.empty((), dtype=dtype).element_size()
    signed = [(w + 2 ** (bits - 1)) % 2 ** bits - 2 ** (bits - 1) for w in words]
    return torch.tensor(signed, dtype=_SIGNED[bits // 8]).view(dtype)


def _int_range(dtype):
    bits = 8 * torch.empty((), dtype=dtype).element_size()
    signed = dtype in (torch.int8, torch.int16, torch.int32, torch.int64)
    lo = -(2 ** (bits - 1)) if signed else 0
    return bits, lo, lo + 2 ** bits - 1


# NaN bit patterns per float width: torch's NaN comes from float("nan"); a negative NaN and a quiet NaN with payload
_NANS = {torch.float16: (0xFE00, 0x7E55), torch.bfloat16: (0xFFC0, 0x7FC5),
         torch.float32: (0xFFC00000, 0x7FC12345), torch.float64: (0xFFF8000000000000, 0x7FF8000000012345)}


def edge_values(dtype) -> torch.Tensor:
    """A fixed pattern of the values where reductions go wrong, as a 1-D tensor of `dtype`.

    Integers: min, min+1, -1, 0, 1, 2, max-1, max, 2^(bits/2) +- 1 (whose squares wrap), and for 64-bit
    types 2^53+1 (not a double) and 2^62+3 (lost by a 32-bit or double path); duplicates removed.
    Floats: +-0, +-smallest and +-largest subnormal, +-smallest normal, +-1, 1+ulp, +-max, +-Inf, torch's
    NaN, a negative NaN and a NaN with a payload.  f16 / bf16 add the addend that puts 1 (and 1+ulp) on a
    rounding tie of the type in fp32 (ties to even: down, and up) and the addend that takes max to Inf.
    f32 adds the values the fused mean rounds to a 16-bit wire: bf16 / f16 ties both ways, 65519 (rounds
    to the f16 max), 65520 (the first value that rounds to f16 Inf), 70000 / 60000, 2^-25 (half the
    smallest f16 subnormal: a tie to 0), 3*2^-25 (a tie up to 2^-23), values in the f16 subnormal range
    and one below it."""
    if not dtype.is_floating_point:
        bits, lo, hi = _int_range(dtype)
        vals = [lo, lo + 1, -1, 0, 1, 2, hi - 1, hi, 2 ** (bits // 2) - 1, 2 ** (bits // 2) + 1]
        if bits == 64:
            vals += [2 ** 53 + 1, 2 ** 62 + 3]
        out = []
        for v in vals:
            v = (v - lo) % 2 ** bits + lo
            if v not in out:
                out.append(v)
        return torch.tensor(out, dtype=torch.int64).to(dtype) if bits < 64 else _from_bits(out, dtype)
    fi = torch.finfo(dtype)
    sub_min = fi.tiny * fi.eps
    vals = [0.0, -0.0, sub_min, -sub_min, fi.tiny - sub_min, -(fi.tiny - sub_min), fi.tiny, -fi.tiny,
            1.0, -1.0, 1.0 + fi.eps, fi.max, -fi.max, float("inf"), float("-inf"), float("nan")]
    if dtype in (torch.float16, torch.bfloat16):
        vals += [fi.eps / 2]                                   # 1 + eps/2: tie, down to 1; 1+eps + eps/2: tie, up
        vals += [16.0 if dtype == torch.float16 else 2.0 ** 119]   # max + half an ulp of max: a tie that rounds to Inf
    if dtype == torch.float32:
        vals += [1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -11, 1 + 3 * 2 ** -11, 65519.0, 65520.0, 70000.0, 60000.0,
                 2.0 ** -25, 3 * 2.0 ** -25, 3e-5, 1e-6, 1e-8]
    t = torch.tensor(vals, dtype=torch.float64 if dtype == torch.float64 else torch.float32).to(dtype)
    return torch.cat([t, _from_bits(list(_NANS[dtype]), dtype)])


def make_edge_inputs(dtype, n, W, seed):
    """Per-rank inputs of n elements, every element a value of edge_values(dtype).

    When n leaves room, the first elements are fixed blocks (P = pattern length):
      [P]   only rank 0 holds pattern value k, every other rank holds 1;
      [P]   only rank W-1 holds it;
      [P*P] ranks 0 and 1 hold every ordered pair of pattern values, the other ranks hold the SUM
            identity (-0.0, integer 0), so a pair's tie or overflow reaches the output at any W;
      [P*P] the same for ranks W-2 and W-1.
    The rest (all of it for smaller n) is drawn per rank and element from the pattern, seeded, so
    every 16-byte vector, every tail and every bulk-copy tile holds edge values."""
    # built on the raw bits (a signed integer type of the same width): torch's CPU kernels do not cover
    # indexing and filling of every dtype (uint32 / uint64)
    pat = bits_of(edge_values(dtype))
    P = pat.numel()
    g = torch.Generator().manual_seed(seed)
    ins = [pat[torch.randint(0, P, (n,), generator=g)] for _ in range(W)]
    if W >= 2 and n >= 2 * P + 2 * P * P:
        if dtype.is_floating_point:
            one, ident = bits_of(torch.tensor([1.0, -0.0], dtype=dtype))
        else:
            one, ident = bits_of(_from_bits([1, 0], dtype))
        k = torch.arange(P * P)
        first, second = pat[k // P], pat[k % P]
        for holder, start in ((0, 0), (W - 1, P)):
            for r in range(W):
                ins[r][start:start + P] = pat if r == holder else one
        for (ra, rb), start in (((0, 1), 2 * P), ((W - 2, W - 1), 2 * P + P * P)):
            for r in range(W):
                ins[r][start:start + P * P] = first if r == ra else (second if r == rb else ident)
        # every ordered pair of pattern values sits at ranks (0, 1) and at ranks (W-2, W-1)
        want = {(a, b) for a in pat.tolist() for b in pat.tolist()}
        end = 2 * P + 2 * P * P
        for ra, rb in ((0, 1), (W - 2, W - 1)):
            got = set(zip(ins[ra][:end].tolist(), ins[rb][:end].tolist()))
            assert want <= got, f"{dtype}: ranks ({ra}, {rb}) miss {len(want - got)} ordered pairs"
    return [t.view(dtype) for t in ins]


def assert_same_values(a: torch.Tensor, b: torch.Tensor, what=""):
    """Bit-exact, except that a position where both sides hold a NaN passes whatever the sign and payload
    (x86 and the GPU produce different NaN bits for the same invalid operation)."""
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, f"{what}: {a.dtype}{tuple(a.shape)} vs {b.dtype}{tuple(b.shape)}"
    a, b = a.flatten(), b.flatten()   # the first differing element is reported by its flat index
    same = bits_of(a) == bits_of(b)
    if a.dtype.is_floating_point:
        same |= torch.isnan(a) & torch.isnan(b)
    if not bool(same.all()):
        bad = (~same).nonzero().flatten()
        i = int(bad[0])
        ba, bb = int(bits_of(a)[i]), int(bits_of(b)[i])
        va, vb = (a[i].item(), b[i].item()) if a.dtype.is_floating_point else ("", "")
        raise AssertionError(f"{what}: {bad.numel()}/{a.numel()} elements differ; first at {i}: "
                             f"{va} (bits {ba:#x}) vs {vb} (bits {bb:#x})")


# ---- fused batch norm: launch shapes of the reducing kernels -------------------------------------------
# torch's MAX_BLOCK_SIZE, ELEMENTS_PER_THREAD, OPTIMAL_TILE_W and MAX_H_BLOCK (norm_kernels.cuh)
BN_MAX_BLOCK, BN_ELEMS_PER_THREAD, BN_TILE_W, BN_MAX_H_BLOCK = 512, 16, 32, 128
BN_MAX_CHANNELS = 1 << 17
BN_SEMAPHORES = BN_MAX_CHANNELS // BN_TILE_W   # the fixed semaphore region at the start of every scratch buffer


class BnLaunch(NamedTuple):
    block_x: int
    block_y: int
    grid_x: int
    grid_y: int   # 1 when the grid merge is collapsed (fewer than 8 rows of blocks)


def _last_pow2(n):
    for s in (1, 2, 4, 8, 16):
        n |= n >> s
    return max(1, n - (n >> 1))


def bn_launch_config(m, c):
    """Block and grid of the statistics and backward-reduce kernels for m rows of c channels: reduce_config in
    inst_norm.cu, which is torch's flexible_launch_configs with coop_flag set.  Each channel's rounding follows
    from this shape, so it is the map from shapes to the regimes the tests must reach."""
    block_x = min(_last_pow2(c), BN_TILE_W)
    block_y = min(_last_pow2(-(-m // BN_ELEMS_PER_THREAD)), BN_MAX_BLOCK // block_x)
    if block_x * block_y != BN_MAX_BLOCK:
        block_x = min(_last_pow2(c), BN_MAX_BLOCK // block_y)
    grid_y = min(-(-m // (block_y * BN_ELEMS_PER_THREAD)), BN_MAX_H_BLOCK)
    return BnLaunch(block_x, block_y, -(-c // block_x), grid_y if grid_y >= 8 else 1)


# (N, C, H, W) -> bn_launch_config(N*H*W, C): one site per launch regime of the reducing kernels.  A partial
# channel tile is C % block_x != 0 (its threads past C leave the backward reduce early); C % 8 != 0 takes the
# scalar elementwise kernels.
BN_REGIME_SHAPES = {
    (2, 256, 32, 32): BnLaunch(32, 16, 8, 8),          # the smallest merged grid
    (4, 100, 16, 16): BnLaunch(32, 16, 4, 1),          # 4 rows of blocks collapsed to 1, partial tile
    (8, 100, 28, 28): BnLaunch(32, 16, 4, 25),         # partial tile with the grid merge
    (64, 100, 28, 28): BnLaunch(32, 16, 4, 128),
    (2, 256, 3, 3): BnLaunch(256, 2, 1, 1),            # block.x widened past 32 by a small M
    (2, 2048, 5, 5): BnLaunch(128, 4, 16, 1),
    (2, 64, 1, 1): BnLaunch(64, 1, 1, 1),              # M = 2 and M = 3
    (3, 64, 1, 1): BnLaunch(64, 1, 1, 1),
    (64, 1, 32, 32): BnLaunch(1, 512, 1, 8),           # C = 1 (with stride(1) == 1: NHWC strides)
    (64, 3, 32, 32): BnLaunch(2, 256, 2, 16),          # C < 32, not a power of two: partial tiles, merged
    (64, 7, 32, 32): BnLaunch(4, 128, 2, 32),
    (64, 17, 32, 32): BnLaunch(16, 32, 2, 128),
    (64, 8, 32, 32): BnLaunch(8, 64, 1, 64),           # vector elementwise kernels
    (16, 24, 28, 28): BnLaunch(16, 32, 2, 25),         # vector, partial tile
    (16, 36, 28, 28): BnLaunch(32, 16, 2, 49),         # scalar elementwise kernels
    (8, 4104, 8, 8): BnLaunch(32, 16, 129, 1),         # one column past a power of two
    (2, 131072, 32, 32): BnLaunch(32, 16, 4096, 8),    # the most channels, merged: the last semaphore (512 MiB per tensor)
}
# The same regimes for a dual tail (two batch norms of one shape in one grid.z = 2 launch), whose plane 1 counts on the
# semaphores after plane 0's: at most half the channels.  The last entry is that limit on a merged grid, where plane 1
# uses semaphores 2048 .. 4095.
BN_DUAL_REGIME_SHAPES = {s: cfg for s, cfg in BN_REGIME_SHAPES.items() if s[1] != BN_MAX_CHANNELS}
BN_DUAL_REGIME_SHAPES[(2, BN_MAX_CHANNELS // 2, 32, 32)] = BnLaunch(32, 16, 2048, 8)
