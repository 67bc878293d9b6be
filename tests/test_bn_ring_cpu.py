"""The launch of the reducing kernels' rings (inst_norm.cu), restated: no GPU needed.

The statistics kernel's vector path (kStatsVec channels per hardware thread) and the backward reduce's (kBwdVec)
read rows through per-thread rings in dynamic shared memory.  Each launch keeps torch's logical block and grid
(gpu_common.bn_launch_config) and must stay within the 48 KB of shared memory a block gets without an opt-in
attribute, beside the kernel's static shared memory.  The backward ring has 3 stages of dy and x, or 2 stages where
it holds 3 or more operands.

The tables of tests/test_gpu_bn_ring.py and tests/test_gpu_sync_norm.py live here, with what they must cover: every
walk length at every channel count, on one row of blocks and on merged grids (ABI_RING_WALKS); every backward operand
set from 2 to 5 operands with its stage count (BWD_VARIANTS); each operand the launcher checks, moved off the 16-byte
grid alone, turning the ring off; and per-rank row counts whose walks differ between a world's ranks."""
import pytest

from gpu_common import BN_MAX_CHANNELS, bn_launch_config

# norm_kernels.cuh / inst_norm.cu
PARALLEL_LOADS, MAX_BLOCK = 4, 512
STATS_VEC, BWD_VEC, STATS_STAGES = 4, 4, 4
BLOCK_SMEM = 48 * 1024
STATS_STATIC, BWD_STATIC = 3 * MAX_BLOCK * 4 + 16, 2 * MAX_BLOCK * 4 + 16

# The channel counts of tests/test_gpu_bn_ring.py: hardware blocks of 2 to 128 threads, partial channel tiles (24, 40,
# 4104), the most channels of a dual site (65536) and of a local one (131072).
RING_CHANNELS = (8, 16, 24, 32, 40, 64, 256, 2048, 4104, 65536, 131072)
# The row walks every ring must survive: 1, D - 1, D, D + 1 and 2D + 1 iterations for D = 4, 3 and 2.
WALK_LENGTHS = (1, 2, 3, 4, 5, 7, 9)
# A merged grid (grid_y >= 8) walks at least 4 iterations: between 8 and 127 rows of blocks it walks exactly 4, and
# only the 128-row grid walks further, from M > 128 * 4 * block_y rows on.  Those longer merged walks run only where
# one operand stays within MERGED_WALK_ELEMENTS elements.
MERGED_WALKS = (4, 5, 7, 9)
MERGED_WALK_ELEMENTS = 1 << 29


def launch_rows(m, c):
    """Rows of one iteration of the row walk: kParallelLoads rows per thread, over every block row of the grid."""
    cfg = bn_launch_config(m, c)
    return PARALLEL_LOADS * cfg.block_y * cfg.grid_y


def walk(m, c):
    return 1 + (m - 1) // launch_rows(m, c)


def rows_for_walk(c, length, merged):
    """The fewest rows (at least 2) at C channels whose walk has `length` iterations, the last one partly past M, on
    one row of blocks or on a merged grid.  Past the 128-row grid's saturation the walk grows by one iteration per
    launch_rows, so those row counts are computed rather than searched."""
    full = launch_rows(1 << 24, c)
    if merged and length > 4:
        return (length - 1) * full + 1
    for m in range(2, 32 * full):
        if walk(m, c) == length and (bn_launch_config(m, c).grid_y > 1) == merged and m % launch_rows(m, c):
            return m
    raise AssertionError((c, length, merged))


def ring_walks():
    out = {}
    for c in RING_CHANNELS:
        for length in WALK_LENGTHS:
            out[(c, rows_for_walk(c, length, False))] = length
        for length in MERGED_WALKS:
            m = rows_for_walk(c, length, True)
            if length == 4 or m * c <= MERGED_WALK_ELEMENTS:
                out[(c, m)] = length
    return out


# (C, M) -> iterations of each thread's row walk: the shapes tests/test_gpu_bn_ring.py runs against eager torch's
# modules, and the wider sweep it runs through the C-ABI
RING_WALKS = {(64, 2): 1, (64, 5): 2, (64, 9): 3, (64, 13): 4, (64, 33): 5, (64, 97): 7, (64, 513): 9,
              (64, 5 * 8192 - 37): 5, (64, 7 * 8192 - 37): 7, (64, 9 * 8192 - 37): 9,
              (24, 9): 3, (24, 1025): 9, (4104, 13): 4, (4104, 97): 7}
ABI_RING_WALKS = ring_walks()

# The backward reduce's ring operands by C-ABI variant: which of y, dy2 and a downsample branch's x2 the ring holds
# besides dy and x, and whether the call writes g (which the launcher checks for the 16-byte grid too).
#   mask*: b200c_bn_backward_mask (the ReLU's bits), y: b200c_bn_backward, dy: b200c_bn_backward_res without noise
#   (g = dy), dual_*: b200c_bn_backward_dual from the bits or from y.
BWD_VARIANTS = {
    "mask": dict(src="mask", y=False, dy2=False, dual=False, g=False),
    "mask_g": dict(src="mask", y=False, dy2=False, dual=False, g=True),
    "mask_dy2": dict(src="mask", y=False, dy2=True, dual=False, g=False),
    "mask_dy2_g": dict(src="mask", y=False, dy2=True, dual=False, g=True),
    "y": dict(src="y", y=True, dy2=False, dual=False, g=False),
    "dy": dict(src="dy", y=False, dy2=False, dual=False, g=False),
    "dual_mask": dict(src="mask", y=False, dy2=False, dual=True, g=False),
    "dual_mask_dy2": dict(src="mask", y=False, dy2=True, dual=True, g=False),
    "dual_y": dict(src="y", y=True, dy2=False, dual=True, g=False),
    "dual_y_dy2": dict(src="y", y=True, dy2=True, dual=True, g=False),
}
# (operands, stages) of each variant's ring
BWD_RINGS = {"mask": (2, 3), "mask_g": (2, 3), "mask_dy2": (3, 2), "mask_dy2_g": (3, 2), "y": (3, 2), "dy": (2, 3),
             "dual_mask": (3, 2), "dual_mask_dy2": (4, 2), "dual_y": (4, 2), "dual_y_dy2": (5, 2)}


def launcher_operands(v):
    """The operands whose pointers bwd_reduce_launch hands to vec_ok for a variant, by name (inst_norm.cu: x, dy,
    dy2, y and g at a local site, x, dy, dy2, y and x_ds at a dual site; an absent one stands in as dy)."""
    names = ["x", "dy"] + ["dy2"] * v["dy2"] + ["y"] * v["y"]
    return names + (["x_ds"] if v["dual"] else ["g"] * v["g"])


# Per-rank row counts of tests/test_gpu_sync_norm.py's sync ring test at C = SYNC_RING_C (H = W = 1): an empty rank, a
# one-row rank and ranks of every walk length, on one row of blocks and on merged grids, dealt to the ranks of each
# world in turn so that a world's ranks walk different lengths.  Every split holds more than one row in all.
SYNC_RING_C = 64
SYNC_RING_ROWS = [0, rows_for_walk(SYNC_RING_C, 2, False), 1] + [rows_for_walk(SYNC_RING_C, n, False) for n in (1,) + WALK_LENGTHS[2:]] + \
    [rows_for_walk(SYNC_RING_C, n, True) for n in (4, 5)]


def sync_splits(world):
    rows = SYNC_RING_ROWS
    k = -(-len(rows) // world)
    return [[rows[(i * world + r) % len(rows)] for r in range(world)] for i in range(k)]


def bwd_stages(ops):
    """bwd_ring_stages: 3 stages for dy and x, 2 for 3 or more operands."""
    return 2 if ops >= 3 else 3


def stats_launch(m, c):
    """(hardware block threads, dynamic shared memory bytes) of the statistics kernel's vector path."""
    cfg = bn_launch_config(m, c)
    threads = cfg.block_x // STATS_VEC * cfg.block_y
    return threads, STATS_STAGES * PARALLEL_LOADS * threads * 2 * STATS_VEC


def bwd_launch(m, c, y, dy2, dual, g=False, off_grid=()):
    """(channels per hardware thread, hardware block threads, dynamic shared memory bytes) of a backward reduce
    whose operands named in `off_grid` lie off the 16-byte grid, the others on it: bwd_reduce_launch."""
    cfg = bn_launch_config(m, c)
    if c % 8 or set(off_grid) & set(launcher_operands(dict(y=y, dy2=dy2, dual=dual, g=g))):
        return 1, cfg.block_x * cfg.block_y, 0
    threads = cfg.block_x // BWD_VEC * cfg.block_y
    ops = 2 + dy2 + y + dual
    ring = bwd_stages(ops) * ops * PARALLEL_LOADS * threads * 2 * BWD_VEC
    if BWD_STATIC + ring > BLOCK_SMEM:
        return 1, cfg.block_x * cfg.block_y, 0
    return BWD_VEC, threads, ring


CHANNELS = sorted({c for k in range(3, 18) for c in (1 << k, 3 << (k - 1), (1 << k) + 8) if 8 <= c <= BN_MAX_CHANNELS})
ROWS = [2, 3, 13, 64, 100, 513, 2048, 12544, 50176, 200704, 802816, 3211264]


@pytest.mark.parametrize("c", CHANNELS)
def test_no_launch_asks_for_more_shared_memory_than_a_block_has(c):
    for m in ROWS:
        if m * c >= 1 << 31:
            continue
        cfg = bn_launch_config(m, c)
        assert cfg.block_x % 8 == 0   # C % 8 == 0 gives a power-of-two block.x >= 8: whole vectors per hardware thread
        threads, smem = stats_launch(m, c)
        assert threads * STATS_VEC == cfg.block_x * cfg.block_y and STATS_STATIC + smem <= BLOCK_SMEM
        for dual in (False, True):
            for y in (False, True):
                for dy2 in (False, True):
                    vec, threads, smem = bwd_launch(m, c, y, dy2, dual)
                    assert threads * vec == cfg.block_x * cfg.block_y
                    assert BWD_STATIC + smem <= BLOCK_SMEM


def test_every_site_with_aligned_operands_takes_the_ring():
    # dy and the mask bits (ReLU site), plus dy2 (tail), plus x2 (downsample tail), and the same reading y
    for c in (64, 128, 256, 512, 1024, 2048):
        for m in (12544, 50176, 200704, 802816, 3211264):
            for y in (False, True):
                for dy2 in (False, True):
                    for dual in (False, True):
                        vec, threads, smem = bwd_launch(m, c, y, dy2, dual)
                        assert vec == BWD_VEC and smem <= 40 * 1024, (m, c, y, dy2, dual)
    # a ReLU site's ring is 3 stages of 2 operands, a tail's 2 stages of 3: 24 KB per 512-thread block each
    assert bwd_launch(802816, 64, False, False, False)[2] == bwd_launch(802816, 256, False, True, False)[2] == 24 * 1024


def test_the_ring_shapes_walk_their_lengths():
    for (c, m), want in list(RING_WALKS.items()) + list(ABI_RING_WALKS.items()):
        assert walk(m, c) == want, (c, m)
        assert m % launch_rows(m, c), "the last iteration is partly past M"
    lengths = {walk(m, c) for c, m in RING_WALKS}
    for d in (STATS_STAGES, bwd_stages(2), bwd_stages(3)):
        assert {1, d - 1, d, d + 1, 2 * d + 1} - {0} <= lengths, d
    assert any(bn_launch_config(m, c).grid_y > 1 for c, m in RING_WALKS)
    assert any(c % bn_launch_config(m, c).block_x for c, m in RING_WALKS)   # a partial channel tile


def test_the_c_abi_sweep_walks_every_length_at_every_channel_count():
    for c in RING_CHANNELS:
        one_row = {n for (cc, m), n in ABI_RING_WALKS.items() if cc == c and bn_launch_config(m, c).grid_y == 1}
        merged = {n for (cc, m), n in ABI_RING_WALKS.items() if cc == c and bn_launch_config(m, c).grid_y > 1}
        assert one_row == set(WALK_LENGTHS) and 4 in merged, (c, one_row, merged)
    for d in (STATS_STAGES, bwd_stages(2), bwd_stages(3)):
        assert {1, d - 1, d, d + 1, 2 * d + 1} - {0} <= set(WALK_LENGTHS), d
    # every walk length a merged grid can have runs on one
    assert {n for (c, m), n in ABI_RING_WALKS.items() if bn_launch_config(m, c).grid_y > 1} == set(MERGED_WALKS)
    assert {c for c, m in ABI_RING_WALKS if c % bn_launch_config(m, c).block_x} == {24, 40, 4104}   # partial channel tiles
    threads = {bn_launch_config(m, c).block_x // BWD_VEC * bn_launch_config(m, c).block_y for c, m in ABI_RING_WALKS}
    assert min(threads) == 2 and max(threads) == 128


@pytest.mark.parametrize("c", [8, 24, 64, 4104])
def test_a_merged_grid_walks_at_least_four_iterations(c):
    # why walks of 1 to 3 iterations run on one row of blocks only: 8 .. 127 rows of blocks always walk 4
    for m in range(2, 4 * launch_rows(1 << 24, c)):
        if bn_launch_config(m, c).grid_y > 1:
            assert walk(m, c) >= 4, m
            if bn_launch_config(m, c).grid_y < 128:
                assert walk(m, c) == 4, m


def test_every_operand_count_takes_its_stage_count():
    m, c = 802816, 256
    threads = bn_launch_config(m, c).block_x // BWD_VEC * bn_launch_config(m, c).block_y
    for name, v in BWD_VARIANTS.items():
        ops = 2 + v["y"] + v["dy2"] + v["dual"]
        assert (ops, bwd_stages(ops)) == BWD_RINGS[name], name
        assert len(set(launcher_operands(v))) == ops + v["g"], name   # g is written, not copied through the ring
        assert bwd_launch(m, c, v["y"], v["dy2"], v["dual"], v["g"]) == (BWD_VEC, threads, bwd_stages(ops) * ops * PARALLEL_LOADS * threads * 2 * BWD_VEC)
    assert {ops for ops, _ in BWD_RINGS.values()} == {2, 3, 4, 5}
    # the 5-operand dual ring is the largest: 40 KB per 512-thread block
    assert bwd_launch(m, c, True, True, True)[2] == 40 * 1024


@pytest.mark.parametrize("name", list(BWD_VARIANTS))
def test_each_operand_off_the_grid_turns_the_ring_off(name):
    v = BWD_VARIANTS[name]
    for c, m in ABI_RING_WALKS:
        if c % 8 == 0 and bn_launch_config(m, c).grid_y > 1:
            cfg = bn_launch_config(m, c)
            for op in launcher_operands(v):
                assert bwd_launch(m, c, v["y"], v["dy2"], v["dual"], v["g"], off_grid=(op,)) == (1, cfg.block_x * cfg.block_y, 0), (op, c, m)
            # operands the reduce does not copy (the ReLU's bits, dx) leave the ring on
            assert bwd_launch(m, c, v["y"], v["dy2"], v["dual"], v["g"], off_grid=("mask", "dx"))[0] == BWD_VEC
    assert set(launcher_operands(v)) <= {"x", "x_ds", "dy", "dy2", "y", "g"}


@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_sync_splits_give_the_ranks_different_walks(world):
    splits = sync_splits(world)
    assert sorted({m for s in splits for m in s}) == sorted(set(SYNC_RING_ROWS))
    walks = set()
    for sizes in splits:
        assert len(sizes) == world and sum(sizes) > 1
        lengths = {walk(m, SYNC_RING_C) for m in sizes if m}
        assert len(lengths) > 1 or world == 2, sizes
        walks |= lengths
    assert walks == set(WALK_LENGTHS)
    assert 0 in SYNC_RING_ROWS and 1 in SYNC_RING_ROWS
    assert any(bn_launch_config(m, SYNC_RING_C).grid_y > 1 for m in SYNC_RING_ROWS if m)
