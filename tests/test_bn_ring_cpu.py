"""The launch of the reducing kernels' rings (inst_norm.cu), restated: no GPU needed.

The statistics kernel's vector path (kStatsVec channels per hardware thread) and the backward reduce's (kBwdVec)
read rows through per-thread rings in dynamic shared memory.  Each launch keeps torch's logical block and grid
(gpu_common.bn_launch_config) and must stay within the 48 KB of shared memory a block gets without an opt-in
attribute, beside the kernel's static shared memory.  The backward ring has 3 stages of dy and x, or 2 stages where
it holds 3 or more operands."""
import pytest

from gpu_common import BN_MAX_CHANNELS, bn_launch_config

# norm_kernels.cuh / inst_norm.cu
PARALLEL_LOADS, MAX_BLOCK = 4, 512
STATS_VEC, BWD_VEC, STATS_STAGES = 4, 4, 4
BLOCK_SMEM = 48 * 1024
STATS_STATIC, BWD_STATIC = 3 * MAX_BLOCK * 4 + 16, 2 * MAX_BLOCK * 4 + 16

# (C, M) -> iterations of each thread's row walk, the shapes of tests/test_gpu_bn_ring.py
RING_WALKS = {(64, 2): 1, (64, 5): 2, (64, 9): 3, (64, 13): 4, (64, 33): 5, (64, 97): 7, (64, 513): 9,
              (64, 5 * 8192 - 37): 5, (64, 7 * 8192 - 37): 7, (64, 9 * 8192 - 37): 9,
              (24, 9): 3, (24, 1025): 9, (4104, 13): 4, (4104, 97): 7}


def bwd_stages(ops):
    """bwd_ring_stages: 3 stages for dy and x, 2 for 3 or more operands."""
    return 2 if ops >= 3 else 3


def stats_launch(m, c):
    """(hardware block threads, dynamic shared memory bytes) of the statistics kernel's vector path."""
    cfg = bn_launch_config(m, c)
    threads = cfg.block_x // STATS_VEC * cfg.block_y
    return threads, STATS_STAGES * PARALLEL_LOADS * threads * 2 * STATS_VEC


def bwd_launch(m, c, y, dy2, dual):
    """(channels per hardware thread, hardware block threads, dynamic shared memory bytes) of a backward reduce
    whose operands are all on the 16-byte grid: bwd_reduce_launch."""
    cfg = bn_launch_config(m, c)
    if c % 8:
        return 1, cfg.block_x * cfg.block_y, 0
    threads = cfg.block_x // BWD_VEC * cfg.block_y
    ops = 2 + dy2 + y + dual
    ring = bwd_stages(ops) * ops * PARALLEL_LOADS * threads * 2 * BWD_VEC
    if BWD_STATIC + ring > BLOCK_SMEM:
        return 1, cfg.block_x * cfg.block_y, 0
    return BWD_VEC, threads, ring


def walk(m, c):
    cfg = bn_launch_config(m, c)
    return 1 + (m - 1) // (cfg.block_y * cfg.grid_y * PARALLEL_LOADS)


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
    for (c, m), want in RING_WALKS.items():
        assert walk(m, c) == want, (c, m)
        cfg = bn_launch_config(m, c)
        assert m % (cfg.block_y * cfg.grid_y * PARALLEL_LOADS), "the last iteration is partly past M"
    lengths = {walk(m, c) for c, m in RING_WALKS}
    for d in (STATS_STAGES, bwd_stages(2), bwd_stages(3)):
        assert {1, d - 1, d, d + 1, 2 * d + 1} - {0} <= lengths, d
    assert any(bn_launch_config(m, c).grid_y > 1 for c, m in RING_WALKS)
    assert any(c % bn_launch_config(m, c).block_x for c, m in RING_WALKS)   # a partial channel tile
