"""Launch shapes of the sites that tests/test_gpu_fused_norm_paths.py runs for the vector statistics kernel."""
from gpu_common import BnLaunch, bn_launch_config

# (N, C, H, W) -> bn_launch_config(N*H*W, C), with C % 8 == 0 (the vector statistics kernel)
VECTOR_PATH_SHAPES = {
    (8, 64, 15, 15): BnLaunch(32, 16, 2, 8),     # merged grid; the last iteration covers rows 1,800..2,047 of M = 1,800
    (3, 64, 9, 9): BnLaunch(32, 16, 2, 1),       # collapsed grid; rows 243..255 of M = 243
    (8, 64, 28, 28): BnLaunch(32, 16, 2, 25),    # the momentum / eps site
}


def test_vector_path_shapes_reach_their_launch_regimes():
    for (n, c, h, w), want in VECTOR_PATH_SHAPES.items():
        m = n * h * w
        cfg = bn_launch_config(m, c)
        assert cfg == want, (n, c, h, w)
        assert c % 8 == 0 and cfg.block_x % 4 == 0
    for n, c, h, w in [(8, 64, 15, 15), (3, 64, 9, 9)]:
        m = n * h * w
        cfg = bn_launch_config(m, c)
        rows_per_pass = cfg.block_y * cfg.grid_y
        loop_count = 1 + (m - 1) // (rows_per_pass * 4)
        assert loop_count * 4 * rows_per_pass > m, (n, c, h, w)


def test_every_vector_channel_count_tiles_its_blocks():
    # C % 8 == 0 selects k_bn_stats<4>: every block.x is then a multiple of 4, so no thread's four channels straddle
    # C or a block
    for m in (2, 3, 17, 243, 1800, 10 ** 5, 3 * 10 ** 6):
        for c in range(8, 1 << 17, 8):
            if m * c < 2 ** 31:
                assert bn_launch_config(m, c).block_x % 4 == 0, (m, c)
