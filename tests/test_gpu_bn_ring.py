"""The vector paths' row rings (norm_kernels.cuh) against eager torch, bit for bit.

k_bn_stats<4>, k_bn_stats_dual<4> and the vector path of k_bn_bwd_reduce (kBwdVec channels per hardware thread)
read their rows through per-thread cp.async rings of kStatsStages or bwd_ring_stages(dual) iterations.  Each case
runs a row walk of 1, D - 1, D, D + 1 and 2D + 1 iterations for every ring depth D, with the last iteration partly
past M, through every ring kernel: the statistics, the dual statistics, and the reduce from the ReLU bits, from y,
from dy (no ReLU), for a tail with dy2 that writes g, and for a downsample tail (dual, from the bits and from y).
tests/test_bn_ring_cpu.py checks that these shapes walk those lengths."""
import copy

import pytest
import torch
import torch.nn as nn

import test_gpu_fused_dual as D
import test_gpu_fused_norm as L
import test_gpu_fused_res as R
from ant_ray_b200 import fused_norm
from gpu_common import same_bits
from test_bn_ring_cpu import RING_WALKS

pytestmark = pytest.mark.gpu

# M = 2 .. 513 keep one row of blocks, the others merge a grid of 128 rows of blocks.  C = 24 has a 16-wide tile
# with 8 channels past C, C = 4104 8 valid channels in its last tile.
SHAPES = [(m, c, 1, 1) for c, m in RING_WALKS]


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
@pytest.mark.parametrize("residual", [False, True], ids=["relu_bits", "tail_g"])
def test_stats_and_reduce_from_the_mask(n, c, h, w, residual):
    L.check_site(n, c, h, w, residual)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_reduce_from_y(n, c, h, w):
    L.check_native_site(n * h * w, c, c + n)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_reduce_from_dy(n, c, h, w):
    R.check_gauss_site("plain", n, c, h, w)


@pytest.mark.parametrize("n,c,h,w", SHAPES)
def test_tail_with_two_gradients_writes_g(n, c, h, w):
    g = torch.Generator(device="cuda").manual_seed(n + c)
    t = lambda s, o: nhwc((torch.randn(n, c, h, w, device="cuda", generator=g) * s + o).to(torch.bfloat16))  # noqa: E731
    x, identity, dy, dy2 = t(2.0, 0.5), t(1.0, -0.2), t(1.0, 0.0), t(1.0, 0.0)
    bn = L.make_bn(c, 4)

    def run(fused):
        b = copy.deepcopy(bn)
        xg, ig = x.clone().requires_grad_(), identity.clone().requires_grad_()
        relu = nn.ReLU(inplace=True)
        if fused:
            ys = fused_norm.bn_add_relu(b, relu, xg, ig, pair=True)
        else:
            out = b(xg)
            out += ig
            y = relu(out)
            ys = (y, y)
        torch.autograd.backward([ys[0], ys[1]], [dy, dy2])
        return [ys[0].detach(), xg.grad, ig.grad, b.weight.grad, b.bias.grad, b.running_mean, b.running_var]

    want, got = run(False), run(True)
    bad = [i for i, (a, b) in enumerate(zip(got, want)) if not same_bits(a, b)]
    assert not bad, bad


@pytest.mark.parametrize("n,c,h,w", SHAPES)
@pytest.mark.parametrize("mode", ["one", "pair"])
def test_dual_stats_and_reduce(n, c, h, w, mode):
    x3, x_ds, dy1, dy2 = D.inputs(n, c, h, w, c + n)
    D.check_dual(x3, x_ds, dy1, dy2, mode, L.make_bn(c, 1), L.make_bn(c, 2))


@pytest.mark.parametrize("n,c,h,w", [s for s in SHAPES if s[1] <= 2048])
def test_dual_reduce_from_y(n, c, h, w):
    D.check_dual_through_the_c_abi(n, c, h, w)
