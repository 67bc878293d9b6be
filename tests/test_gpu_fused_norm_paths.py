"""Which statistics kernel a fused batch-norm site runs, and the sites only the vector statistics kernel reaches.

k_bn_stats<4> (four channels per thread) runs when C % 8 == 0 and x is on the 16-byte grid; k_bn_stats<1> runs
otherwise.  Both give eager torch's bits, so a silent fall-back to the scalar kernel would pass every bit
comparison: the kernel names in a torch.profiler trace show which one ran.  The bit comparisons here add what the
vector kernel meets nowhere else: rows past M inside a thread's last iteration (on a merged and on a collapsed
grid), non-finite channels crossing those rows, and the momentum / eps range at C % 8 == 0."""
import re

import pytest
import torch
import torch.nn as nn
from torch.profiler import ProfilerActivity, profile

from ant_ray_b200 import fused_norm
from gpu_common import bn_launch_config
from test_gpu_fused_norm import (NONFINITE, ONE_NAN, RESNET50_BN_SHAPES, check_site, edge_bn_setup, edge_site_inputs,
                                 make_bn, misaligned)

pytestmark = pytest.mark.gpu

CL = torch.channels_last
# (N, C, H, W): C % 8 == 0 with rows past M in the last iteration of the row loop
TAIL_ROW_SHAPES = [(8, 64, 15, 15), (3, 64, 9, 9)]


def reducing_kernels(n, c, h, w, misalign=()):
    """Names of the batch-norm reducing kernels that one fused forward and backward launch."""
    g = torch.Generator(device="cuda").manual_seed(n + c + h)
    x = torch.randn(n, c, h, w, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    dy = torch.randn(n, c, h, w, device="cuda", generator=g).to(torch.bfloat16).contiguous(memory_format=CL)
    x = (misaligned(x) if "x" in misalign else x).requires_grad_()
    dy = misaligned(dy) if "dy" in misalign else dy
    bn = make_bn(c, 0)
    # A forward and backward always launch reducing kernels (ours or torch's), so an empty set means the profiler
    # delivered the session without its kernel records, which happens now and then late in a long process: the
    # launches are the same on every attempt, so profile them again.
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fused_norm.bn_relu(bn, nn.ReLU(inplace=True), x).backward(dy)
            torch.cuda.synchronize()
        names = {e.key for e in prof.key_averages() if re.search(r"k_bn_stats|k_bn_bwd_reduce|batch_norm_(collect|backward_reduce)", e.key)}
        if names:
            break
    return names


def stats_widths(names):
    return {int(m.group(1)) for k in names for m in [re.search(r"k_bn_stats<(\d+)>", k)] if m}


@pytest.mark.parametrize("n", [256, 32])
def test_resnet50_shapes_run_the_vector_statistics_kernel(n):
    for c, h, w in RESNET50_BN_SHAPES:
        names = reducing_kernels(n, c, h, w)
        assert stats_widths(names) == {4}, (n, c, h, w, names)
        assert not any("batch_norm" in k for k in names), names
        assert any("k_bn_bwd_reduce" in k for k in names), names


@pytest.mark.parametrize("n,c,h,w,misalign", [(3, 100, 9, 9, ()), (64, 7, 32, 32, ()), (16, 36, 28, 28, ()),
                                              (8, 64, 16, 16, ("x",)), (4, 256, 7, 7, ("x",))])
def test_other_channel_counts_and_a_misaligned_input_run_the_scalar_statistics_kernel(n, c, h, w, misalign):
    assert stats_widths(reducing_kernels(n, c, h, w, misalign)) == {1}


def test_a_misaligned_gradient_keeps_the_vector_statistics_kernel():
    # dy is not an operand of the statistics kernel
    assert stats_widths(reducing_kernels(8, 64, 16, 16, ("dy",))) == {4}


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("n,c,h,w", TAIL_ROW_SHAPES)
def test_rows_past_m_on_the_vector_path(n, c, h, w, residual):
    m = n * h * w
    cfg = bn_launch_config(m, c)
    rows_per_pass = cfg.block_y * cfg.grid_y
    loop_count = 1 + (m - 1) // (rows_per_pass * 4)
    assert loop_count * 4 * rows_per_pass > m
    check_site(n, c, h, w, residual)


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("grad_edges", [False, True], ids=["input_edges", "gradient_edges"])
def test_value_edges_across_rows_past_m(grad_edges, residual):
    n, c, h, w = TAIL_ROW_SHAPES[0]
    inputs = edge_site_inputs(n, c, h, w, 11 + grad_edges, grad_edges)
    want, got = check_site(n, c, h, w, residual, inputs=inputs, bn_setup=edge_bn_setup(grad_edges))
    if not grad_edges:
        finite = [k for k in range(c) if k not in NONFINITE]
        for k in ("running_mean", "running_var", "dweight", "dbias"):
            assert torch.isfinite(got[k][finite]).all(), k
        assert torch.isnan(got["y"][:, ONE_NAN]).all()


@pytest.mark.parametrize("residual", [False, True], ids=["bn_relu", "bn_add_relu"])
@pytest.mark.parametrize("momentum,eps", [(0.0, 1e-5), (1.0, 1e-3), (1 / 3, 0.5)])
def test_hyperparameters_on_the_vector_path(momentum, eps, residual):
    check_site(8, 64, 28, 28, residual, momentum=momentum, eps=eps, nbt=2 ** 40)
