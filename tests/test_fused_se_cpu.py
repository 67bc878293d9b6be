"""The squeeze-and-excitation sites without a GPU: fuse_model swaps torchvision's SqueezeExcitation only inside the
inverted-residual blocks it swaps and keeps the model, the fused module computes its parent's bits where nothing is
fused (CPU, NCHW, fp32), the C-ABI calls reject bad arguments before any launch, and `se_reduce_config` restates the
launch torch's reduce kernel takes for the mean / sum over (H, W) of a channels-last tensor, with one named shape per
branch (SE_REGIME_SHAPES, which test_gpu_fused_se.py runs)."""
import copy
import ctypes
import os
import subprocess
import sys
from typing import NamedTuple

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

torchvision = pytest.importorskip("torchvision")
from torchvision.models import efficientnet, mobilenetv3  # noqa: E402
from torchvision.ops.misc import SqueezeExcitation  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = {"efficientnet_b0": 16, "mobilenet_v3_large": 8, "efficientnet_v2_s": 30}   # SE modules per model
# an H100 SXM: multiProcessorCount and maxThreadsPerMultiProcessor
H100 = (132, 2048)
SEMAPHORES = 4096   # se_kernels.cuh's kSemaphores


class SeLaunch(NamedTuple):
    vec: int          # output_vec_size: channels per thread
    block_x: int
    block_y: int
    split: bool       # the rows are split across threadIdx.y (block_y_reduce)
    ctas: int         # ctas_per_output: blocks per output along grid.y (global_reduce when > 1)
    grid_x: int


def _last_pow2(n):
    for s in (1, 2, 4, 8, 16, 32):
        n |= n >> s
    return max(1, n - (n >> 1))


def _div_up(a, b):
    return -(-a // b)


def se_reduce_config(n, c, hw, addr=0, num_mp=H100[0], max_tpm=H100[1]):
    """torch's setReduceConfig<float, bf16, vt0 = 4> (Reduce.cuh) for x.mean((-1, -2)) or the keepdim sum over (H, W) of
    a channels-last bf16 [n, c, H, W] at address `addr`, c > 1 and hw > 1: C is the fastest output dimension and
    H * W one reduced dimension of stride C, the "vectorize along output" case.  inst_se.cu's reduce_config."""
    vec = 4
    while (addr // 2) % vec or c % vec:   # get_output_vec_size: the element address, C and the strides C and HW * C
        vec //= 2
    dim0, dim1 = n * c // vec, hw
    mnt = 512 // vec
    d0 = _last_pow2(dim0) if dim0 < mnt else mnt
    d1 = _last_pow2(dim1) if dim1 < mnt else mnt
    bw = min(d0, 32)
    bh = min(d1, mnt // bw)
    bw = min(d0, mnt // bh)
    split = hw >= min(bh * 16, 256)
    step_output, step_input = (bw, bh) if split else (bw * bh, 1)
    grid_x = _div_up(dim0, step_output)
    target = num_mp * (max_tpm // (bw * bh))
    vpt, ctas = _div_up(hw, step_input), 1
    if split and vpt >= 256 and grid_x <= target:
        ctas = max(min(_div_up(target, grid_x), _div_up(vpt, 16)), _div_up(vpt, 256))
    return SeLaunch(vec, bw, bh, split, ctas, grid_x)


# ((N, C, H, W), x's address mod 16) -> the launch on an H100: one shape per branch of se_reduce_config.  The backward
# reduce always takes the aligned launch (torch reduces a fresh product tensor).
SE_REGIME_SHAPES = {
    ((2, 64, 7, 7), 0): SeLaunch(4, 32, 4, False, 1, 1),          # vec 4, each warp its own outputs
    ((1, 1152, 7, 7), 0): SeLaunch(4, 32, 4, False, 1, 3),
    ((4, 100, 16, 16), 0): SeLaunch(4, 32, 4, True, 1, 4),        # rows split across warps, C = 100
    ((4, 100, 56, 56), 0): SeLaunch(4, 32, 4, True, 49, 4),       # ... and across blocks
    ((2, 64, 32, 32), 0): SeLaunch(4, 32, 4, True, 16, 1),
    ((1, 32, 224, 224), 0): SeLaunch(4, 8, 16, True, 196, 1),     # a narrow block, many blocks per output
    ((8, 64, 7, 7), 4): SeLaunch(2, 32, 8, False, 1, 1),          # x off the 8-byte grid: vec 2
    ((8, 64, 56, 56), 4): SeLaunch(2, 32, 8, True, 25, 8),
    ((8, 64, 7, 7), 2): SeLaunch(1, 32, 16, False, 1, 1),         # x off the 4-byte grid: vec 1
    ((8, 64, 56, 56), 2): SeLaunch(1, 32, 16, True, 1, 16),
    ((2, 6, 9, 9), 0): SeLaunch(2, 4, 64, False, 1, 1),           # C % 4 == 2
    ((2, 6, 64, 64), 0): SeLaunch(2, 4, 64, True, 1, 2),
    ((16, 3, 8, 8), 0): SeLaunch(1, 32, 16, False, 1, 1),         # C = 3
    ((16, 3, 32, 32), 0): SeLaunch(1, 32, 16, True, 1, 2),
    ((8, 64, 64, 64), 2): SeLaunch(1, 32, 16, True, 16, 16),      # vec 1 across blocks
    ((4, 3, 128, 128), 0): SeLaunch(1, 8, 64, True, 16, 2),
}


def test_regime_shapes_reach_every_branch():
    for (shape, addr), want in SE_REGIME_SHAPES.items():
        n, c, h, w = shape
        assert se_reduce_config(n, c, h * w, addr) == want, (shape, addr)
    launches = SE_REGIME_SHAPES.values()
    assert {l.vec for l in launches} == {1, 2, 4}
    for vec in (1, 2, 4):
        assert {(l.split, l.ctas > 1) for l in launches if l.vec == vec} == {(False, False), (True, False), (True, True)}, vec


def test_every_row_index_a_thread_starts_at_is_inside_the_sample():
    # the kernels start a thread's walk at threadIdx.y + blockIdx.y * block_y; torch leaves a thread past the rows
    # without a value, so the restatement must never produce one, and a split grid stays within the semaphores
    for n in (1, 2, 3, 8, 32, 256):
        for c in (2, 3, 6, 8, 24, 100, 672, 1536):
            for hw in (2, 3, 15, 16, 49, 196, 255, 256, 784, 3136, 12544, 50176):
                for addr in (0, 2, 4):
                    l = se_reduce_config(n, c, hw, addr)
                    assert l.block_x * l.block_y * l.vec <= 512
                    if l.split:
                        assert l.block_y * l.ctas <= hw, (n, c, hw, addr, l)
                    if l.ctas > 1:
                        assert l.grid_x <= SEMAPHORES and l.block_x * l.block_y >= 128, (n, c, hw, l)


def make_model(arch):
    torch.manual_seed(0)
    return getattr(torchvision.models, arch)(weights=None, num_classes=10)


@pytest.mark.parametrize("arch", sorted(MODELS))
def test_fuse_model_swaps_the_se_modules_of_swapped_blocks_and_keeps_the_model(arch):
    model = make_model(arch)
    ses = [m for m in model.modules() if type(m) is SqueezeExcitation]
    assert len(ses) == MODELS[arch]
    hook_calls = []
    ses[0].register_forward_hook(lambda *a: hook_calls.append(1))
    keys, params = list(model.state_dict()), [id(p) for p in model.parameters()]
    ids = [id(m) for m in model.modules()]
    assert fused_norm.fuse_model(model) is model
    assert all(type(m) is fused_norm.FusedSqueezeExcitation for m in ses)
    assert [id(m) for m in model.modules()] == ids and list(model.state_dict()) == keys
    assert [id(p) for p in model.parameters()] == params
    classes = [type(m) for m in model.modules()]
    fused_norm.fuse_model(model)
    assert [type(m) for m in model.modules()] == classes
    with torch.no_grad():
        model.eval()(torch.zeros(1, 3, 32, 32))
    assert hook_calls == [1]


def test_only_se_inside_swapped_blocks_is_swapped_and_regnet_is_untouched():
    class SubSE(SqueezeExcitation):
        pass

    class SubBlock(efficientnet.MBConv):
        pass

    cnf = efficientnet.MBConvConfig(4, 3, 1, 16, 16, 1)
    norm = nn.BatchNorm2d
    plain, sub_block = efficientnet.MBConv(cnf, 0.0, norm), SubBlock(cnf, 0.0, norm)
    sub_se = efficientnet.MBConv(cnf, 0.0, norm)
    sub_se.block[2].__class__ = SubSE
    lone = SqueezeExcitation(16, 4)
    regnet = make_model("regnet_y_400mf")
    regnet_classes = [type(m) for m in regnet.modules()]
    assert any(type(m) is SqueezeExcitation for m in regnet.modules())
    model = nn.Sequential(plain, sub_block, sub_se, lone, regnet)
    fused_norm.fuse_model(model)
    assert type(plain.block[2]) is fused_norm.FusedSqueezeExcitation
    assert type(sub_block.block[2]) is SqueezeExcitation    # the block is not swapped, nor its SE
    assert type(sub_se.block[2]) is SubSE
    assert type(lone) is SqueezeExcitation
    assert [type(m) for m in regnet.modules()] == regnet_classes
    v3 = make_model("mobilenet_v3_large")
    fused_norm.fuse_model(v3)
    blocks = [m for m in v3.modules() if isinstance(m, mobilenetv3.InvertedResidual)]
    assert all(type(m) is fused_norm.FusedInvertedResidualV3 for m in blocks)
    assert sum(type(m) is fused_norm.FusedSqueezeExcitation for m in v3.modules()) == MODELS["mobilenet_v3_large"]


@pytest.mark.parametrize("act", ["silu_sigmoid", "relu_hardsigmoid"])
@pytest.mark.parametrize("case", ["cpu_fp32", "cpu_bf16_channels_last", "nchw_fp32"])
def test_fused_se_gives_its_parent_s_bits_where_nothing_is_fused(act, case):
    torch.manual_seed(3)
    kw = {"activation": nn.SiLU} if act == "silu_sigmoid" else {"scale_activation": nn.Hardsigmoid}
    parent = SqueezeExcitation(24, 6, **kw)
    fused = copy.deepcopy(parent)
    fused.__class__ = fused_norm.FusedSqueezeExcitation
    x = torch.randn(2, 24, 5, 5)
    if case == "cpu_bf16_channels_last":
        parent, fused, x = parent.bfloat16(), fused.bfloat16(), x.bfloat16().contiguous(memory_format=torch.channels_last)
    xa, xb = x.clone().requires_grad_(), x.clone().requires_grad_()
    ya, yb = parent(xa), fused(xb)
    assert torch.equal(ya, yb)
    dy = torch.randn_like(ya)
    ya.backward(dy)
    yb.backward(dy)
    assert torch.equal(xa.grad, xb.grad)
    for pa, pb in zip(parent.parameters(), fused.parameters()):
        assert torch.equal(pa.grad, pb.grad)


def test_se_ok_needs_a_plain_hook_free_pool():
    se = fused_norm.FusedSqueezeExcitation(8, 2)
    x = torch.zeros(2, 8, 4, 4)   # a CPU input is never fused, whatever the module
    assert not fused_norm._se_ok(se, x)
    pool = se.avgpool
    assert type(pool) is nn.AdaptiveAvgPool2d and pool.output_size == 1


def test_se_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_fused_se_cpu as t; t.se_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def se_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def pool(n=2, c=8, hw=16, **null):
        a = {k: None if k in null else p for k in ("x", "pooled", "scratch")}
        return lib.b200c_se_pool(a["x"], a["pooled"], n, c, hw, a["scratch"], 1 << 20, None)

    def scale(n=2, c=8, hw=16, **null):
        a = {k: None if k in null else p for k in ("x", "s", "y")}
        return lib.b200c_se_scale(a["x"], a["s"], a["y"], n, c, hw, None)

    def reduce(n=2, c=8, hw=16, **null):
        a = {k: None if k in null else p for k in ("dy", "x", "ds", "scratch")}
        return lib.b200c_se_backward_reduce(a["dy"], a["x"], a["ds"], n, c, hw, a["scratch"], 1 << 20, None)

    def elemt(n=2, c=8, hw=16, **null):
        a = {k: None if k in null else p for k in ("dy", "s", "gp", "dx")}
        return lib.b200c_se_backward_elemt(a["dy"], a["s"], a["gp"], a["dx"], n, c, hw, None)

    calls = {pool: ("x", "pooled", "scratch"), scale: ("x", "s", "y"), reduce: ("dy", "x", "ds", "scratch"),
             elemt: ("dy", "s", "gp", "dx")}
    for call, names in calls.items():
        # n, c, hw >= 1 and n * c * hw < 2^31
        for n, c, hw in ((0, 8, 16), (-1, 8, 16), (2, 0, 16), (2, -8, 16), (2, 8, 0), (2, 8, -1), (1 << 16, 1 << 15, 1),
                         (2, 1 << 15, 1 << 15), (1, 2, 1 << 30)):
            assert call(n=n, c=c, hw=hw) == N.EINVAL, (call.__name__, n, c, hw)
            assert "bad shape" in N.last_error()
        for name in names:
            assert call(**{name: 1}) == N.EINVAL, (call.__name__, name)
            assert "null" in N.last_error()
        assert lib.b200c_se_scratch_bytes(2, 0, 16) == 0 and lib.b200c_se_scratch_bytes(1 << 16, 1 << 15, 1) == 0
    for call in (pool, reduce):   # one channel over many rows is reduced along its fastest dimension by torch
        assert call(c=1, hw=16) == N.EINVAL and "fastest" in N.last_error()
    assert lib.b200c_launch_count() == before
    # past the checks the reducing calls size their scratch on the device, and the elementwise ones launch: without a
    # device both fail as CUDA errors
    for call in calls:
        assert call() == N.ECUDA, call.__name__
    assert scale(c=1, hw=16) == N.ECUDA and elemt(n=1, c=1, hw=(1 << 31) - 1) == N.ECUDA
    assert lib.b200c_launch_count() == before
