"""fused_norm.fuse_resnet rewrites torchvision ResNets in place without changing what they are or compute.

The rewrite keeps the model object, its submodules, parameters and state_dict keys; the rewritten blocks are still
instances of torchvision's classes.  Inputs that cannot run fused (here: CPU tensors in train and eval mode, fp32,
NCHW and channels-last) take the parent classes' ops and give the same bits as the untouched model."""
import copy

import pytest
import torch

from ant_ray_b200 import fused_norm

torchvision = pytest.importorskip("torchvision")
from torchvision.models.resnet import BasicBlock, Bottleneck, ResNet  # noqa: E402


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
def test_rewrite_keeps_identity_state_and_keys(arch):
    torch.manual_seed(0)
    model = getattr(torchvision.models, arch)(weights=None)
    keys = list(model.state_dict().keys())
    mods = list(model.modules())
    params = list(model.parameters())
    assert fused_norm.fuse_resnet(model) is model
    assert list(model.state_dict().keys()) == keys
    assert [id(m) for m in model.modules()] == [id(m) for m in mods]
    assert all(a is b for a, b in zip(model.parameters(), params)) and len(list(model.parameters())) == len(params)
    assert type(model) is fused_norm.FusedResNet and isinstance(model, ResNet)
    blocks = [m for m in model.modules() if isinstance(m, (BasicBlock, Bottleneck))]
    assert blocks and all(type(m) in (fused_norm.FusedBasicBlock, fused_norm.FusedBottleneck) for m in blocks)
    assert fused_norm.fuse_resnet(model) is model   # idempotent
    assert type(model) is fused_norm.FusedResNet


@pytest.mark.parametrize("arch", ["resnet18", "resnet50"])
@pytest.mark.parametrize("mode", ["train", "eval"])
@pytest.mark.parametrize("fmt", ["nchw", "channels_last"])
def test_fallback_computes_what_the_parent_classes_compute(arch, mode, fmt):
    torch.manual_seed(0)
    ref = getattr(torchvision.models, arch)(weights=None)
    fused = fused_norm.fuse_resnet(copy.deepcopy(ref))
    memory_format = torch.channels_last if fmt == "channels_last" else torch.contiguous_format
    for m in (ref, fused):
        m.to(memory_format=memory_format).train(mode == "train")
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(1)).contiguous(memory_format=memory_format)
    want, got = ref(x), fused(x)
    assert torch.equal(got, want)
    if mode == "train":
        want.sum().backward()
        got.sum().backward()
        for (name, a), b in zip(fused.named_parameters(), ref.parameters()):
            assert torch.equal(a.grad, b.grad), name
    for (name, a), b in zip(fused.state_dict().items(), ref.state_dict().values()):
        assert torch.equal(a, b), name


def test_named_shapes_reach_their_launch_regimes():
    # The GPU tests run these shapes for the regimes named beside them (gpu_common.BN_REGIME_SHAPES).  A change of
    # reduce_config or its constants must come with shapes that reach the same regimes.
    from gpu_common import BN_REGIME_SHAPES, bn_launch_config

    for (n, c, h, w), want in BN_REGIME_SHAPES.items():
        assert bn_launch_config(n * h * w, c) == want, (n, c, h, w)
    # the collapsed case has 2..7 rows of blocks before collapsing, and the partial tiles really are partial
    assert bn_launch_config(4 * 16 * 16, 100).block_y * 16 * 4 == 4 * 16 * 16
    partial = [(s, cfg) for s, cfg in BN_REGIME_SHAPES.items() if s[1] % cfg.block_x]
    assert any(cfg.grid_y > 1 for _, cfg in partial) and any(cfg.grid_y == 1 for _, cfg in partial)
    assert any(cfg.block_x > 32 for cfg in BN_REGIME_SHAPES.values())
    assert any(s[1] % 8 for s in BN_REGIME_SHAPES) and any(s[1] % 8 == 0 for s in BN_REGIME_SHAPES)


def test_dual_shapes_reach_their_launch_regimes_within_half_the_semaphores():
    # A dual tail's plane 1 counts on semaphores[grid_x + x], so both planes' columns must fit the region; the limit
    # shape's plane 1 reaches its last semaphore.
    from gpu_common import BN_DUAL_REGIME_SHAPES, BN_MAX_CHANNELS, BN_REGIME_SHAPES, BN_SEMAPHORES, BnLaunch, bn_launch_config

    assert len(BN_DUAL_REGIME_SHAPES) == len(BN_REGIME_SHAPES)
    assert {s: cfg for s, cfg in BN_DUAL_REGIME_SHAPES.items() if s[1] != BN_MAX_CHANNELS // 2} == \
        {s: cfg for s, cfg in BN_REGIME_SHAPES.items() if s[1] != BN_MAX_CHANNELS}
    assert BN_DUAL_REGIME_SHAPES[(2, 65536, 32, 32)] == BnLaunch(32, 16, 2048, 8)
    for (n, c, h, w), want in BN_DUAL_REGIME_SHAPES.items():
        assert bn_launch_config(n * h * w, c) == want, (n, c, h, w)
        assert 2 * want.grid_x <= BN_SEMAPHORES, (n, c, h, w)
    last = max(cfg.grid_x + cfg.grid_x - 1 for cfg in BN_DUAL_REGIME_SHAPES.values() if cfg.grid_y > 1)
    assert last == BN_SEMAPHORES - 1 == 4095


def test_merged_grids_fit_the_semaphore_region():
    # Each column of a merged grid owns one semaphore of the fixed region at the start of the scratch buffer, so no
    # shape the kernels take may merge over more columns than the region holds.  The largest channel count uses
    # every semaphore.
    from gpu_common import BN_MAX_CHANNELS, BN_SEMAPHORES, bn_launch_config

    worst = 0
    for m in (2, 3, 17, 100, 1000, 2048, 5000, 10 ** 5, 10 ** 6):
        for c in range(1, min(BN_MAX_CHANNELS, (2 ** 31 - 1) // m) + 1):
            cfg = bn_launch_config(m, c)
            assert cfg.block_x * cfg.block_y <= 512 and cfg.grid_y <= 128
            if cfg.grid_y > 1:
                worst = max(worst, cfg.grid_x)
    assert worst == BN_SEMAPHORES == 4096
