"""The fused stem's C-ABI calls reject bad arguments before any launch, and FusedResNet picks the stem site only for
nn.MaxPool2d(3, 2, 1) without hooks; no GPU needed."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bn_pool_calls_reject_bad_arguments_before_any_launch():
    # as test_native_abi_mask: a made-up pointer in a process that sees no CUDA device
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_native_abi_pool as t; t.bn_pool_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def bn_pool_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def fwd(n=2, h=4, w=4, c=8, scratch=p, **null):
        a = {k: None if k in null else p for k in ("x", "y", "am", "wt", "b", "rm", "rv", "nbt", "sm", "si")}
        return lib.b200c_bn_forward_pool(a["x"], a["y"], a["am"], a["wt"], a["b"], a["rm"], a["rv"], a["nbt"], a["sm"], a["si"],
                                         n, h, w, c, 0.1, 1e-5, scratch, None)

    def bwd(n=2, h=4, w=4, c=8, scratch=p, **null):
        a = {k: None if k in null else p for k in ("dy", "am", "x", "g", "dx", "wt", "sm", "si", "gw", "gb")}
        return lib.b200c_bn_backward_pool(a["dy"], a["am"], a["x"], a["g"], a["dx"], a["wt"], a["sm"], a["si"], a["gw"], a["gb"],
                                          n, h, w, c, scratch, None)

    for call in (fwd, bwd):
        for n, h, w, c in ((0, 4, 4, 8), (2, 0, 4, 8), (2, 4, 0, 8), (-1, 4, 4, 8), (2, 4, 4, 0), (2, 4, 4, 131073),
                           (65536, 256, 256, 1), (1 << 14, 1 << 10, 1 << 10, 1), (256, 112, 112, 1024)):
            assert call(n=n, h=h, w=w, c=c) == N.EINVAL, (call.__name__, n, h, w, c)
        assert "pool" in N.last_error()
        assert call(scratch=None) == N.EINVAL
    for name in ("x", "y", "am", "wt", "b", "rm", "rv", "sm", "si"):
        assert fwd(**{name: 1}) == N.EINVAL, name
    for name in ("dy", "am", "x", "g", "dx", "wt", "sm", "si", "gw", "gb"):
        assert bwd(**{name: 1}) == N.EINVAL, name
    assert "batch norm pool" in N.last_error()
    assert lib.b200c_launch_count() == before


@pytest.mark.parametrize("pool,fusable", [
    (nn.MaxPool2d(3, 2, 1), True),
    (nn.MaxPool2d((3, 3), (2, 2), (1, 1)), True),
    (nn.MaxPool2d(3, 2, 1, ceil_mode=True), False),
    (nn.MaxPool2d(3, 2, 1, return_indices=True), False),
    (nn.MaxPool2d(3, 2, 1, dilation=2), False),
    (nn.MaxPool2d(3, 1, 1), False),
    (nn.MaxPool2d(2, 2, 1), False),
    (nn.MaxPool2d(3, 2, 0), False),
    (nn.AvgPool2d(3, 2, 1), False),
])
def test_stem_site_takes_only_the_resnet_maxpool(pool, fusable):
    assert fused_norm._pool_fusable(pool) is fusable


def test_a_hook_on_the_maxpool_keeps_the_module_call():
    pool = nn.MaxPool2d(3, 2, 1)
    h = pool.register_forward_pre_hook(lambda mod, args: None)
    assert not fused_norm._pool_fusable(pool)
    h.remove()
    assert fused_norm._pool_fusable(pool)
