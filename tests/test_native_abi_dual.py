"""The dual tail's C-ABI calls reject bad arguments before any launch, and a block takes the dual tail only for a
plain nn.Sequential(nn.Conv2d, batch norm) downsample without hooks; no GPU needed."""
import ctypes
import os
import subprocess
import sys

import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FWD = ("x", "xds", "y", "mask", "w", "b", "rm", "rv", "nbt", "sm", "si", "wd", "bd", "rmd", "rvd", "nbtd", "smd", "sid")
BWD = ("dy", "dy2", "y", "mask", "x", "xds", "dx", "dxds", "w", "sm", "si", "gw", "gb", "wd", "smd", "sid", "gwd", "gbd")


def test_bn_dual_calls_reject_bad_arguments_before_any_launch():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_native_abi_dual as t; t.bn_dual_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def bn_dual_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()
    assert lib.b200c_bn_dual_scratch_bytes(0) == 0 and lib.b200c_bn_dual_scratch_bytes(65537) == 0
    assert lib.b200c_bn_dual_scratch_bytes(65536) > lib.b200c_bn_scratch_bytes(65536)

    def fwd(m=8, c=8, scratch=p, **null):
        a = [None if k in null else p for k in FWD]
        return lib.b200c_bn_forward_dual(*a[:11], 0.1, 1e-5, *a[11:], 0.1, 1e-5, m, c, scratch, None)

    def bwd(m=8, c=8, scratch=p, **null):
        a = [None if k in null else p for k in BWD]
        return lib.b200c_bn_backward_dual(*a, m, c, scratch, None)

    for call in (fwd, bwd):
        for m, c in ((0, 8), (8, 0), (-1, 8), (8, 65544), (2 ** 16, 2 ** 15)):
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
        for c in (4, 12, 100):   # with a mask
            assert call(c=c) == N.EINVAL, (call.__name__, c)
        assert call(scratch=None) == N.EINVAL
    for name in set(FWD) - {"mask", "nbt", "nbtd"}:
        assert fwd(**{name: 1}) == N.EINVAL, name
    for name in set(BWD) - {"dy2", "y", "mask"}:
        assert bwd(**{name: 1}) == N.EINVAL, name
    assert bwd(y=1, mask=1) == N.EINVAL
    assert "batch norm dual" in N.last_error()
    assert lib.b200c_launch_count() == before


def test_only_a_plain_conv_and_batch_norm_downsample_takes_the_dual_tail():
    conv, bn = nn.Conv2d(8, 16, 1, stride=2, bias=False), nn.BatchNorm2d(16)
    assert fused_norm._downsample_bn(nn.Sequential(conv, bn)) is bn
    assert fused_norm._downsample_bn(nn.Sequential(conv, bn, nn.Identity())) is None
    assert fused_norm._downsample_bn(nn.Sequential(nn.AvgPool2d(2), bn)) is None
    assert fused_norm._downsample_bn(conv) is None
    hooked = nn.Sequential(conv, bn)
    h = hooked.register_forward_hook(lambda mod, args, out: None)
    assert fused_norm._downsample_bn(hooked) is None
    h.remove()
    h = bn.register_forward_pre_hook(lambda mod, args: None)
    assert fused_norm._downsample_bn(nn.Sequential(conv, bn)) is None
    h.remove()
