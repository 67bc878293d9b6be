"""The batch-norm C-ABI calls with a ReLU mask reject bad arguments before any launch; no GPU needed."""
import ctypes
import os
import subprocess
import sys

from ant_ray_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bn_mask_calls_reject_bad_arguments_before_any_launch():
    # As in test_native_abi: a made-up pointer that a correct library never dereferences, in a process that sees
    # no CUDA device, so that a lost check fails with a CUDA error instead of launching.
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_native_abi_mask as t; t.bn_mask_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def bn_mask_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def fwd(m=8, c=8, scratch=p, **null):
        a = {k: None if k in null else p for k in ("x", "id", "y", "mask", "w", "b", "rm", "rv", "nbt", "sm", "si")}
        return lib.b200c_bn_forward_mask(a["x"], a["id"], a["y"], a["mask"], a["w"], a["b"], a["rm"], a["rv"], a["nbt"], a["sm"],
                                         a["si"], m, c, 0.1, 1e-5, scratch, None)

    def bwd(m=8, c=8, scratch=p, **null):
        a = {k: None if k in null else p for k in ("dy", "dy2", "mask", "x", "gid", "dx", "w", "sm", "si", "gw", "gb")}
        return lib.b200c_bn_backward_mask(a["dy"], a["dy2"], a["mask"], a["x"], a["gid"], a["dx"], a["w"], a["sm"], a["si"],
                                          a["gw"], a["gb"], m, c, scratch, None)

    for call in (fwd, bwd):
        for m, c in ((0, 8), (8, 0), (-1, 8), (8, 131080), (2 ** 16, 2 ** 15), (2 ** 14, 2 ** 17)):   # m * c = 2^31 last
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
        for c in (4, 12, 100, 131071):   # the mask packs 8 channels per byte
            assert call(c=c) == N.EINVAL, (call.__name__, c)
        assert call(mask=1) == N.EINVAL
        assert "mask" in N.last_error()
        assert call(scratch=None) == N.EINVAL
    for name in ("x", "y", "w", "b", "rm", "rv", "sm", "si"):
        assert fwd(**{name: 1}) == N.EINVAL, name
    for name in ("dy", "x", "dx", "w", "sm", "si", "gw", "gb"):
        assert bwd(**{name: 1}) == N.EINVAL, name
    assert "batch norm" in N.last_error()
    assert lib.b200c_launch_count() == before
