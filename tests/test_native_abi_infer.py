"""The eval batch-norm C-ABI calls reject bad arguments before any launch; no GPU needed."""
import ctypes
import os
import subprocess
import sys

import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bn_infer_calls_reject_bad_arguments_before_any_launch():
    # as test_native_abi_pool: a made-up pointer in a process that sees no CUDA device
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_native_abi_infer as t; t.bn_infer_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def bn_infer_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()
    names = ("x", "y", "wt", "b", "rm", "rv")

    def one(m=64, c=8, bf16=0, identity=None, **null):
        a = {k: None if k in null else p for k in names}
        return lib.b200c_bn_infer(a["x"], identity, a["y"], a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-5, m, c, None)

    def dual(m=64, c=8, bf16=0, **null):
        a = {k: None if k in null else p for k in names + ("xd", "wd", "bd", "rmd", "rvd")}
        return lib.b200c_bn_infer_dual(a["x"], a["xd"], a["y"], a["wt"], a["b"], a["rm"], a["rv"], 1e-5, a["wd"], a["bd"], a["rmd"],
                                       a["rvd"], 1e-3, bf16, m, c, None)

    def pool(m=None, c=8, bf16=0, n=2, h=4, w=4, **null):
        a = {k: None if k in null else p for k in names}
        return lib.b200c_bn_infer_pool(a["x"], a["y"], a["wt"], a["b"], a["rm"], a["rv"], bf16, 1e-5, n, h, w, c, None)

    for call, site in ((one, "batch norm infer"), (dual, "batch norm infer dual")):
        # m >= 1 (one value per channel is an eval batch norm's minimum), c >= 1, fewer than 2^31 elements
        for m, c in ((0, 8), (-1, 8), (64, 0), (64, -8), (1 << 28, 8), (65536, 32768), (2, 1 << 30)):
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
            assert site in N.last_error()
        for bf16 in (2, -1):
            assert call(bf16=bf16) == N.EINVAL and "param_bf16" in N.last_error()
    for name in names:
        assert one(**{name: 1}) == N.EINVAL, name
        assert "batch norm infer: null buffer" in N.last_error()
        assert pool(**{name: 1}) == N.EINVAL, name
        assert "batch norm infer pool: null buffer" in N.last_error()
    for name in names + ("xd", "wd", "bd", "rmd", "rvd"):
        assert dual(**{name: 1}) == N.EINVAL, name
        assert "batch norm infer dual: null buffer" in N.last_error()
    for n, h, w, c in ((0, 4, 4, 8), (2, 0, 4, 8), (2, 4, 0, 8), (-1, 4, 4, 8), (2, 4, 4, 0), (65536, 256, 256, 1),
                       (1 << 14, 1 << 10, 1 << 10, 1), (256, 112, 112, 1024)):
        assert pool(n=n, h=h, w=w, c=c) == N.EINVAL, (n, h, w, c)
        assert "pool" in N.last_error()
    assert pool(bf16=3) == N.EINVAL and "param_bf16" in N.last_error()
    assert lib.b200c_launch_count() == before
    # the largest accepted shape gets past the checks: without a device the launch itself fails, as a CUDA error
    assert one(m=(1 << 31) - 1, c=1) == N.ECUDA
    assert lib.b200c_launch_count() == before


def test_a_training_or_cpu_site_is_not_an_eval_site():
    bn, relu = nn.BatchNorm2d(8), nn.ReLU()
    x = torch.zeros(2, 8, 4, 4, dtype=torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert fused_norm._site(bn, x, (relu,)) is not fused_norm._EVAL           # training mode
    bn.eval()
    assert fused_norm._site(bn, x, (relu,)) is not fused_norm._EVAL           # a CPU tensor
    assert fused_norm._site(nn.BatchNorm2d(8, track_running_stats=False).eval(), x, (relu,)) is not fused_norm._EVAL
