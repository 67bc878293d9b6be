"""The ShuffleNetV2 block-end sites under torch.profiler, each trace in a process of its own (test_gpu_fused_shuffle.py
and test_gpu_zz_shuffle_models.py have the traced code), after every other GPU file for the reason
test_gpu_zz_trace_dense.py gives.

Every `b200c::bn_shuffle` kernel is launched by the case test_fused_shuffle_cpu.KERNELS gives it.  A training step of
shufflenet_v2_x0_5 and x1_0 runs all 56 batch norms on native sites: the stem, 17 ReLU sites, 19 sites without
activation after the depthwise convolutions, and 16 block ends (13 of one batch norm, 3 of two), and no torch
batch-norm or threshold_backward kernel; the only torch cat kernels left are the backward of each stride-1 block's
x.chunk, which builds the block input's gradient outside the block end."""
import json
import os
import subprocess
import sys

import pytest

from test_fused_shuffle_cpu import KERNELS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_every_shuffle_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_shuffle as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    for kernel, case in KERNELS.items():
        assert kernel in launched[case], (kernel, launched)
    assert {k for names in launched.values() for k in names} <= set(KERNELS), launched


def test_training_step_runs_every_batch_norm_on_a_native_site():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_shuffle_models as t; t.trace_cases()")
    # torch's only cats are the 13 stride-1 blocks' SplitBackward of x.chunk (the block input's gradient, outside the
    # block end); statistics: one launch per batch norm, the stride-2 ends' two batch norms in one dual launch; the stem (pool),
    # 17 ReLU sites and 19 sites without activation (bn_res without identity runs k_bn_transform)
    expect = {"batch_norms": 56, "bn_stats": 56 - 2 * 3, "bn_stats_dual": 3, "shuffle_transform": 16, "shuffle_reduce": 16,
              "shuffle_elemt": 16, "bn_pool": 1, "bn_transform": 17 + 19, "res_transform": 0, "bn_reduce": 1 + 17 + 19,
              "bn_elemt": 1 + 17 + 19, "torch_bn": 0, "torch_cat": 13, "torch_relu": 0}
    for arch, c in got.items():
        assert {k: c[k] for k in expect} == expect, (arch, c)
