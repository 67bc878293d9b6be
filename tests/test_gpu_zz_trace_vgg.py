"""The VGG stage-end sites under torch.profiler, each trace in a process of its own (test_gpu_fused_vgg.py and
test_gpu_zz_vgg_models.py have the traced code), after every other GPU file for the reason test_gpu_zz_trace_dense.py
gives.

Every `b200c::bn_pool2` kernel is launched by the case test_fused_vgg_cpu.KERNELS gives it.  A training step of
vgg16_bn runs all 13 batch norms on native sites: 5 stage ends and 8 ReLU sites, and no torch batch-norm or max_pool2d
kernel in either direction; the only torch ReLU kernels are the classifier's two nn.ReLU, which follow Linear layers,
not batch norms."""
import json
import os
import subprocess
import sys

import pytest

from test_fused_vgg_cpu import KERNELS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_every_pool2_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_vgg as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    for kernel, case in KERNELS.items():
        assert kernel in launched[case], (kernel, launched)
    assert {k for names in launched.values() for k in names} <= set(KERNELS), launched


def test_training_step_runs_every_batch_norm_on_a_native_site():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_vgg_models as t; t.trace_cases()")
    # torch_relu: the classifier's two nn.ReLU (after Linear layers, not batch-norm sites)
    expect = {"batch_norms": 13, "bn_stats": 13, "pool2_fwd": 5, "pool2_reduce": 5, "pool2_elemt": 5, "bn_transform": 8,
              "bn_reduce": 8, "bn_elemt": 8, "torch_bn": 0, "torch_relu": 2, "torch_max_pool": 0}
    assert {k: got["vgg16_bn"][k] for k in expect} == expect, got
