"""The concatenation batch-norm sites under torch.profiler, each trace in a process of its own (test_gpu_fused_cat.py
and test_gpu_zz_dense_models.py have the traced code).

This file runs after every other GPU file: a profiler session in a subprocess on the same GPU has been seen to cost a
later in-process session of the test process its first kernel records (test_gpu_zz_infer_trace.py), so these sessions
come after every other one.

Every `b200c::bn_cat` kernel is launched by the case test_fused_cat_cpu.KERNELS gives it.  A densenet121 training step
launches one concatenation site per concatenating batch norm and one ReLU site per norm2, and no torch batch-norm, cat
or ReLU kernel; with memory_efficient, the checkpointed layers run torchvision's own ops while the sites of the
model's walk stay fused."""
import json
import os
import subprocess
import sys

import pytest

from test_fused_cat_cpu import KERNELS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_every_cat_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_cat as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    for kernel, case in KERNELS.items():
        assert kernel in launched[case], (kernel, launched)
    assert {k for names in launched.values() for k in names} <= set(KERNELS), launched


def test_training_step_runs_on_the_sites():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_dense_models as t; t.trace_cases()")
    c = got["densenet121"]
    cat_sites = c["layers"] + c["transitions"] + 1   # norm1 of each layer, each transition's norm, norm5
    for f in ("cat_stats", "cat_transform", "cat_reduce", "cat_elemt"):
        assert c[f] == cat_sites, (f, c)
    # one ReLU site per norm2, and the stem
    assert c["bn_stats"] == c["layers"] + 1 and c["bn_transform"] == c["layers"] and c["pool_fwd"] == 1, c
    assert c["torch_bn"] == 0 and c["torch_cat"] == 0 and c["torch_relu"] == 0, c
    # checkpointed layers run torchvision's forward, whose cat runs in the forward and again in the recompute (a block's
    # first layer concatenates one tensor, a plain copy); the walk's sites stay fused
    e = got["densenet121_memory_efficient"]
    assert e["cat_stats"] == e["transitions"] + 1 and e["bn_stats"] == 1 and e["pool_fwd"] == 1, e
    assert e["torch_cat"] == 2 * (e["layers"] - 4) and e["torch_bn"] > 0, e
