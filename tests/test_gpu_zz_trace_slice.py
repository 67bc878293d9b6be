"""The slice batch-norm sites under torch.profiler, each trace in a process of its own (test_gpu_fused_slice.py and
test_gpu_zz_slice_models.py have the traced code), after every other GPU file for the reason
test_gpu_zz_trace_dense.py gives.

Every `b200c::bn_slice` kernel is launched by the case test_fused_slice_cpu.KERNELS gives it.  A training step of
googlenet (59 batch norms) and of inception_v3 (96), aux heads on, runs every batch norm as a native site, a slice site
inside each Inception module and a ReLU site everywhere else, and no torch batch-norm or cat kernel; the only torch
ReLU kernels are those of GoogLeNet's aux heads' F.relu after fc1, outside the swapped modules."""
import json
import os
import subprocess
import sys

import pytest

from test_fused_slice_cpu import KERNELS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


def test_every_slice_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_slice as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    for kernel, case in KERNELS.items():
        assert kernel in launched[case], (kernel, launched)
    assert {k for names in launched.values() for k in names} <= set(KERNELS), launched


def test_training_step_runs_every_batch_norm_on_a_native_site():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_slice_models as t; t.trace_cases()")
    # GoogLeNet's two aux heads run F.relu after fc1: at most one forward and one backward kernel each
    for case, norms, aux_relus in (("googlenet", 59, 4), ("inception_v3", 96, 0)):
        c = got[case]
        assert c["batch_norms"] == norms and c["bn_stats"] == norms, (case, c)
        slices = c["slice_sites"]
        for f in ("slice_transform", "slice_reduce", "slice_elemt"):
            assert c[f] == slices, (case, f, c)
        for f in ("bn_transform", "bn_reduce", "bn_elemt"):
            assert c[f] == norms - slices, (case, f, c)
        assert c["torch_bn"] == 0 and c["torch_cat"] == 0 and c["torch_relu"] <= aux_relus, (case, c)
