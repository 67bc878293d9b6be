"""The eval batch-norm sites under torch.profiler, each trace in a process of its own (test_gpu_fused_infer.py has the
traced code): a resnet50 eval forward runs none of torch's batch-norm, ReLU, add or max-pool kernels, and every
`b200c::bn_infer` kernel is launched by the case test_gpu_fused_infer.KERNELS gives it.

These run after the other GPU files: a profiler session in a subprocess on the same GPU has been seen to cost a later
in-process session of this test process its first kernel records (test_gpu_fused_norm_paths.py)."""
import json
import os
import re
import subprocess
import sys

import pytest

from test_gpu_fused_infer import KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_resnet50_eval_trace_runs_no_torch_batch_norm_relu_add_or_max_pool():
    pytest.importorskip("torchvision")
    # in a process of its own, as test_gpu_fused_stem's trace
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_gpu_fused_infer as t; t.infer_trace_kernels()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    got = json.loads(out.stdout.strip().splitlines()[-1])
    names = got["kernels"]
    assert names, "the profiler saw no CUDA kernel"
    assert got["launches"] == 49
    torch_ops = [k for k in names if re.search(r"batch_norm|invstd|clamp_min|relu|threshold|CUDAFunctor_add|max_pool", k, re.I)
                 and "b200c::" not in k and "at::native" in k]
    assert not torch_ops, f"torch kernels in the eval forward: {sorted(set(torch_ops))}"
    ours = [k for k in names if "b200c::bn_infer::" in k]
    assert len(ours) == 49 and sum("k_infer_pool" in k for k in ours) == 1, sorted(set(ours))
    assert not [k for k in names if "b200c::bn::k_" in k], "a training kernel ran in the eval forward"


@pytest.mark.gpu
def test_every_eval_kernel_is_launched_by_its_case():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_gpu_fused_infer as t; t.trace_cases()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    launched = json.loads(out.stdout.strip().splitlines()[-1])
    assert set(launched) == set(KERNELS.values())
    missing = {k: case for k, case in KERNELS.items() if k not in launched[case]}
    assert not missing, f"kernels their case did not launch: {missing}"
    # one kernel per case: the case names its kernel
    assert all(len(v) == 1 for v in launched.values()), launched
