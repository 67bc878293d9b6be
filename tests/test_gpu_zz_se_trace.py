"""Every `b200c::se` kernel under torch.profiler, in a process of its own (test_gpu_zz_infer_trace.py explains why):
each kernel of test_gpu_fused_se.KERNELS is launched by the case the table gives it, and no case launches a
`b200c::se` kernel the table lacks."""
import json
import os
import subprocess
import sys

import pytest

from test_gpu_fused_se import KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_every_se_kernel_is_launched_by_its_case():
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_gpu_fused_se as t; t.trace_cases()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    launched = json.loads(out.stdout.strip().splitlines()[-1])
    assert set(launched) == set(KERNELS.values())
    missing = {k: case for k, case in KERNELS.items() if k not in launched[case]}
    assert not missing, f"kernels their case did not launch: {missing}"
    unknown = {k for names in launched.values() for k in names} - set(KERNELS)
    assert not unknown, f"launched kernels missing from KERNELS: {unknown}"
