"""The ReLU6 / SiLU / Hardswish batch-norm sites under torch.profiler, each trace in a process of its own
(test_gpu_fused_act.py and test_gpu_zz_act_models.py have the traced code), after the other GPU files as test_gpu_zz_infer_trace.py explains.

A fused model's training step launches one `b200c::bn_act` transform per ReLU6, SiLU or Hardswish site and exactly that
many fewer of torch's forward kernels for those activations than the untouched model (which still runs them
elsewhere, e.g. in EfficientNet's squeeze-excitation).  Each site's backward runs one `b200c::bn_act` reduce and no
torch activation backward, except where the gradient arrives in NCHW: in these models, the block before the average
pool, which keeps eager torch's backward ops.  Every `b200c::bn_act`
kernel is launched by the case test_gpu_fused_act.KERNELS gives it."""
import json
import os
import subprocess
import sys

import pytest

from test_gpu_fused_act import KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# torch's forward and backward kernel families of each activation
TORCH_FAMILIES = {"relu6": ("clamp", "hardtanh_backward"), "silu": ("silu", "silu_backward"),
                  "hardswish": ("hardswish", "hardswish_backward")}


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
def test_model_steps_run_no_torch_activation_kernel_at_a_fused_site():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_act_models as t; t.trace_models()")
    for arch, counts in got.items():
        sites, fused, unfused = counts["sites"], counts["fused"], counts["unfused"]
        n = sum(sites.values())   # regnet_y_400mf has only ReLU sites
        # a site whose gradient arrives in NCHW keeps eager torch's backward ops (in these models: the block before the
        # average pool)
        assert fused["act_transform"] == n and fused["act_reduce"] == n - counts["nchw_gradient_sites"], (arch, counts)
        assert unfused["act_transform"] == 0, arch
        # only for the activations the model fuses: ReLU runs on clamp_scalar as well, and its sites are fused too
        for act, (forward, backward) in TORCH_FAMILIES.items():
            if not sites[act]:
                continue
            assert fused[forward] == unfused[forward] - sites[act], (arch, forward, fused, unfused, sites)
            assert fused[backward] == unfused[backward] - fused[f"act_reduce_{act}"], (arch, backward, fused, unfused, sites)


@pytest.mark.gpu
def test_every_act_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_act as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    missing = {k: case for k, case in KERNELS.items() if k not in launched[case]}
    assert not missing, f"kernels their case did not launch: {missing}"
    unknown = {k for names in launched.values() for k in names} - set(KERNELS)
    assert not unknown, f"launched kernels missing from KERNELS: {unknown}"
