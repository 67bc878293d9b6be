"""Whole torchvision models with fused squeeze-excitation sites (fused_norm.FusedSqueezeExcitation) against the untouched
models, bit for bit: efficientnet_b0, mobilenet_v3_large and efficientnet_v2_s (num_classes 10, 96 x 96) after
`fuse_model` and after `prepare_model`, three reseeded SGD-momentum steps under bf16 autocast, channels-last, with
EfficientNet's stochastic depth active, then an eval forward under inference_mode.  Losses, gradients, parameters,
buffers and logits must have the same bits.

A profiler trace in a process of its own (test_gpu_zz_infer_trace.py explains why): a fused training step launches one
pool, one scale, one backward reduce and one backward elementwise kernel per SE site, and against the same model with
its SE modules back on torchvision's class it launches, per SE site, two fewer torch reductions (the mean and the sum),
four fewer multiplies (s * x, dy * x, dy * s and the mean backward's division) and one fewer add."""
import copy
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits
from test_gpu_zz_act_models import batches, mismatches, train_steps
from test_gpu_zz_res_models import make_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SE_SITES = {"efficientnet_b0": 16, "mobilenet_v3_large": 8, "efficientnet_v2_s": 30}


@pytest.fixture(scope="module")
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def se_sites(model):
    return [m for m in model.modules() if type(m) is fused_norm.FusedSqueezeExcitation]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["fuse_model", "prepare_model"])
@pytest.mark.parametrize("arch", sorted(SE_SITES))
def test_model_trains_and_evaluates_bit_identically(arch, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(arch)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert len(se_sites(fused)) == SE_SITES[arch]
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


FAMILIES = {"se_pool": r"b200c::se::k_se_pool", "se_scale": r"b200c::se::k_se_scale", "se_reduce": r"b200c::se::k_se_bwd_reduce",
            "se_elemt": r"b200c::se::k_se_bwd_elemt", "torch_reduce": r"at::native::reduce_kernel",
            "torch_mul": r"MulFunctor", "torch_add": r"CUDAFunctor(OnSelf|OnOther)?_add"}


def step_counts(model):
    """Per family, the kernels of the second of two bf16-autocast training steps of `model` at batch 4."""
    (x, y), = batches(4, 64)[:1]
    model.train()
    for _ in range(2):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.manual_seed(7)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {f: sum(bool(re.search(p, k)) for k in names) for f, p in FAMILIES.items()}


def trace_models():
    from torchvision.ops.misc import SqueezeExcitation

    got = {}
    for arch in SE_SITES:
        fused = fused_norm.fuse_model(make_model(arch))
        no_se = copy.deepcopy(fused)
        for m in no_se.modules():
            if type(m) is fused_norm.FusedSqueezeExcitation:
                m.__class__ = SqueezeExcitation
        got[arch] = {"sites": len(se_sites(fused)), "fused": step_counts(fused), "no_se": step_counts(no_se)}
    print(json.dumps(got))


@pytest.mark.gpu
def test_model_steps_run_four_native_kernels_and_no_full_size_torch_op_per_se_site():
    pytest.importorskip("torchvision")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", "import test_gpu_zz_se_models as t; t.trace_models()"], env=env, cwd=ROOT,
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    got = json.loads(out.stdout.strip().splitlines()[-1])
    for arch, c in got.items():
        n, fused, no_se = c["sites"], c["fused"], c["no_se"]
        assert n == SE_SITES[arch]
        for fam in ("se_pool", "se_scale", "se_reduce", "se_elemt"):
            assert fused[fam] == n and no_se[fam] == 0, (arch, fam, c)
        assert no_se["torch_reduce"] - fused["torch_reduce"] == 2 * n, (arch, c)
        assert no_se["torch_mul"] - fused["torch_mul"] == 4 * n, (arch, c)
        assert no_se["torch_add"] - fused["torch_add"] == n, (arch, c)
