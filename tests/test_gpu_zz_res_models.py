"""Whole torchvision models with fused inverted-residual projection sites (fused_norm.bn_res) against the untouched
models, bit for bit: mobilenet_v2, mobilenet_v3_large and efficientnet_b0 (num_classes 10, 96 x 96) after `fuse_model`
and after `prepare_model`, three reseeded SGD-momentum steps under bf16 autocast, channels-last, with EfficientNet's
stochastic depth active (p raised to 0.5 so that rows are dropped at batch 8), then an eval forward under
inference_mode.  Losses, gradients, parameters, buffers and logits must have the same bits.

Two profiler traces, each in a process of its own (test_gpu_zz_infer_trace.py explains why): a fused training step
launches one projection site per projection batch norm (`b200c::bn_res` with an identity, the plain `b200c::bn` site
without), and the torch batch-norm kernels left in it are exactly the model's unfused batch norms (mobilenet_v3_large's
ReLU blocks) plus, in the backward, the sites whose gradient arrived in NCHW, both counted from the model.  Every
`b200c::bn_res` kernel is launched by the case test_gpu_fused_res.KERNELS gives it."""
import copy
import json
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from ant_ray_b200 import fused_norm, train
from gpu_common import same_bits
from test_gpu_fused_res import KERNELS
from test_gpu_zz_act_models import batches, mismatches, train_steps
from test_gpu_zz_act_models import make_model as make_act_model

CL = torch.channels_last
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODELS = ["mobilenet_v2", "mobilenet_v3_large", "efficientnet_b0"]


@pytest.fixture(scope="module")
def deterministic_cudnn():
    saved = torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = False, True
    yield
    torch.backends.cudnn.benchmark, torch.backends.cudnn.deterministic = saved


def make_model(arch):
    model = make_act_model(arch)
    for m in model.modules():
        if type(m).__name__ == "StochasticDepth":
            m.p = 0.5
    return model


def res_sites(model):
    return [m for m in model.modules() if type(m) in fused_norm._RES_SWAP.values()]


@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["fuse_model", "prepare_model"])
@pytest.mark.parametrize("arch", MODELS)
def test_model_trains_and_evaluates_bit_identically(arch, entry, deterministic_cudnn):
    pytest.importorskip("torchvision")
    base = make_model(arch)
    data = batches()
    ref = copy.deepcopy(base)
    want = train_steps(ref, data)
    fused = copy.deepcopy(base)
    fused = fused_norm.fuse_model(fused) if entry == "fuse_model" else train.prepare_model(fused, parallel_strategy=None)
    assert len(res_sites(fused)) == {"mobilenet_v2": 17, "mobilenet_v3_large": 15, "efficientnet_b0": 16}[arch]
    got = train_steps(fused, data)
    torch.cuda.synchronize()
    assert all(same_bits(a, b) for a, b in zip(got[0], want[0])), "losses differ"
    grads = lambda m: [(k, p.grad) for k, p in m.named_parameters()]
    assert not mismatches(grads(fused), grads(ref)), "gradients differ"
    assert not mismatches(fused.named_parameters(), ref.named_parameters()), "parameters differ"
    assert not mismatches(fused.named_buffers(), ref.named_buffers()), "buffers differ"
    assert same_bits(got[1], want[1]), "eval logits differ"


def model_trace_counts(arch):
    """Per family, the kernels one bf16-autocast training step (forward and backward) of the fused model launches, the
    model's projection sites with and without an identity, its batch norms on no fused site, and how many fused sites
    received their gradient in NCHW."""
    model = fused_norm.fuse_model(make_model(arch)).train()
    (x, y), = batches(4, 64)[:1]
    families = {"res_transform": r"b200c::bn_res::k_res_transform", "res_reduce": r"b200c::bn_res::k_res_bwd_reduce",
                "plain_transform": r"k_bn_transform<\d+, \(b200c::bn::Tail\)0>",
                "plain_reduce": r"k_bn_bwd_reduce<\(b200c::bn::GradSrc\)3, false>",
                "torch_bn_stats": r"batch_norm_collect_statistics",
                "torch_bn_backward": r"batch_norm_backward_reduce|batch_norm_backward_kernel"}
    nchw = []   # per fused site and step: whether its output's gradient arrived in another layout than channels-last

    def record(mod, inputs, out):
        out.register_hook(lambda g: nchw.append(not g.is_contiguous(memory_format=CL)))

    acts = [m for m in model.modules() if type(m) is fused_norm.FusedConv2dNormActivation]
    for m in acts + res_sites(model):   # a block's own hook keeps the block fused
        m.register_forward_hook(record)
    for step in range(2):   # the second step is traced
        nchw.clear()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            torch.manual_seed(7)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = F.cross_entropy(model(x).float(), y)
            loss.backward()
            torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    counts = {f: sum(bool(re.search(p, k)) for k in names) for f, p in families.items()}
    fused_bns = {id(m[1]) for m in acts}
    for b in res_sites(model):
        proj = b.conv if type(b) is fused_norm.FusedInvertedResidualV2 else b.block[-1]
        fused_bns.add(id(proj[-1]))
    counts["res_sites"] = sum(b.use_res_connect for b in res_sites(model))
    counts["plain_sites"] = sum(not b.use_res_connect for b in res_sites(model))
    counts["unfused_bns"] = sum(isinstance(m, nn.BatchNorm2d) and id(m) not in fused_bns for m in model.modules())
    counts["nchw_gradient_sites"] = sum(nchw)
    return counts


def trace_models():
    print(json.dumps({arch: model_trace_counts(arch) for arch in MODELS}))


def run_traced(code):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return json.loads(out.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
def test_model_steps_run_one_native_site_per_projection_batch_norm():
    pytest.importorskip("torchvision")
    got = run_traced("import test_gpu_zz_res_models as t; t.trace_models()")
    for arch, c in got.items():
        assert c["res_transform"] == c["res_sites"] and c["plain_transform"] == c["plain_sites"], (arch, c)
        # the projection batch norms' gradients arrive from the next convolution, in channels-last; only a site with
        # stochastic depth (EfficientNet's residual blocks) needs k_res_bwd_reduce, the others reduce dy itself
        assert c["res_reduce"] + c["plain_reduce"] == c["res_sites"] + c["plain_sites"], (arch, c)
        assert c["res_reduce"] == (c["res_sites"] if arch == "efficientnet_b0" else 0), (arch, c)
        assert c["torch_bn_stats"] == c["unfused_bns"], (arch, c)
        assert c["torch_bn_backward"] == c["unfused_bns"] + c["nchw_gradient_sites"], (arch, c)
    assert got["mobilenet_v3_large"]["unfused_bns"] > 0 and got["mobilenet_v2"]["unfused_bns"] == 0


@pytest.mark.gpu
def test_every_res_kernel_is_launched_by_its_case():
    launched = run_traced("import test_gpu_fused_res as t; t.trace_cases()")
    assert set(launched) == set(KERNELS.values())
    missing = {k: case for k, case in KERNELS.items() if k not in launched[case]}
    assert not missing, f"kernels their case did not launch: {missing}"
    unknown = {k for names in launched.values() for k in names} - set(KERNELS)
    assert not unknown, f"launched kernels missing from KERNELS: {unknown}"
