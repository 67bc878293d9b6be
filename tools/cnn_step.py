#!/usr/bin/env python
"""Training step and eval forward of torchvision CNNs whose batch norms sit in Conv2dNormActivation blocks
(mobilenet_v2, mobilenet_v3_large, efficientnet_b0, efficientnet_v2_s, regnet_y_400mf), in DenseNet's dense layers
(densenet121, densenet161, densenet169, densenet201, by `--models` only) or in Inception's BasicConv2d blocks
(inception_v3 at 299 x 299 and googlenet, aux heads on, by `--models` only) or in ShuffleNetV2's blocks
(shufflenet_v2_x0_5, x1_0, x1_5, x2_0, by `--models` only) or in VGG-BN's stages (vgg11_bn, vgg16_bn, by `--models`
only), with and without
`fused_norm.fuse_model`.  The builds (`--builds`): "fused" (fuse_model), "unfused" (the untouched model), "act_only"
(fuse_model without the inverted-residual blocks' projection sites: only the Conv2dNormActivation sites are fused) and
"no_se" (fuse_model with the squeeze-excitation modules back on torchvision's class).

Batch `--batch` (256) at 224 x 224 (inception_v3: 299 x 299), bf16 autocast with fp32 parameters, channels-last, SGD
with momentum; the training loss sums the cross-entropies of the main and aux logits.  Per model,
alternating the builds in one process, `--runs` times each, the order reversed every run (ABBA):
  train_images_per_sec   `--iters` training steps between device events, after `--warmup` steps
  eval_images_per_sec    `--iters` forwards under inference_mode, the same way
All builds start from the same weights and train on the same batches, reseeded per step, so after the timed runs
their parameters and eval logits must have identical bits ("identical", each build against the first).  Then the host's time per training step
(forward and backward, no optimizer step): the wall time per step at batch `--host-batch` (4), where the GPU work is
too small to set the pace.  Then the peak of torch.cuda.max_memory_allocated over one training step, and, in a
separate profiled run per build, the kernel time per step by family.

Writes OUT/cnn_step.json; prints the summary.  The card's name and power limit are read in the same run.

  python tools/cnn_step.py --out DIR [--models a,b] [--builds fused,unfused] [--batch 256] [--runs 4] [--iters 10]
                           [--warmup 3] [--host-batch 4]
"""
import argparse
import copy
import json
import os
import re
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from step_profile import gpu_identity  # noqa: E402

MODELS = ["mobilenet_v2", "mobilenet_v3_large", "efficientnet_b0", "efficientnet_v2_s", "regnet_y_400mf"]
# first match wins
FAMILIES = [
    ("bn_shuffle", r"b200c::bn_shuffle::k_shuffle"),   # ShuffleNetV2's block ends, every direction but the statistics
    ("bn_pool2", r"b200c::bn_pool2::k_pool2"),       # VGG's stage ends, every direction but the statistics
    ("torch_max_pool", r"max_pool"),                  # torch's max_pool2d forward and backward
    ("bn_cat", r"b200c::bn_cat::k_cat"),             # DenseNet's concatenation sites, every direction
    ("bn_slice", r"b200c::bn_slice::k_slice"),       # Inception's slice sites, every direction but the statistics
    ("torch_cat", r"CatArrayBatchedCopy"),
    ("torch_copy", r"copy_kernel|direct_copy"),       # layout copies: channel_shuffle's .contiguous(), a gradient's reshape
    ("bn_stats", r"k_bn_stats|batch_norm_collect_statistics"),
    ("bn_transform_act", r"k_act_transform|k_act_infer|k_res_transform|k_res_infer|k_bn_transform|k_infer_transform"
                         r"|batch_norm_transform_input"),
    ("bn_bwd_reduce", r"k_act_bwd_reduce|k_res_bwd_reduce|k_bn_bwd_reduce|batch_norm_backward_reduce"),
    ("bn_bwd_elemt", r"k_act_bwd_elemt|k_bn_bwd_elemt|batch_norm_backward_elemt"),
    ("se", r"b200c::se::k_se"),
    ("torch_reduce", r"at::native::reduce_kernel"),   # torch's mean and sum (the squeeze-excitation's among them)
    ("torch_add_mul", r"CUDAFunctor_add|MulFunctor|bernoulli"),
    ("torch_act", r"silu|hardswish|hardsigmoid|clamp|hardtanh|threshold|relu"),
    ("conv", r"conv|cudnn|xmma|gemm|nvjet|cutlass|fprop|dgrad|wgrad|implicit_|nhwc|nchw|sm90_"),
]


# input size per model, where it is not 224
SIZES = {"inception_v3": 299}


def loss_of(out, y):
    """The cross-entropy of the main logits plus those of the aux heads (Inception v3, GoogLeNet) in training."""
    import torch
    import torch.nn.functional as F

    logits = [out] if isinstance(out, torch.Tensor) else [t for t in out if t is not None]
    return sum(F.cross_entropy(t.float(), y) for t in logits)


def family_of(name):
    for fam, pat in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", required=True)
    p.add_argument("--models", default=",".join(MODELS))
    p.add_argument("--builds", default="fused,unfused")
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--runs", type=int, default=4)
    p.add_argument("--iters", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--host-batch", type=int, default=4)
    args = p.parse_args()

    import torch
    import torch.nn.functional as F
    import torchvision
    from torch.profiler import ProfilerActivity, profile

    from ant_ray_b200 import fused_norm

    if not torch.cuda.is_available():
        raise SystemExit("cnn_step.py measures the GPU step: it needs a CUDA device")
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True   # the two builds' results are compared bit for bit
    device = torch.device("cuda", 0)
    g = torch.Generator(device=device).manual_seed(3)
    inputs = {}
    for size in {SIZES.get(a, 224) for a in args.models.split(",")}:
        inputs[size] = torch.randn(args.batch, 3, size, size, device=device, generator=g).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (args.batch,), device=device, generator=g)
    out = {**gpu_identity(), "batch": args.batch, "runs": args.runs, "iters": args.iters, "models": {}}

    for arch in args.models.split(","):
        x = inputs[SIZES.get(arch, 224)]
        torch.manual_seed(0)
        base = getattr(torchvision.models, arch)(weights=None).to(device).to(memory_format=torch.channels_last)
        builds = args.builds.split(",")
        models = {}
        for b in builds:
            m = copy.deepcopy(base)
            if b in ("fused", "act_only", "no_se"):
                fused_norm.fuse_model(m)
            if b == "no_se":   # the squeeze-excitation sites back to torchvision's class
                for mod in m.modules():
                    if type(mod) is fused_norm.FusedSqueezeExcitation:
                        mod.__class__ = fused_norm.SqueezeExcitation
            if b == "act_only":   # the projection sites' blocks back to torchvision's classes
                parents = {cls: parent for parent, cls in fused_norm._RES_SWAP.items()}
                for mod in m.modules():
                    if type(mod) in parents:
                        mod.__class__ = parents[type(mod)]
            models[b] = m
        opts = {b: torch.optim.SGD(m.parameters(), lr=0.01, momentum=0.9) for b, m in models.items()}
        steps = {b: 0 for b in models}

        def train_step(b):
            torch.manual_seed(1000 + steps[b])   # dropout and stochastic depth draw the same masks in both builds
            steps[b] += 1
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = loss_of(models[b](x), y)
            opts[b].zero_grad(set_to_none=True)
            loss.backward()
            opts[b].step()

        def forward(b):
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16):
                return models[b](x)

        def timed(b, fn):
            for _ in range(args.warmup):
                fn(b)
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(args.iters):
                fn(b)
            end.record()
            torch.cuda.synchronize()
            return round(args.batch * args.iters / (start.elapsed_time(end) / 1e3), 1)

        res = {b: {"train_images_per_sec": [], "eval_images_per_sec": []} for b in models}
        for r in range(args.runs):
            for b in (builds if r % 2 == 0 else builds[::-1]):   # alternating builds, ABBA
                models[b].train()
                res[b]["train_images_per_sec"].append(timed(b, train_step))
                models[b].eval()
                res[b]["eval_images_per_sec"].append(timed(b, forward))
        ints = {2: torch.int16, 4: torch.int32}
        same = lambda a, c: a.dtype == c.dtype and bool(torch.equal(a.view(ints[a.element_size()]), c.view(ints[c.element_size()])))  # noqa: E731
        first = models[builds[0]]
        entry = {"builds": res, "act_sites": len([m for m in first.modules() if type(m) is fused_norm.FusedConv2dNormActivation and len(m) == 3]),
                 "res_sites": len([m for m in first.modules() if type(m) in fused_norm._RES_SWAP.values()]),
                 "se_sites": len([m for m in first.modules() if type(m) is fused_norm.FusedSqueezeExcitation]),
                 "identical": {b: {"parameters": all(same(a, c) for a, c in zip(models[b].parameters(), first.parameters())),
                                   "buffers": all(same(a, c) for a, c in zip(models[b].buffers(), first.buffers()) if a.is_floating_point()),
                                   "eval_logits": same(forward(b), forward(builds[0]))} for b in builds[1:]}}
        # host time: at batch `--host-batch` the GPU work is small, so a step's wall time is what the host needs to issue it
        xs, ys = x[:args.host_batch].clone(), y[:args.host_batch].clone()

        def host_step(b):
            torch.manual_seed(0)
            with torch.autocast("cuda", dtype=torch.bfloat16):
                loss = loss_of(models[b](xs), ys)
            opts[b].zero_grad(set_to_none=True)
            loss.backward()

        host = {b: [] for b in models}
        for r in range(args.runs):
            for b in (builds if r % 2 == 0 else builds[::-1]):
                models[b].train()
                for _ in range(args.warmup):
                    host_step(b)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    host_step(b)
                torch.cuda.synchronize()
                host[b].append(round((time.perf_counter() - t0) / args.iters * 1e3, 2))
        entry["host_ms_per_step"] = {"batch": args.host_batch, **host}
        peak = {}
        for b in models:
            models[b].train()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            train_step(b)
            torch.cuda.synchronize()
            peak[b] = torch.cuda.max_memory_allocated()
        entry["peak_train_bytes"] = peak
        profiled = {}
        for b in models:
            models[b].train()
            for _ in range(args.warmup):
                train_step(b)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    train_step(b)
                torch.cuda.synchronize()
            fams = {}
            for ev in prof.key_averages():
                t = getattr(ev, "self_device_time_total", None)
                if t is None:
                    t = ev.self_cuda_time_total
                if t > 0:
                    fam = family_of(ev.key)
                    fams[fam] = fams.get(fam, 0.0) + t / args.iters / 1e3
            profiled[b] = {"kernel_ms_per_step": round(sum(fams.values()), 3),
                           "families_ms_per_step": {k: round(v, 3) for k, v in sorted(fams.items(), key=lambda kv: -kv[1])}}
        entry["profile"] = profiled
        out["models"][arch] = entry
        del models, opts, base
        torch.cuda.empty_cache()

    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "cnn_step.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
