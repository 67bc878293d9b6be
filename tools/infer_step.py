#!/usr/bin/env python
"""ResNet-50 eval forward under torch.inference_mode(), channels-last, with and without fused_norm's eval sites.

Two setups: (a) "autocast": bf16 autocast with fp32 parameters; (b) "bf16_model": the model cast to bf16.  For each
setup and each build ("fused": `fuse_resnet` applied; "unfused": torchvision's own classes), alternating the builds
in one process, `--runs` times each:
  images_per_sec         at batch 256 (`--iters` forwards between device events, after a synchronise)
  ms_per_forward         at batch 1 and 32, the same way
Then, per setup: whether the two builds' logits have identical bits at each batch, and in a separate profiled run
at batch 256 the kernel time per family per forward and the bytes the batch-norm sites move per forward (computed
from the shapes of resnet50's 53 batch norms and the byte model below).

Writes OUT/infer_step.json; prints the summary.  The card's name and power limit are read in the same run.

  python tools/infer_step.py --out DIR [--runs 3] [--iters 20] [--warmup 5] [--unfused]

--unfused measures the unfused build alone.
"""
import argparse
import copy
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from step_profile import bn_sites, gpu_identity  # noqa: E402

# first match wins
FAMILIES = [
    ("bn_infer", r"b200c::bn_infer::"),
    ("bn_transform_torch", r"batch_norm_transform_input"),
    ("bn_invstd_torch", r"batch_norm_calc_invstd"),
    ("max_pool", r"max_pool"),
    ("conv", r"conv|cudnn|xmma|gemm|nvjet|cutlass|fprop|implicit_|nhwc|nchw"),
    ("relu", r"clamp|relu"),
    ("add", r"CUDAFunctor_add"),
    ("copy", r"copy"),
]

# Bytes per element of a site's activation (bf16), by site kind.  torch: relu = transform read + write, ReLU read +
# write; tail = transform 4, add 6, ReLU 4; ds_tail = two transforms 8, add 6, ReLU 4 (the downsample's batch norm
# included); stem = transform 4, ReLU 4, max-pool read 2 + a quarter-size output 0.5 + int64 indices 2.  fused: the
# kernel reads x (and the identity or x_ds) and writes y, or the pooled output at the stem.
BYTES = {"unfused": {"stem": 12.5, "relu": 8, "tail": 14, "last_tail": 14, "ds_tail": 18},
         "fused": {"stem": 2.5, "relu": 4, "tail": 6, "last_tail": 6, "ds_tail": 6}}


def family_of(name):
    for fam, pat in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def same_bits(a, b):
    import torch

    ints = {2: torch.int16, 4: torch.int32}
    return a.dtype == b.dtype and a.shape == b.shape and bool(torch.equal(a.view(ints[a.element_size()]), b.view(ints[b.element_size()])))


def site_bytes(build, batch):
    # the downsample branch's batch norm ("plain") belongs to its ds_tail, whose element count is the same
    return sum(BYTES[build].get(kind, 0) * e for kind, e in bn_sites(batch))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", required=True)
    p.add_argument("--runs", type=int, default=3)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--unfused", action="store_true")
    args = p.parse_args()

    import torch
    import torchvision
    from torch.profiler import ProfilerActivity, profile

    from ant_ray_b200 import fused_norm

    if not torch.cuda.is_available():
        raise SystemExit("infer_step.py measures the GPU forward: it needs a CUDA device")
    torch.backends.cudnn.benchmark = False
    device = torch.device("cuda", 0)
    torch.manual_seed(0)
    base = torchvision.models.resnet50(weights=None).to(device).to(memory_format=torch.channels_last).eval()
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():   # non-trivial running statistics and affine parameters
        for m in base.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                c = m.num_features
                m.weight.copy_(1 + 0.2 * torch.randn(c, generator=g))
                m.bias.copy_(0.2 * torch.randn(c, generator=g))
                m.running_mean.copy_(0.1 * torch.randn(c, generator=g))
                m.running_var.copy_(1 + 0.1 * torch.rand(c, generator=g))
    builds = ["unfused"] if args.unfused else ["fused", "unfused"]
    inputs = {b: torch.randn(b, 3, 224, 224, generator=torch.Generator().manual_seed(b)).contiguous(memory_format=torch.channels_last)
              .to(device) for b in (1, 32, 256)}
    out = {**gpu_identity(), "runs": args.runs, "iters": args.iters, "setups": {}}

    for setup in ("autocast", "bf16_model"):
        ref = base if setup == "autocast" else copy.deepcopy(base).to(torch.bfloat16)
        models = {"unfused": ref}
        if "fused" in builds:
            models["fused"] = fused_norm.fuse_resnet(copy.deepcopy(ref))
        dtype = torch.float32 if setup == "autocast" else torch.bfloat16
        xs = {b: x.to(dtype) for b, x in inputs.items()}

        def forward(model, x):
            with torch.inference_mode(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=setup == "autocast"):
                return model(x)

        def timed(model, x, iters):
            for _ in range(args.warmup):
                forward(model, x)
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(iters):
                forward(model, x)
            end.record()
            torch.cuda.synchronize()
            return start.elapsed_time(end) / iters

        res = {b: {"images_per_sec": [], "ms_per_forward_b1": [], "ms_per_forward_b32": []} for b in builds}
        for _ in range(args.runs):
            for b in builds:   # alternating builds
                res[b]["images_per_sec"].append(round(256 / (timed(models[b], xs[256], args.iters) / 1e3), 1))
                res[b]["ms_per_forward_b32"].append(round(timed(models[b], xs[32], 2 * args.iters), 3))
                res[b]["ms_per_forward_b1"].append(round(timed(models[b], xs[1], 5 * args.iters), 3))
        entry = {"builds": res}
        if "fused" in builds:
            entry["identical_logits"] = {str(b): same_bits(forward(models["fused"], x), forward(models["unfused"], x))
                                         for b, x in xs.items()}
        profiled = {}
        for b in builds:
            for _ in range(args.warmup):
                forward(models[b], xs[256])
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    forward(models[b], xs[256])
                torch.cuda.synchronize()
            fams = {}
            for ev in prof.key_averages():
                t = getattr(ev, "self_device_time_total", None)
                if t is None:
                    t = ev.self_cuda_time_total
                if t > 0:
                    fam = family_of(ev.key)
                    fams[fam] = fams.get(fam, 0.0) + t / args.iters / 1e3
            profiled[b] = {"kernel_ms_per_forward": round(sum(fams.values()), 3),
                           "families_ms_per_forward": {k: round(v, 3) for k, v in sorted(fams.items(), key=lambda kv: -kv[1])},
                           "bn_site_bytes_per_forward": site_bytes(b, 256)}
        entry["profile_batch256"] = profiled
        out["setups"][setup] = entry

    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "infer_step.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
