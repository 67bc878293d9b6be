#!/usr/bin/env python
"""What the sync batch-norm path costs and saves.  Writes OUT/syncbn_<mode>.json; reads the card's name and power
limit in the same run.

  python tools/syncbn_step.py --mode step  --out DIR [--torch-bn] [--batch 256] [--steps 20] [--warmup 5]
      ResNet-50 converted with nn.SyncBatchNorm.convert_sync_batchnorm, bf16 autocast, channels-last, SGD momentum,
      through train.prepare_model: images/s (CUDA events) and the kernel-family table of tools/step_profile.py
      (a profiled run of its own).  Under torchrun with WORLD_SIZE > 1 the SyncBatchNorm layers sync over peer
      memory; also counts NCCL kernels per step.  --torch-bn keeps torch's own SyncBatchNorm (NCCL at world size > 1,
      F.batch_norm at 1) for the comparison.  --dump-outputs DIR writes the last timed step's loss and a fixed, seeded
      sample of 2^20 parameter values as .npy files, to compare two builds (as bench.py --dump-outputs does).
  python tools/syncbn_step.py --mode sites --world W --out DIR
      Loopback world of W ranks on one GPU: microseconds per ResNet-50 batch-norm site (forward + backward, ReLU
      site, global batch 256 split evenly) on the sync path, next to the local fused site of one rank's shape.  The
      exchange here is local HBM traffic, not NVLink.
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

CL = torch.channels_last
SHAPES = [(64, 112, 112), (256, 56, 56), (512, 28, 28), (1024, 14, 14), (2048, 7, 7)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def families(prof):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import re

    from step_profile import FAMILIES

    # bn_sync: the sync statistics and merge kernels only; a sync site's transform, backward reduce and backward
    # elementwise kernels are the local sites' and count in their families
    fams = [("bn_sync", r"k_bn_sync_(stats|merge)")] + FAMILIES
    out = {}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA and not getattr(e, "self_device_time_total", 0):
            continue
        us = getattr(e, "self_device_time_total", 0) or getattr(e, "self_cuda_time_total", 0)
        fam = next((f for f, pat in fams if re.search(pat, e.key)), "other")
        out[fam] = out.get(fam, 0.0) + us / 1000.0
    return out


def step_mode(args):
    import torchvision

    from ant_ray_b200 import train

    dist = None
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        import torch.distributed as dist

        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl")
    torch.backends.cudnn.benchmark = False
    torch.manual_seed(0)   # the same initial model in every run, so that two builds' dumps can be compared
    model = nn.SyncBatchNorm.convert_sync_batchnorm(torchvision.models.resnet50()).cuda().to(memory_format=CL)
    if args.torch_bn:
        if dist is not None:
            model = nn.parallel.DistributedDataParallel(model)
    else:
        model = train.prepare_model(model)
    opt = torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(args.batch, 3, 224, 224, device="cuda", generator=g).contiguous(memory_format=CL)
    y = torch.randint(0, 1000, (args.batch,), device="cuda", generator=g)

    def one():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x), y)
        loss.backward()
        opt.step()
        return loss

    for _ in range(args.warmup):
        one()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        loss = one()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    if args.dump_outputs:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        flat = torch.cat([p.detach().float().flatten() for p in model.parameters()]).cpu()
        idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:1 << 20]
        np.save(os.path.join(args.dump_outputs, "loss.npy"), loss.detach().float().cpu().numpy())
        np.save(os.path.join(args.dump_outputs, "params_sample.npy"), flat[idx].numpy())
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        one()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    res = {"mode": "step", "torch_bn": args.torch_bn, "world_size": dist.get_world_size() if dist else 1,
           "batch_per_gpu": args.batch, "ms_per_step": ms, "images_per_s": args.batch * (dist.get_world_size() if dist else 1) / ms * 1e3,
           "loss": float(loss), "nccl_kernels_per_step": sum("nccl" in n.lower() for n in names),
           "families_ms": families(prof), "gpu": card()}
    return res


def sites_mode(args):
    from ant_ray_b200 import fused_norm
    from ant_ray_b200.loopback import LoopbackWorld

    W = args.world
    relu = nn.ReLU(inplace=True)
    t = torch.zeros(8, 8, 2, 2, dtype=torch.bfloat16, device="cuda")
    torch.zeros(16, dtype=torch.uint8, device="cuda")
    torch.zeros_like(t, memory_format=CL)
    world = LoopbackWorld(W, device=0, key=f"syncbn-sites{W}", staging_bytes=1 << 20, max_blocks=8)
    out = []
    try:
        for c, h, w in SHAPES:
            n = 256 // W
            x = torch.randn(n, c, h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=CL).requires_grad_()
            dy = torch.randn_like(x)
            base = nn.SyncBatchNorm(c).cuda()
            reps = [fused_norm.sync_batch_norm(copy.deepcopy(base), world.comms[r]) for r in range(W)]
            local = copy.deepcopy(base)

            def sync_site(r, comm):
                fused_norm.bn_relu(reps[r], relu, x).backward(dy)

            def local_site():
                fused_norm.bn_relu(local, relu, x).backward(dy)

            def timed(fn, iters=20):
                for _ in range(3):
                    fn()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / iters * 1e3

            us_local = timed(local_site)   # first: it also loads the torch kernels the sync sites use (lazy loading)
            us_sync = timed(lambda: world.run(sync_site))
            world.check()
            out.append({"c": c, "h": h, "w": w, "images_per_rank": n, "us_sync_all_ranks": us_sync, "us_local_one_rank": us_local})
    finally:
        torch.cuda.synchronize()
        world.destroy()
    return {"mode": "sites", "world_size": W, "sites": out, "gpu": card(),
            "note": "us_sync_all_ranks: forward + backward of all W ranks' sites, which share one GPU"}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--mode", choices=["step", "sites"], required=True)
    p.add_argument("--out", required=True)
    p.add_argument("--torch-bn", action="store_true")
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--world", type=int, default=2)
    p.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = p.parse_args()
    if not torch.cuda.is_available():
        sys.exit("syncbn_step.py measures on a GPU; there is none here")
    res = step_mode(args) if args.mode == "step" else sites_mode(args)
    os.makedirs(args.out, exist_ok=True)
    tag = args.mode + ("_torchbn" if args.torch_bn else "") + (f"_w{args.world}" if args.mode == "sites" else "")
    with open(os.path.join(args.out, f"syncbn_{tag}.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k not in ("families_ms", "sites")}))


if __name__ == "__main__":
    main()
