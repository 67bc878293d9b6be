#!/usr/bin/env python
"""Where the GPU time of bench.py's headline step goes: ResNet-50, DDP at world size 1 with the fused gradient
hook, bf16 autocast, SGD momentum, channels-last, cuDNN heuristics (no autotuning), built exactly as bench.py builds it.

Writes OUT/step_profile_<fused|unfused>.json:
  ms_per_step            CUDA events around `--steps` steps (profiler off)
  families               kernel time per step per family from torch.profiler (CUDA activity, a run of its own),
                         with the largest kernels of each family by name
  bytes / GB/s           for the memory-bound families: the bytes their kernels must move per step, computed from
                         the shapes of the 53 batch-norm sites, and the rate this implies
  gpu, power_limit_w     read in the same run

  python tools/step_profile.py --out DIR [--unfused] [--batch 256] [--steps 10] [--warmup 5]

--unfused builds the model without fused_norm's rewrite (torch's own batch norm, ReLU and add), so that two runs
of one session can compare the two.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# first match wins: convolutions before anything that may share a word with a fused cuDNN kernel name
FAMILIES = [
    ("hook", r"b200c::k_(local|allreduce)"),
    ("bn_stats", r"k_bn_stats"),                          # ours; torch's kernels (downsample sites, --unfused): *_torch
    ("bn_stats_torch", r"batch_norm_collect_statistics"),
    ("bn_update_invert", r"batch_norm_update_stats"),
    ("bn_transform", r"batch_norm_transform_input|k_bn_transform"),
    ("bn_pool", r"k_bn_pool_fwd"),                        # ours: the stem's transform, ReLU and max-pool forward
    ("max_pool", r"max_pool"),                            # torch's (before conv: its kernels' names say nhwc)
    ("bn_bwd_reduce", r"k_bn_bwd_reduce"),
    ("bn_bwd_reduce_torch", r"batch_norm_backward_reduce"),
    ("bn_bwd_elemt", r"batch_norm_backward_elemt|k_bn_bwd_elemt"),
    ("conv", r"conv|cudnn|xmma|gemm|nvjet|cutlass|dgrad|wgrad|fprop|implicit_|nhwc|nchw"),
    ("threshold_backward", r"threshold"),
    ("relu", r"clamp|relu"),
    ("add", r"add|Add"),
    ("optimizer", r"multi_tensor|sgd|SGD|foreach"),
]

# bytes each family's kernels move per element of a batch-norm site, by site kind (stem: BN -> ReLU -> 3x3 / 2
# max-pool, a quarter as many pooled elements; relu: BN -> ReLU; tail: BN -> += identity -> ReLU whose output feeds
# another block; ds_tail: such a tail whose identity is a downsample branch; last_tail: the tail that feeds the
# pooling; plain: the downsample branch's BN, which the fused build runs inside the ds_tail's kernels)
TORCH_BYTES = {  # family -> {kind: bytes per element}
    "bn_stats_torch": {"stem": 2, "relu": 2, "tail": 2, "last_tail": 2, "plain": 2},
    "bn_transform": {"stem": 4, "relu": 4, "tail": 4, "last_tail": 4, "plain": 4},
    "relu": {"stem": 4, "relu": 4, "tail": 4, "last_tail": 4},
    "max_pool": {"stem": 9},   # y -> pooled, int64 indices; indices, dpool -> dy
    "add": {"tail": 6, "ds_tail": 6, "last_tail": 6},
    "threshold_backward": {"stem": 6, "relu": 6, "tail": 6, "ds_tail": 6, "last_tail": 6},
    "bn_bwd_reduce_torch": {"stem": 4, "relu": 4, "tail": 4, "ds_tail": 4, "last_tail": 4, "plain": 4},
    "bn_bwd_elemt": {"stem": 6, "relu": 6, "tail": 6, "ds_tail": 6, "last_tail": 6, "plain": 6},
}
for _fam in ("bn_stats_torch", "bn_transform", "relu"):
    TORCH_BYTES[_fam]["ds_tail"] = TORCH_BYTES[_fam]["tail"]
# the fused sites' ReLU mask is 1 bit (1/8 byte) per element; the stem's argmax is 1 byte per pooled element
# (ds_tail: the identity read is the branch's input, and the backward writes no g: the elementwise kernel reads dy,
# dy2 and the mask again; plain: the branch's input read by each kernel, its dx written)
FUSED_BYTES = {
    "bn_stats": {"stem": 2, "relu": 2, "tail": 2, "ds_tail": 2, "last_tail": 2, "plain": 2},
    "bn_transform": {"relu": 4.125, "tail": 6.125, "ds_tail": 6.125, "last_tail": 6.125},   # x (, identity) -> y, mask
    "bn_pool": {"stem": 2.75},                                                              # x -> pooled, argmax
    # stem: dpool, argmax, x -> g; others: dy (, dy2), mask, x (tail: -> dy')
    "bn_bwd_reduce": {"stem": 4.75, "relu": 4.125, "tail": 8.125, "ds_tail": 6.125, "last_tail": 6.125, "plain": 2},
    # dy, mask, x -> dx (tail, stem: g, x -> dx; ds_tail: dy, dy2, mask, x -> dx)
    "bn_bwd_elemt": {"stem": 6, "relu": 6.125, "tail": 6, "ds_tail": 8.125, "last_tail": 6, "plain": 4},
}


def bn_sites(batch):
    """(kind, elements) of every batch norm of resnet50 at this batch, from one CPU forward at batch 1."""
    import torch
    import torchvision

    model = torchvision.models.resnet50(weights=None).eval()
    kinds = {id(model.bn1): "stem"}
    for mod in model.modules():
        if isinstance(mod, torchvision.models.resnet.Bottleneck):
            kinds.update({id(mod.bn1): "relu", id(mod.bn2): "relu", id(mod.bn3): "tail"})
            if mod.downsample is not None:
                kinds.update({id(mod.bn3): "ds_tail", id(mod.downsample[1]): "plain"})
    kinds[id(model.layer4[-1].bn3)] = "last_tail"
    sites = []
    hooks = [m.register_forward_pre_hook(lambda m, a: sites.append((kinds[id(m)], a[0].numel() * batch)))
             for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        model(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    assert len(sites) == 53, len(sites)
    return sites


def family_of(name):
    for fam, pat in FAMILIES:
        if re.search(pat, name):
            return fam
    return "other"


def gpu_identity():
    import torch

    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["sm_max_mhz"] = float(q[0]), float(q[1])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        out["power_limit_w"] = None
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", required=True)
    p.add_argument("--unfused", action="store_true")
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=5)
    args = p.parse_args()

    import torch
    import torch.distributed as dist
    from torch.profiler import ProfilerActivity, profile

    import bench
    from ant_ray_b200 import fused_norm
    from ant_ray_b200 import train as b200_train

    if not torch.cuda.is_available():
        raise SystemExit("step_profile.py measures the GPU step: it needs a CUDA device")
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29541")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    dist.init_process_group("nccl", rank=0, world_size=1, device_id=device)
    torch.backends.cudnn.benchmark = False

    model = b200_train.prepare_model(bench.build_model(device), grad_wire="bf16", wrap_single=True)
    if args.unfused:  # back to torchvision's own classes
        fused_classes = set(fused_norm._SWAP.values())
        for mod in model.modules():
            if type(mod) in fused_classes:
                mod.__class__ = type(mod).__mro__[1]
    state = model.b200_grad_state
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.9)
    step = bench.make_step(model, opt, True, device)
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(args.batch, 3, 224, 224, generator=g).contiguous(memory_format=torch.channels_last).to(device)
    y = torch.randint(0, 1000, (args.batch,), generator=g).to(device)
    for _ in range(args.warmup):
        step(x, y)
    ms, _, _ = bench.timed_steps(step, x, y, args.steps, dist, 1)

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step(x, y)
        torch.cuda.synchronize()
    per_family, names = {}, {}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = ev.self_cuda_time_total
        if t <= 0:
            continue
        fam = family_of(ev.key)
        per_family[fam] = per_family.get(fam, 0.0) + t / args.steps / 1e3
        names.setdefault(fam, []).append((t / args.steps / 1e3, ev.key[:160], ev.count // args.steps))

    table = FUSED_BYTES if not args.unfused else TORCH_BYTES
    sites = bn_sites(args.batch)
    total = sum(per_family.values())
    fams = {}
    for fam in sorted(per_family, key=per_family.get, reverse=True):
        entry = {"ms_per_step": round(per_family[fam], 3), "share": round(per_family[fam] / total, 4),
                 "top_kernels": [{"ms": round(t, 3), "launches_per_step": c, "name": n}
                                 for t, n, c in sorted(names[fam], reverse=True)[:4]]}
        if fam in table:
            nbytes = sum(table[fam].get(kind, 0) * e for kind, e in sites)
            entry["bytes_per_step"] = nbytes
            entry["gb_per_s"] = round(nbytes / (per_family[fam] * 1e-3) / 1e9, 1)
        fams[fam] = entry
    out = {"mode": "unfused" if args.unfused else "fused", "batch": args.batch, "steps": args.steps,
           "ms_per_step": round(ms / args.steps, 3), "kernel_ms_per_step": round(total, 3),
           "images_per_sec": round(args.batch * args.steps / (ms / 1e3), 1), **gpu_identity(), "families": fams,
           "bn_site_elements": {k: sum(e for kind, e in sites if kind == k) for k in ("stem", "relu", "tail", "ds_tail", "last_tail", "plain")}}
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, f"step_profile_{out['mode']}.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({k: v for k, v in out.items() if k != "families"}))
    print(json.dumps({k: (v["ms_per_step"], v.get("gb_per_s")) for k, v in fams.items()}))
    state.comm.destroy()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
