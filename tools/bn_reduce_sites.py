#!/usr/bin/env python
"""Per-site time of the batch-norm statistics and backward-reduce kernels at ResNet-50's shapes, through the C-ABI.

Every batch-norm shape of resnet50 at `--batch` runs as the kind of site the fused model makes of it:
  relu       statistics (k_bn_stats); reduce from dy and the ReLU mask bits
  tail       statistics; reduce from dy, dy2 and the mask bits, writing g
  last_tail  statistics; reduce from dy and the mask bits, writing g (the tail that feeds the pooling)
  ds_tail    the tail and its downsample branch's batch norm: k_bn_stats_dual and the dual reduce, dy2 and mask bits
  stem       the stem's shape run as a relu site (the stem's own reduce gathers through the pooling instead)

Each library given with --lib (the first is the reference; add the parent build's to compare) runs `--iters`
back-to-back forward and backward calls per site, rotating over two buffer sets so that every call reads from HBM
(each operand is at least 51 MB at batch 256, the H100's L2 is 50 MB).  The libraries alternate in rounds in one
process.  The C-ABI launches the statistics kernel with the transform and the reduce with the backward elementwise
kernel, so each kernel's device time is taken from torch.profiler's CUDA kernel records of the timed calls.

Reports per site and library: µs per call of the statistics and reduce kernels (median over rounds), GB/s from
tools/step_profile.py's byte model, the per-step totals weighted by how often each shape occurs, and whether every
library wrote the same bits (statistics, running statistics, dweight, dbias, g) as the first.  The card name and
power limit are read in the same run.

  python tools/bn_reduce_sites.py --lib ant-ray_b200/libb200coll.so [--lib OTHER.so] --out DIR [--rounds 3] [--iters 20]
"""
import argparse
import collections
import ctypes
import hashlib
import json
import os
import statistics
import sys
from ctypes import c_float, c_int, c_size_t, c_void_p

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from tools.step_profile import FUSED_BYTES, gpu_identity  # noqa: E402

# bytes per element of each site kind, by family: step_profile's model (a ds_tail's kernels also carry its
# downsample branch's batch norm, the "plain" kind there); the stem runs here as a relu site
STATS_BYTES = {k: FUSED_BYTES["bn_stats"]["relu" if k == "stem" else k] for k in ("stem", "relu", "tail", "last_tail", "ds_tail")}
STATS_BYTES["ds_tail"] += FUSED_BYTES["bn_stats"]["plain"]
REDUCE_BYTES = {k: FUSED_BYTES["bn_bwd_reduce"]["relu" if k == "stem" else k] for k in ("stem", "relu", "tail", "last_tail", "ds_tail")}
REDUCE_BYTES["ds_tail"] += FUSED_BYTES["bn_bwd_reduce"]["plain"]


def resnet50_sites(batch):
    """{(kind, m, c): count} of resnet50's batch norms at this batch, the downsample branches inside their ds_tail."""
    import torch
    import torchvision

    model = torchvision.models.resnet50(weights=None).eval()
    kinds = {id(model.bn1): "stem"}
    for mod in model.modules():
        if isinstance(mod, torchvision.models.resnet.Bottleneck):
            kinds.update({id(mod.bn1): "relu", id(mod.bn2): "relu", id(mod.bn3): "tail"})
            if mod.downsample is not None:
                kinds.update({id(mod.bn3): "ds_tail", id(mod.downsample[1]): None})
    kinds[id(model.layer4[-1].bn3)] = "last_tail"
    sites = collections.Counter()
    hooks = [m.register_forward_pre_hook(lambda m, a: kinds[id(m)] and sites.update([(kinds[id(m)], batch * a[0].shape[2] * a[0].shape[3], a[0].shape[1])]))
             for m in model.modules() if isinstance(m, torch.nn.BatchNorm2d)]
    with torch.no_grad():
        model(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    assert sum(sites.values()) == 49, sites
    return dict(sites)


def bind(path):
    lib = ctypes.CDLL(os.path.abspath(path), mode=ctypes.RTLD_LOCAL)
    P, I, F = c_void_p, c_int, c_float
    lib.b200c_bn_scratch_bytes.restype = c_size_t
    lib.b200c_bn_dual_scratch_bytes.restype = c_size_t
    lib.b200c_bn_scratch_bytes.argtypes = lib.b200c_bn_dual_scratch_bytes.argtypes = [I]
    lib.b200c_bn_forward_mask.argtypes = [P] * 11 + [I, I, F, F, P, P]
    lib.b200c_bn_backward_mask.argtypes = [P] * 11 + [I, I, P, P]
    lib.b200c_bn_forward_dual.argtypes = [P] * 11 + [F, F] + [P] * 7 + [F, F, I, I, P, P]
    lib.b200c_bn_backward_dual.argtypes = [P] * 18 + [I, I, P, P]
    for f in ("b200c_bn_forward_mask", "b200c_bn_backward_mask", "b200c_bn_forward_dual", "b200c_bn_backward_dual"):
        getattr(lib, f).restype = c_int
    return lib


class Site:
    """Two buffer sets of one site and the C-ABI calls of one forward and one backward on set `i`."""

    def __init__(self, kind, m, c, seed):
        import torch

        self.kind, self.m, self.c = kind, m, c
        g = torch.Generator(device="cuda").manual_seed(seed)
        dual = kind == "ds_tail"

        def act():
            return (torch.randn(m, c, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)

        def params():
            return [torch.rand(c, device="cuda", generator=g) + 0.5, torch.randn(c, device="cuda", generator=g),
                    torch.zeros(c, device="cuda"), torch.ones(c, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"),
                    torch.empty(c, device="cuda"), torch.empty(c, device="cuda"), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")]

        self.sets = []
        for _ in range(2):
            s = {"x": act(), "y": torch.empty(m, c, dtype=torch.bfloat16, device="cuda"), "dy": act(),
                 "mask": torch.empty(m * c // 8, dtype=torch.uint8, device="cuda"), "dx": torch.empty(m, c, dtype=torch.bfloat16, device="cuda"),
                 "p": params()}
            if kind == "tail" or dual:
                s["dy2"] = act()
            if kind in ("tail", "last_tail"):
                s["g"] = torch.empty(m, c, dtype=torch.bfloat16, device="cuda")
            if dual:
                s["x_ds"], s["dx_ds"], s["p_ds"] = act(), torch.empty(m, c, dtype=torch.bfloat16, device="cuda"), params()
            self.sets.append(s)

    def run(self, lib, i, scratch, stream):
        s = self.sets[i]
        p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
        w, b, rm, rv, nbt, sm, si, gw, gb = [p(t) for t in s["p"]]
        m, c = self.m, self.c
        if self.kind == "ds_tail":
            w2, b2, rm2, rv2, nbt2, sm2, si2, gw2, gb2 = [p(t) for t in s["p_ds"]]
            rc = lib.b200c_bn_forward_dual(p(s["x"]), p(s["x_ds"]), p(s["y"]), p(s["mask"]), w, b, rm, rv, nbt, sm, si, 0.1, 1e-5,
                                           w2, b2, rm2, rv2, nbt2, sm2, si2, 0.1, 1e-5, m, c, scratch, stream)
            rc = rc or lib.b200c_bn_backward_dual(p(s["dy"]), p(s["dy2"]), None, p(s["mask"]), p(s["x"]), p(s["x_ds"]), p(s["dx"]),
                                                  p(s["dx_ds"]), w, sm, si, gw, gb, w2, sm2, si2, gw2, gb2, m, c, scratch, stream)
        else:
            rc = lib.b200c_bn_forward_mask(p(s["x"]), None, p(s["y"]), p(s["mask"]), w, b, rm, rv, nbt, sm, si, m, c, 0.1, 1e-5,
                                           scratch, stream)
            rc = rc or lib.b200c_bn_backward_mask(p(s["dy"]), p(s.get("dy2")), p(s["mask"]), p(s["x"]), p(s.get("g")), p(s["dx"]), w,
                                                  sm, si, gw, gb, m, c, scratch, stream)
        if rc:
            raise RuntimeError(f"{self.kind} m={m} c={c}: status {rc}")

    def digest(self):
        """Hash of what set 0's calls wrote and accumulated, after one reset of its running statistics."""
        h = hashlib.sha256()
        s = self.sets[0]
        for t in [s["mask"], s["dx"], s.get("g"), s.get("dx_ds")] + s["p"][2:] + s.get("p_ds", [])[2:]:
            if t is not None:
                h.update(t.contiguous().view(-1).view(__import__("torch").uint8).cpu().numpy().tobytes())
        return h.hexdigest()[:16]

    def reset(self):
        for s in self.sets:
            for ps in [s["p"]] + ([s["p_ds"]] if "p_ds" in s else []):
                ps[2].zero_(), ps[3].fill_(1.0), ps[4].zero_()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="libb200coll.so to time; repeat to compare builds")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    if not torch.cuda.is_available():
        raise SystemExit("bn_reduce_sites.py times GPU kernels: it needs a CUDA device")
    libs = [bind(p) for p in args.lib]
    sites = resnet50_sites(args.batch)
    c_max = max(c for _, _, c in sites)
    scratch = torch.zeros(libs[0].b200c_bn_dual_scratch_bytes(c_max), dtype=torch.uint8, device="cuda")
    stream = c_void_p(torch.cuda.current_stream().cuda_stream)

    times = {}   # (site, lib) -> {"stats": [us per round], "reduce": [...]}
    digests = {}
    for n, key in enumerate(sorted(sites, key=lambda k: (-k[1] * k[2], k[0]))):
        site = Site(*key, seed=n)
        for li, lib in enumerate(libs):
            site.reset()
            site.run(lib, 0, scratch.data_ptr(), stream)
            digests[(key, li)] = site.digest()
        for r in range(args.rounds):
            for li, lib in enumerate(libs):
                for i in range(4):   # warm-up
                    site.run(lib, i % 2, scratch.data_ptr(), stream)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for i in range(args.iters):
                        site.run(lib, i % 2, scratch.data_ptr(), stream)
                    torch.cuda.synchronize()
                acc = times.setdefault((key, li), {"stats": [], "reduce": []})
                us = collections.defaultdict(float)
                for ev in prof.events():
                    if ev.device_type == torch.autograd.DeviceType.CUDA:
                        fam = "stats" if "k_bn_stats" in ev.name else "reduce" if "k_bn_bwd_reduce" in ev.name else None
                        if fam:
                            us[fam] += ev.time_range.elapsed_us() / args.iters
                for fam in ("stats", "reduce"):
                    acc[fam].append(us[fam])
        del site
        torch.cuda.empty_cache()

    rows, totals = [], [{"stats_ms_per_step": 0.0, "reduce_ms_per_step": 0.0} for _ in libs]
    for key, count in sorted(sites.items(), key=lambda kv: (-kv[0][1] * kv[0][2], kv[0][0])):
        kind, m, c = key
        row = {"kind": kind, "m": m, "c": c, "count": count}
        for li in range(len(libs)):
            t = times[(key, li)]
            st, rd = statistics.median(t["stats"]), statistics.median(t["reduce"])
            row[f"lib{li}"] = {"stats_us": round(st, 1), "stats_gb_s": round(STATS_BYTES[kind] * m * c / (st * 1e-6) / 1e9, 1),
                               "reduce_us": round(rd, 1), "reduce_gb_s": round(REDUCE_BYTES[kind] * m * c / (rd * 1e-6) / 1e9, 1),
                               "stats_us_rounds": [round(x, 1) for x in t["stats"]], "reduce_us_rounds": [round(x, 1) for x in t["reduce"]],
                               "same_bits_as_lib0": digests[(key, li)] == digests[(key, 0)]}
            totals[li]["stats_ms_per_step"] += count * st / 1e3
            totals[li]["reduce_ms_per_step"] += count * rd / 1e3
        rows.append(row)
    for t in totals:
        for k in t:
            t[k] = round(t[k], 3)
    out = {"batch": args.batch, "iters": args.iters, "rounds": args.rounds, "libs": args.lib, **gpu_identity(), "sites": rows,
           "per_step": totals, "all_bits_identical": all(r[f"lib{li}"]["same_bits_as_lib0"] for r in rows for li in range(len(libs)))}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bn_reduce_sites.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(f"{out['gpu']}, power limit {out.get('power_limit_w')} W")
    hdr = "kind        m        c    n" + "".join(f" | lib{li} stats us (GB/s)  reduce us (GB/s)" for li in range(len(libs)))
    print(hdr)
    for r in rows:
        line = f"{r['kind']:9s} {r['m']:8d} {r['c']:5d} {r['count']:3d}"
        for li in range(len(libs)):
            d = r[f"lib{li}"]
            line += f" | {d['stats_us']:8.1f} ({d['stats_gb_s']:6.0f})  {d['reduce_us']:8.1f} ({d['reduce_gb_s']:6.0f})"
        print(line)
    print(json.dumps({"per_step": totals, "all_bits_identical": out["all_bits_identical"]}))


if __name__ == "__main__":
    main()
