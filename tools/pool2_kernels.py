#!/usr/bin/env python
"""Kernel time and achieved bandwidth of VGG's stage-end kernels (norm_pool2.cuh) at vgg16_bn's five pool sites, and of
bn::k_bn_bwd_reduce at the same [m][C] (a ReLU site reading its mask bits) for comparison.

Per site (n = `--batch`, 256, at 224 x 224): `--iters` training forwards and backwards through the C-ABI under
torch.profiler after `--warmup` untraced ones, then the same for b200c_bn_forward_mask / b200c_bn_backward_mask.  Each
kernel's mean device time and the bytes it must move, computed from the shapes (per input element: forward 2 read + 0.5
+ 0.25 written; pool2 reduce 2 + 0.5 + 0.25 read; pool2 elementwise 2 + 0.5 + 0.25 read + 2 written; statistics 2 read;
the ReLU site's reduce 2 + 2 + 1/8 read, its elementwise kernel that and 2 written), give GB/s.  The card's name and power limit are read in the same run.

  python tools/pool2_kernels.py --out DIR [--batch 256] [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from step_profile import gpu_identity  # noqa: E402

SITES = [(64, 224), (128, 112), (256, 56), (512, 28), (512, 14)]
# bytes per input element of each kernel
BYTES = {"k_pool2_fwd": 2.75, "k_pool2_bwd_reduce": 2.75, "k_pool2_bwd_elemt": 4.75, "k_bn_stats": 2.0, "k_bn_bwd_reduce": 4.125,
         "k_bn_bwd_elemt": 6.125}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--out", required=True)
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--warmup", type=int, default=3)
    args = p.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from ant_ray_b200 import _native as N

    if not torch.cuda.is_available():
        raise SystemExit("pool2_kernels.py measures GPU kernels: it needs a CUDA device")
    lib = N.load()
    out = {**gpu_identity(), "batch": args.batch, "iters": args.iters, "sites": []}
    stream = torch.cuda.current_stream().cuda_stream
    for c, h in SITES:
        n = args.batch
        m = n * h * h
        g = torch.Generator(device="cuda").manual_seed(c + h)
        x = torch.randn(m, c, device="cuda", generator=g, dtype=torch.bfloat16)
        y = torch.empty(m // 4, c, device="cuda", dtype=torch.bfloat16)
        dyp = torch.randn(m // 4, c, device="cuda", generator=g, dtype=torch.bfloat16)
        argmax = torch.empty(m // 4 * c, device="cuda", dtype=torch.uint8)
        dx = torch.empty_like(x)
        w, b = torch.ones(c, device="cuda"), torch.zeros(c, device="cuda")
        rm, rv = torch.zeros(c, device="cuda"), torch.ones(c, device="cuda")
        stats, dw, db = torch.empty(2 * c, device="cuda"), torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
        scratch = torch.zeros(lib.b200c_bn_scratch_bytes(c), dtype=torch.uint8, device="cuda")
        s = stats.data_ptr()
        yfull, dyfull = torch.empty_like(x), torch.randn(m, c, device="cuda", generator=g, dtype=torch.bfloat16)
        mask = torch.empty(m * c // 8, device="cuda", dtype=torch.uint8)

        def pool2():
            N.check(lib.b200c_bn_forward_pool2(x.data_ptr(), y.data_ptr(), argmax.data_ptr(), w.data_ptr(), b.data_ptr(), rm.data_ptr(),
                                               rv.data_ptr(), None, s, s + 4 * c, n, h, h, c, 0.1, 1e-5, scratch.data_ptr(), stream))
            N.check(lib.b200c_bn_backward_pool2(dyp.data_ptr(), argmax.data_ptr(), x.data_ptr(), dx.data_ptr(), w.data_ptr(), s, s + 4 * c,
                                                dw.data_ptr(), db.data_ptr(), n, h, h, c, scratch.data_ptr(), stream))

        def relu_site():
            N.check(lib.b200c_bn_forward_mask(x.data_ptr(), None, yfull.data_ptr(), mask.data_ptr(), w.data_ptr(), b.data_ptr(),
                                              rm.data_ptr(), rv.data_ptr(), None, s, s + 4 * c, m, c, 0.1, 1e-5, scratch.data_ptr(), stream))
            N.check(lib.b200c_bn_backward_mask(dyfull.data_ptr(), None, mask.data_ptr(), x.data_ptr(), None, dx.data_ptr(), w.data_ptr(),
                                               s, s + 4 * c, dw.data_ptr(), db.data_ptr(), m, c, scratch.data_ptr(), stream))

        site = {"c": c, "h": h, "elements": m * c, "kernels": {}}
        for fn in (pool2, relu_site):
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.iters):
                    fn()
                torch.cuda.synchronize()
            for ev in prof.key_averages():
                t = getattr(ev, "self_device_time_total", None)
                if t is None:
                    t = ev.self_cuda_time_total
                name = ev.key
                for k in BYTES:
                    if k in name and t > 0:
                        key = f"{'relu_site.' if fn is relu_site else ''}{k}"
                        us = t / ev.count
                        site["kernels"][key] = {"us": round(us, 1), "GB_per_s": round(BYTES[k] * m * c / us / 1e3, 1)}
        out["sites"].append(site)
        del x, y, dyp, argmax, dx, yfull, dyfull, mask
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "pool2_kernels.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
