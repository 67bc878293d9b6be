"""FSDP gradient reduce-scatter micro-benchmark: `reducescatter_scaled` (fp32 gradients, fp32 / bf16 wire, mean)
next to the plain `reducescatter` (fp32 SUM) and, under torchrun, `dist.reduce_scatter_tensor` (NCCL, AVG).

  python tools/fsdp_sweep.py --loopback 2,4,8 [--sizes ...] [--iters N]
      one GPU: every rank of a loopback world is a communicator on the same device, so the figures are
      single-GPU HBM traffic of W ranks' kernels running side by side, NOT NVLink; NCCL is not run.
  python -m torch.distributed.run --nproc-per-node W tools/fsdp_sweep.py [--sizes ...]
      one process per GPU: all three over NVLink.
--sizes are bytes of one rank's fp32 reduce-scatter INPUT (W shards).  Prints one JSON object: microseconds per
call (mean of a back-to-back loop timed with CUDA events; under torchrun the maximum over ranks), the device name
and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ant_ray_b200 import _native as N  # noqa: E402
from ant_ray_b200.fsdp import fsdp_config  # noqa: E402


def _device_info():
    name = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"device": name, "power_limit": power}


def _time_us(launch, iters):
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / iters


def loopback(W, sizes, iters):
    from ant_ray_b200.loopback import LoopbackWorld

    cfg = fsdp_config()
    # every rank's grid must be resident at once on the one GPU
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    world = LoopbackWorld(W, device=0, key=f"fsdp-sweep{W}", staging_bytes=cfg.staging_bytes, max_blocks=min(cfg.max_blocks, 2 * sm // W - 2))
    rows = []
    try:
        for nbytes in sizes:
            n = nbytes // 4 // W
            ins = [torch.randn(W * n, device="cuda") for _ in range(W)]
            outs = [torch.empty(n, device="cuda") for _ in range(W)]
            ptrs = [[t.data_ptr() + j * n * 4 for j in range(W)] for t in ins]
            row = {"world": W, "input_bytes": W * n * 4}
            calls = {
                "scaled_fp32_wire": lambda r, c: c.reducescatter_scaled(ptrs[r], outs[r].data_ptr(), n, N.FLOAT32, N.FLOAT32, 1.0 / W),
                "scaled_bf16_wire": lambda r, c: c.reducescatter_scaled(ptrs[r], outs[r].data_ptr(), n, N.FLOAT32, N.BFLOAT16, 1.0 / W),
                "plain_sum": lambda r, c: c.reducescatter(ptrs[r], outs[r].data_ptr(), n, N.FLOAT32, N.SUM),
            }
            for name, fn in calls.items():
                row[name + "_us"] = round(_time_us(lambda: world.run(fn), iters), 2)
            world.check()
            rows.append(row)
            del ins, outs
    finally:
        world.destroy()
    return rows


def distributed(sizes, iters):
    import torch.distributed as dist

    from ant_ray_b200.b200_group import PeerMemoryComm

    rank, W = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    comm = PeerMemoryComm(W, rank, "b200coll/fsdp-sweep/0", torch.cuda.current_device(), None, fsdp_config())
    rows = []
    try:
        for nbytes in sizes:
            n = nbytes // 4 // W
            x, out = torch.randn(W * n, device="cuda"), torch.empty(n, device="cuda")
            ptrs = [x.data_ptr() + j * n * 4 for j in range(W)]
            calls = {
                "scaled_fp32_wire": lambda: comm.reducescatter_scaled(ptrs, out.data_ptr(), n, N.FLOAT32, N.FLOAT32, 1.0 / W),
                "scaled_bf16_wire": lambda: comm.reducescatter_scaled(ptrs, out.data_ptr(), n, N.FLOAT32, N.BFLOAT16, 1.0 / W),
                "plain_sum": lambda: comm.reducescatter(ptrs, out.data_ptr(), n, N.FLOAT32, N.SUM),
                "nccl_avg": lambda: dist.reduce_scatter_tensor(out, x, op=dist.ReduceOp.AVG),
            }
            row = {"world": W, "input_bytes": W * n * 4}
            for name, fn in calls.items():
                dist.barrier()
                t = torch.tensor([_time_us(fn, iters)], device="cuda")
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                row[name + "_us"] = round(float(t), 2)
            comm.check()
            rows.append(row)
    finally:
        comm.destroy()
        dist.destroy_process_group()
    return rows if rank == 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loopback", default=None, help="comma-separated world sizes of one-GPU loopback worlds")
    ap.add_argument("--sizes", default=",".join(str(1 << k) for k in (20, 24, 26, 28)))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    sizes = [int(s) for s in args.sizes.split(",")]
    if args.loopback:
        rows = [r for W in args.loopback.split(",") for r in loopback(int(W), sizes, args.iters)]
        print(json.dumps({"mode": "loopback (single-GPU HBM traffic, not NVLink)", **_device_info(), "rows": rows}))
    else:
        rows = distributed(sizes, args.iters)
        if rows is not None:
            print(json.dumps({"mode": "one process per GPU (NVLink)", **_device_info(), "rows": rows}))


if __name__ == "__main__":
    main()
