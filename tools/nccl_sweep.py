"""Stock-NCCL allreduce sweep (the NCCL baseline).

Launch: python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/nccl_sweep.py
The reference drives ncclAllReduce through cupy (nccl_collective_group.py:181-188);
cupy is absent in this image so the same NCCL entry point is reached via torch c10d.
"""
import json
import os

import torch
import torch.distributed as dist


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    max_bytes = int(os.environ.get("SWEEP_MAX_BYTES", 1 << 30))
    dtype = {"f32": torch.float32, "bf16": torch.bfloat16}[os.environ.get("SWEEP_DTYPE", "f32")]
    out = []
    size = 1024
    while size <= max_bytes:
        n = size // torch.empty((), dtype=dtype).element_size()
        x = torch.ones(n, dtype=dtype, device="cuda")
        iters = 200 if size <= (1 << 20) else (50 if size <= (64 << 20) else 10)
        for _ in range(5):
            dist.all_reduce(x)
        torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            dist.all_reduce(x)
        e1.record(); torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / iters
        t = torch.tensor([us], device="cuda"); dist.all_reduce(t, op=dist.ReduceOp.MAX)
        us = t.item()
        alg = size / us / 1e3
        out.append({"bytes": size, "us": round(us, 2), "algbw": round(alg, 2), "busbw": round(alg * 2 * (world - 1) / world, 2)})
        size *= 4
    if rank == 0:
        print(json.dumps({"impl": "nccl", "nccl_version": ".".join(map(str, torch.cuda.nccl.version())), "world": world,
                          "dtype": str(dtype), "sweep": out}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
