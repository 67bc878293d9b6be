"""Sync batch norm across GPUs: one process per GPU, W = 2, 4, 8 (skipped with fewer GPUs).

Every rank runs plain and ReLU sync sites of a few ResNet-50 shapes on its own uneven share of a global batch (one
rank holds a single image), once through fused_norm.FusedSyncBatchNorm over a peer-memory communicator built as
prepare_model builds it, and once through torch's nn.SyncBatchNorm over NCCL.  At W = 2 the two agree bit for bit (a
sum of two is order-free).  At every W the sync path equals the rank-order reference of test_gpu_sync_norm bit for
bit (each rank regenerates every rank's inputs from their seeds), and torch's NCCL results within fp32 tolerance.
"""
import os
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import copy, os, sys
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn


def worker(rank, W, port, root):
    sys.path[:0] = [root, os.path.join(root, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=W, device_id=dev)
    from ant_ray_b200 import fused_norm, train
    from gpu_common import assert_same_values
    from test_gpu_sync_norm import cl, make_sync_bn, reference

    comm = train._sync_norm_comm(dev)
    sizes = [1] + [2 + r for r in range(1, W)]
    for c, h, w in [(64, 56, 56), (256, 14, 14), (2048, 7, 7), (100, 9, 9)]:
        for kind in ("plain", "relu"):
            def inputs(r):
                g = torch.Generator(device="cuda").manual_seed(1000 * r + c)
                act = lambda s: cl((torch.randn(sizes[r], c, h, w, device="cuda", generator=g) * s).to(torch.bfloat16))
                return act(2.0), act(1.0)
            xs, dys = zip(*[inputs(r) for r in range(W)])
            bn = make_sync_bn(c, c)
            want = reference(bn, list(xs), [None] * W, list(dys), [None] * W, kind)[rank]
            ours = fused_norm.sync_batch_norm(copy.deepcopy(bn), comm)
            theirs = copy.deepcopy(bn)
            got = {}
            for name, mod in (("ours", ours), ("torch", theirs)):
                x = xs[rank].clone().requires_grad_()
                if kind == "relu":
                    y = fused_norm.bn_relu(mod, nn.ReLU(), x) if name == "ours" else torch.relu(mod(x))
                else:
                    y = mod(x)
                y.backward(dys[rank])
                got[name] = {"y": y.detach(), "dx": x.grad, "dweight": mod.weight.grad, "dbias": mod.bias.grad,
                             "running_mean": mod.running_mean, "running_var": mod.running_var,
                             "num_batches_tracked": mod.num_batches_tracked}
            for k in want:
                assert_same_values(got["ours"][k], want[k], f"W={W} rank {rank} {c}x{h}x{w} {kind} {k} vs reference")
                if W == 2:
                    assert_same_values(got["ours"][k], got["torch"][k], f"rank {rank} {c}x{h}x{w} {kind} {k} vs NCCL")
                elif got["ours"][k].is_floating_point():
                    torch.testing.assert_close(got["ours"][k].float(), got["torch"][k].float(), rtol=1e-2, atol=1e-2)
    torch.cuda.synchronize()
    comm.destroy()
    dist.barrier()
    if rank == 0:
        print("SYNCBN_MULTIGPU_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    W, port, root = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    mp.spawn(worker, args=(W, port, root), nprocs=W)
'''


def _ngpu():
    import torch

    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
@pytest.mark.parametrize("W", [2, 4, 8])
def test_sync_batch_norm_across_gpus_matches_torch(W, tmp_path):
    if _ngpu() < W:
        pytest.skip(f"needs {W} GPUs")
    script = tmp_path / "syncbn_workers.py"
    script.write_text(SCRIPT)
    env = dict(os.environ, B200COLL_TIMEOUT_MS="60000")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200COLL_STORE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, str(script), str(W), str(_free_port()), ROOT], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "SYNCBN_MULTIGPU_OK" in r.stdout, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
