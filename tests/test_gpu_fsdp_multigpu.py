"""FSDP on the peer-memory collectives across GPUs: one process per GPU, W = 2, 4, 8 (skipped with fewer GPUs).

A small MLP trains under FSDP2 (`fully_shard` + `use_b200_collectives`, fp32 and bf16 wire) and under FSDP1
(`prepare_model(parallel_strategy="fsdp")`, FULL_SHARD, the sharded comm hook):
  * every sharded gradient equals the oracle's fold of the per-rank unsharded gradients (every contribution rounded
    to the wire, fp32 fold in rank order, one 1/W scale), bit for bit;
  * parameters after three SGD steps match the same model trained by stock FSDP over NCCL within fp32 tolerance.
For FSDP2 the per-rank unsharded gradients come from the same MLP run without FSDP on the rank's batch; for FSDP1
they are the padded flat gradients FSDP hands the hook, gathered from every rank.

The workers run in a subprocess (torch.multiprocessing): FSDP needs a default process group per process.
"""
import os
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r'''
import os, sys
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn


def worker(rank, W, port, root):
    sys.path.insert(0, root)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=W, device_id=dev)
    from torch.distributed.fsdp import FullyShardedDataParallel as FSDP, fully_shard

    from ant_ray_b200 import fsdp
    from ant_ray_b200 import train as b200_train
    from oracle import oracle as O

    def build():
        torch.manual_seed(7)
        return nn.Sequential(nn.Linear(64, 256), nn.ReLU(), nn.Linear(256, 256), nn.ReLU(), nn.Linear(256, 16)).to(dev)

    g = torch.Generator().manual_seed(100 + rank)
    x = torch.randn(32, 64, generator=g).to(dev)
    y = torch.randint(0, 16, (32,), generator=g).to(dev)

    def loss_of(m):
        return nn.functional.cross_entropy(m(x), y)

    def gather_all(t):
        out = [torch.empty_like(t) for _ in range(W)]
        dist.all_gather(out, t.contiguous())
        return [o.cpu() for o in out]

    def same_bits(a, b, what):
        a, b = a.cpu(), b.cpu()
        assert a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32)), \
            (what, rank, float((a - b).abs().max()) if a.shape == b.shape else (a.shape, b.shape))

    def sgd_steps(m, steps=3):
        opt = torch.optim.SGD(m.parameters(), lr=0.05)
        for _ in range(steps):
            opt.zero_grad(set_to_none=True)
            loss_of(m).backward()
            opt.step()

    ref = build()
    loss_of(ref).backward()
    unsharded = [gather_all(p.grad) for p in ref.parameters()]   # [param][source rank]

    def fsdp2(m):
        for layer in m:
            if isinstance(layer, nn.Linear):
                fully_shard(layer)
        return fully_shard(m)

    # ---- FSDP2: all-gathers and reduce-scatters on the peer-memory kernels
    for wire in ("fp32", "bf16"):
        model = fsdp2(build())
        st = fsdp.use_b200_collectives(model, wire=wire)
        loss_of(model).backward()
        torch.cuda.synchronize()
        st.check()
        wdt = None if wire == "fp32" else torch.bfloat16
        for k, (p, contribs) in enumerate(zip(model.parameters(), unsharded)):
            want = torch.chunk(O.allreduce_scaled(contribs, wdt, 1.0 / W), W, dim=0)[rank]
            same_bits(p.grad.to_local(), want, f"fsdp2 wire={wire} param {k}")
        assert st.reduce_scatter.state.launches >= 1
        if wire == "fp32":
            base = fsdp2(build())
            sgd_steps(model)
            sgd_steps(base)
            torch.cuda.synchronize()
            st.check()
            for p, q in zip(model.parameters(), base.parameters()):
                torch.testing.assert_close(p.full_tensor(), q.full_tensor(), rtol=1e-5, atol=1e-6)
        st.destroy()
        del model

    # ---- FSDP1 through prepare_model: the sharded comm hook
    fused = fsdp.b200_reduce_scatter_hook
    for wire in ("fp32", "bf16"):
        seen = []

        def recording(state, grad, output):
            fused(state, grad, output)
            seen.append((grad.detach().clone(), output))

        fsdp.b200_reduce_scatter_hook = recording    # what prepare_model -> fsdp.register_fsdp1 attaches
        model = b200_train.prepare_model(build(), parallel_strategy="fsdp", grad_wire=wire)
        fsdp.b200_reduce_scatter_hook = fused
        state = model.b200_grad_state
        loss_of(model).backward()
        torch.cuda.synchronize()
        state.comm.check()
        assert len(seen) >= 1 and state.launches == len(seen), (len(seen), state.launches)
        wdt = None if wire == "fp32" else torch.bfloat16
        for k, (grad, out) in enumerate(seen):
            n = out.numel()
            contribs = [gr[rank * n:(rank + 1) * n] for gr in gather_all(grad)]
            same_bits(out, O.allreduce_scaled(contribs, wdt, 1.0 / W), f"fsdp1 wire={wire} flat gradient {k}")
        if wire == "fp32":
            base = FSDP(build())
            sgd_steps(model)
            sgd_steps(base)
            torch.cuda.synchronize()
            state.comm.check()
            got, want = model.state_dict(), base.state_dict()   # full (unsharded) parameters on every rank
            assert got.keys() == want.keys()
            for key in got:
                torch.testing.assert_close(got[key], want[key], rtol=1e-5, atol=1e-6)
        state.comm.destroy()
        del model
    dist.barrier()
    if rank == 0:
        print("FSDP_MULTIGPU_OK", flush=True)
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
def test_fsdp_across_gpus_matches_the_oracle_and_nccl(W, tmp_path):
    if _ngpu() < W:
        pytest.skip(f"needs {W} GPUs")
    script = tmp_path / "fsdp_workers.py"
    script.write_text(SCRIPT)
    env = dict(os.environ, B200COLL_TIMEOUT_MS="60000")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200COLL_GRAD_WIRE", "B200COLL_STORE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, str(script), str(W), str(_free_port()), ROOT], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0 and "FSDP_MULTIGPU_OK" in r.stdout, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
