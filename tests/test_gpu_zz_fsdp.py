"""FSDP on the peer-memory collectives inside torch's own FSDP, on one GPU.

`prepare_model(..., parallel_strategy="fsdp", wrap_single=True)` wraps the model in FullyShardedDataParallel at
world size 1, where FSDP1 uses NO_SHARD, and registers `b200_allreduce_hook_no_shard`; every flat gradient then
goes through the library (the W = 1 form of the fused mean: wire rounding and scale).  The hook is wrapped so that
each flat gradient is also reduced the stock way on a copy (FSDP's division by the world size for the fp32 wire,
bf16 rounding for the bf16 wire), and the flat gradient must hold exactly those bits afterwards; with
use_orig_params the per-parameter gradients must also equal those of the same model run without FSDP.  A few SGD
steps then run through the hooked model.  Last, `use_b200_collectives` installs the FSDP2 collectives on a
`fully_shard` model, which then trains a few steps.

The file sorts last among the GPU tests and runs in a subprocess: FSDP needs a default process group, which must
not leak into the other tests of the session.
"""
import os
import socket
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = r"""
import os, sys
sys.path.insert(0, os.environ["B200_TEST_ROOT"])
import torch
import torch.distributed as dist
import torch.nn as nn

torch.cuda.set_device(0)
dev = torch.device("cuda", 0)
dist.init_process_group("nccl", rank=0, world_size=1, device_id=dev)
from ant_ray_b200 import fsdp
from ant_ray_b200 import train as b200_train


def build():
    torch.manual_seed(7)
    return nn.Sequential(nn.Linear(128, 1024), nn.ReLU(), nn.Linear(1024, 1024), nn.ReLU(), nn.Linear(1024, 10)).to(dev)


g = torch.Generator().manual_seed(11)
x = torch.randn(64, 128, generator=g).to(dev)
y = torch.randint(0, 10, (64,), generator=g).to(dev)
ref_model = build()
nn.functional.cross_entropy(ref_model(x), y).backward()
ref_grads = [p.grad.clone() for p in ref_model.parameters()]
fused_hook = fsdp.b200_allreduce_hook_no_shard
for wire in ("fp32", "bf16"):
    seen = []

    def both(st, grad):
        want = grad.clone().div_(1) if wire == "fp32" else grad.to(torch.bfloat16).float()
        fused_hook(st, grad)
        seen.append((grad, want))

    fsdp.b200_allreduce_hook_no_shard = both     # what prepare_model -> fsdp.register_fsdp1 attaches
    model = b200_train.prepare_model(build(), grad_wire=wire, wrap_single=True, parallel_strategy="fsdp",
                                     parallel_strategy_kwargs={"use_orig_params": True})
    fsdp.b200_allreduce_hook_no_shard = fused_hook
    assert isinstance(model, torch.distributed.fsdp.FullyShardedDataParallel)
    state = model.b200_grad_state
    nn.functional.cross_entropy(model(x), y).backward()
    torch.cuda.synchronize()
    state.comm.check()
    assert len(seen) >= 1 and state.launches == len(seen), (len(seen), state.launches)
    for grad, want in seen:
        assert torch.equal(grad.view(torch.int32), want.view(torch.int32)), (wire, float((grad - want).abs().max()))
    for p, r in zip(model.parameters(), ref_grads):
        r = r if wire == "fp32" else r.to(torch.bfloat16).float()
        assert torch.equal(p.grad, r), (wire, tuple(p.shape), float((p.grad - r).abs().max()))
    opt = torch.optim.SGD(model.parameters(), lr=0.05)
    first = None
    for _ in range(5):
        opt.zero_grad(set_to_none=True)
        loss = nn.functional.cross_entropy(model(x), y)
        loss.backward()
        opt.step()
        first = float(loss.detach()) if first is None else first
    torch.cuda.synchronize()
    state.comm.check()
    last = float(loss.detach())
    assert last == last and last <= first, (first, last)
    print("fsdp1 wire", wire, "flat gradients", len(seen), "launches", state.launches, flush=True)
    state.comm.destroy()
    del model, opt

# FSDP2: the collectives are installed on every FSDPModule and a few steps train through them (at world size 1
# FSDP2 itself skips both collectives; the loopback tests run them on the layouts FSDP builds)
from torch.distributed.fsdp import FSDPModule, fully_shard

model = build()
for layer in model:
    if isinstance(layer, nn.Linear):
        fully_shard(layer)
fully_shard(model)
st = fsdp.use_b200_collectives(model)
groups = [m._get_fsdp_state()._fsdp_param_group for m in model.modules() if isinstance(m, FSDPModule)]
assert len(groups) == 4 and all(g._all_gather_comm is st.all_gather and g._reduce_scatter_comm is st.reduce_scatter
                                for g in groups if g is not None)
opt = torch.optim.SGD(model.parameters(), lr=0.05)
for _ in range(3):
    opt.zero_grad(set_to_none=True)
    loss = nn.functional.cross_entropy(model(x), y)
    loss.backward()
    opt.step()
torch.cuda.synchronize()
st.check()
assert float(loss) == float(loss)
print("fsdp2 installed on", len(groups), "modules", flush=True)
st.destroy()
print("FSDP_OK")
dist.destroy_process_group()
"""


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.gpu
def test_fsdp_hooks_inside_torch_fsdp():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    env = dict(os.environ, B200_TEST_ROOT=ROOT, MASTER_ADDR="127.0.0.1", MASTER_PORT=str(_free_port()),
               B200COLL_TIMEOUT_MS="20000")
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "B200COLL_GRAD_WIRE"):
        env.pop(k, None)
    r = subprocess.run([sys.executable, "-c", SCRIPT], env=env, capture_output=True, text=True, timeout=170)
    assert r.returncode == 0 and "FSDP_OK" in r.stdout, r.stdout[-2000:] + "\n" + r.stderr[-4000:]
