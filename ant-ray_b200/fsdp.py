"""FSDP on the peer-memory collectives (R3, call site K13 in SURVEY.md section 2d).

Two seams, one per FSDP generation:

* FSDP2 (`torch.distributed.fsdp.fully_shard`): `FSDPModule.set_custom_all_gather` /
  `set_custom_reduce_scatter` take `AllGather` / `ReduceScatter` objects
  (torch/distributed/fsdp/_fully_shard/_fsdp_api.py).  `use_b200_collectives(module)` installs
  `B200AllGather` (parameter all-gather, in place into FSDP's output buffer) and `B200ReduceScatter`
  (gradient reduce-scatter: `b200c_reducescatter_scaled`, fp32 accumulate in rank order, one scale)
  on every FSDPModule of the tree, so a training step runs no NCCL collective.
* FSDP1 (`FullyShardedDataParallel`, what Ray Train's prepare_model builds): `register_comm_hook`
  with `b200_reduce_scatter_hook(state, grad, output)` for the sharded strategies and
  `b200_allreduce_hook_no_shard(state, grad)` for NO_SHARD.  FSDP1 skips its own pre/post division
  when a hook is set, so both hooks produce the mean.  FSDP1 has no seam for the parameter
  all-gather: that one stays on the torch process group.

The wire type (`grad_wire` / B200COLL_GRAD_WIRE, as for DDP) applies to fp32 gradients: "bf16" /
"fp16" round every contribution to 16 bits on the way across NVLink and accumulate in fp32.
"""
import os
from typing import Optional

import torch
import torch.distributed as dist
from torch.distributed.fsdp import FSDPModule
from torch.distributed.fsdp._fully_shard._fsdp_api import AllGather, ReduceScatter

from . import _native as N
from . import ddp_hook
from .b200_group import PeerMemoryComm, make_config, next_comm_key

# Both collectives run beside compute (the all-gather of the next layer, the reduce-scatter of the previous one):
# the DDP hook's small grid leaves the SMs to the matmuls, and a smaller staging area keeps two communicators cheap.
FSDP_STAGING_BYTES = 64 << 20


def fsdp_config():
    """Communicator config for the FSDP collectives: B200COLL_* environment variables, then the small grid
    (B200COLL_HOOK_MAX_BLOCKS, default 64) and, unless B200COLL_STAGING_MB / B200COLL_NVLS_STREAMS_MIN_BYTES are set,
    64 MiB of staging and no multi-stream NVLS allreduce."""
    over = {"max_blocks": int(os.environ.get("B200COLL_HOOK_MAX_BLOCKS", "64"))}
    if "B200COLL_STAGING_MB" not in os.environ:
        over["staging_bytes"] = FSDP_STAGING_BYTES
    if "B200COLL_NVLS_STREAMS_MIN_BYTES" not in os.environ:
        # the multi-stream NVLS allreduce needs three 128 MiB pieces in the staging area: off for the smaller area
        over["nvls_streams_min_bytes"] = 0
    return make_config(**over)


def _check_group(comm: PeerMemoryComm, group):
    if group.size() != comm.world_size or group.rank() != comm.rank:
        raise ValueError(f"process group (rank {group.rank()} of {group.size()}) does not match the B200 communicator "
                         f"(rank {comm.rank} of {comm.world_size})")


def _grad_dtype(t: torch.Tensor) -> int:
    if t.dtype not in ddp_hook._BUCKET:
        raise RuntimeError(f"B200 gradient reduction supports fp32 / bf16 / fp16 gradients, got {t.dtype}")
    return ddp_hook._BUCKET[t.dtype]


def _reduce_scatter_mean(state: ddp_hook.B200GradState, grad: torch.Tensor, output: torch.Tensor, scale: float):
    """output = scale * (sum over ranks of grad[rank * n:(rank + 1) * n]), n = output.numel(), on state's wire."""
    comm = state.comm
    n = output.numel()
    if grad.numel() != n * comm.world_size or not grad.is_contiguous() or not output.is_contiguous() or grad.dtype != output.dtype:
        raise RuntimeError(f"reduce-scatter needs contiguous tensors of one dtype with input numel = world size x output numel, "
                           f"got {grad.numel()} ({grad.dtype}) and {n} ({output.dtype})")
    dtype = _grad_dtype(grad)
    wire = state.wire if (state.wire is not None and grad.dtype == torch.float32) else dtype
    step = n * grad.element_size()
    comm.reducescatter_scaled([grad.data_ptr() + j * step for j in range(comm.world_size)], output.data_ptr(), n, dtype, wire, scale)
    state.launches += 1
    state.bytes += grad.numel() * grad.element_size()


# ---- FSDP2 -----------------------------------------------------------------------------------------------------

class B200AllGather(AllGather):
    """Parameter all-gather of FSDP2 on the peer-memory allgather.  FSDP passes the rank's own slice of the output
    as the input (in place); the bytes are moved as they are, so every dtype works, including the uint8 FSDP uses
    for parameters of mixed dtypes.  The op is ordered on the caller's stream and returns None: FSDP then waits on
    the event it records on that stream."""

    def __init__(self, comm: PeerMemoryComm):
        self.comm = comm

    def allocate(self, size, *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        return torch.empty(size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group, async_op: bool = False):
        comm = self.comm
        _check_group(comm, group)
        nbytes = input_tensor.numel() * input_tensor.element_size()
        if output_tensor.numel() * output_tensor.element_size() != nbytes * comm.world_size:
            raise RuntimeError(f"all-gather output holds {output_tensor.numel()} elements, expected world size x {input_tensor.numel()}")
        if not input_tensor.is_contiguous() or not output_tensor.is_contiguous():
            raise RuntimeError("all-gather needs contiguous tensors")
        base = output_tensor.data_ptr()
        comm.allgather(input_tensor.data_ptr(), [base + j * nbytes for j in range(comm.world_size)], nbytes, N.UINT8)
        return None


class B200ReduceScatter(ReduceScatter):
    """Gradient reduce-scatter of FSDP2 on `b200c_reducescatter_scaled`.  FSDP asks for AVG on fp32 / bf16
    gradients (one scale by 1/W after the fp32 fold) and for SUM on fp16, where it divides before and after the
    collective itself.  Any other op, e.g. the PREMUL_SUM of `set_gradient_divide_factor`, is refused."""

    def __init__(self, state: ddp_hook.B200GradState):
        self.state = state

    def allocate(self, size, *, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
        return torch.empty(size, dtype=dtype, device=device)

    def __call__(self, output_tensor: torch.Tensor, input_tensor: torch.Tensor, group, op, async_op: bool = False):
        comm = self.state.comm
        _check_group(comm, group)
        if op == dist.ReduceOp.AVG:
            scale = 1.0 / comm.world_size
        elif op == dist.ReduceOp.SUM:
            scale = 1.0
        else:
            raise ValueError(f"B200ReduceScatter supports ReduceOp.AVG and ReduceOp.SUM, got {op}: "
                             "FSDPModule.set_gradient_divide_factor is not supported with the B200 collectives")
        _reduce_scatter_mean(self.state, input_tensor, output_tensor, scale)
        return None


class B200FSDPState:
    """What `use_b200_collectives` installed: one communicator per collective, so a prefetched all-gather is not
    queued behind the previous reduce-scatter."""

    def __init__(self, all_gather: B200AllGather, reduce_scatter: B200ReduceScatter):
        self.all_gather = all_gather
        self.reduce_scatter = reduce_scatter

    def check(self):
        self.all_gather.comm.check()
        self.reduce_scatter.state.comm.check()

    def destroy(self):
        self.all_gather.comm.destroy()
        self.reduce_scatter.state.comm.destroy()


def use_b200_collectives(module: torch.nn.Module, wire: Optional[str] = None, config=None) -> B200FSDPState:
    """Run the parameter all-gathers and gradient reduce-scatters of every FSDPModule in `module` (after
    `fully_shard`) on the peer-memory kernels.  Rank and world size come from torch.distributed, the device from
    the current CUDA device; every rank must call this at the same point."""
    wire = ddp_hook.resolve_wire(wire)
    if config is None:
        config = fsdp_config()
    world_size = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    device = torch.cuda.current_device()
    ag = PeerMemoryComm(world_size, rank, next_comm_key("train/fsdp-allgather"), device, None, config)
    try:
        rs = ddp_hook.make_grad_state(world_size, rank, device, wire=wire, config=config, name="fsdp-reducescatter")
    except BaseException:
        ag.destroy()
        raise
    state = B200FSDPState(B200AllGather(ag), B200ReduceScatter(rs))
    n = 0
    for m in module.modules():
        if isinstance(m, FSDPModule):
            m.set_custom_all_gather(state.all_gather)
            m.set_custom_reduce_scatter(state.reduce_scatter)
            n += 1
    if n == 0:
        state.destroy()
        raise ValueError("no FSDPModule in the module tree: apply fully_shard first")
    return state


# ---- FSDP1 -----------------------------------------------------------------------------------------------------

def b200_reduce_scatter_hook(state: ddp_hook.B200GradState, grad: torch.Tensor, output: torch.Tensor) -> None:
    """FullyShardedDataParallel comm hook for the sharded strategies: `grad` is the padded, flattened unsharded
    gradient (world size x output numel), `output` receives this rank's shard of the mean."""
    _reduce_scatter_mean(state, grad, output, 1.0 / state.comm.world_size)


def b200_allreduce_hook_no_shard(state: ddp_hook.B200GradState, grad: torch.Tensor) -> None:
    """FullyShardedDataParallel comm hook for NO_SHARD: the mean of `grad` over the ranks, in place."""
    comm = state.comm
    dtype = _grad_dtype(grad)
    wire = state.wire if (state.wire is not None and grad.dtype == torch.float32) else dtype
    if not grad.is_contiguous():
        raise RuntimeError("the NO_SHARD gradient must be contiguous")
    comm.allreduce_scaled(grad.data_ptr(), grad.data_ptr(), grad.numel(), dtype, wire, 1.0 / comm.world_size, state.algo)
    state.launches += 1
    state.bytes += grad.numel() * grad.element_size()


def register_fsdp1(fsdp_model, state: Optional[ddp_hook.B200GradState] = None, wire: str = "fp32") -> ddp_hook.B200GradState:
    """Attach the hook matching the root FullyShardedDataParallel's sharding strategy; returns the state."""
    from torch.distributed.fsdp import ShardingStrategy

    # the communicator spans the torch.distributed world: a root wrapped over another process group would be
    # reduced over the wrong ranks
    pg = fsdp_model.process_group
    world_size = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    if pg.size() != world_size or pg.rank() != rank:
        raise ValueError(f"FullyShardedDataParallel's process group (rank {pg.rank()} of {pg.size()}) is not the torch.distributed "
                         f"world (rank {rank} of {world_size}): the B200 FSDP hook reduces over the whole world")
    if state is None:
        state = ddp_hook.make_grad_state(world_size, rank, torch.cuda.current_device(), wire=wire, config=fsdp_config(), name="fsdp")
    else:
        _check_group(state.comm, pg)
    hook = b200_allreduce_hook_no_shard if fsdp_model.sharding_strategy == ShardingStrategy.NO_SHARD else b200_reduce_scatter_hook
    fsdp_model.register_comm_hook(state, hook)
    return state
