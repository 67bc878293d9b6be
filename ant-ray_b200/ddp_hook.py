"""Fused gradient-bucket reduction for torch DDP (R3, call site K13 in SURVEY.md section 2d).

The reference has no hook of its own: Ray Train wraps the model in DistributedDataParallel
(python/ray/train/v2/torch/train_loop_utils.py:220-246) and torch's reducer then runs, per
bucket, `buffer.div_(W)` + ncclAllReduce — or, with bf16 compression
(torch/distributed/algorithms/ddp_comm_hooks/default_hooks.py: bf16_compress_hook),
`buffer.to(bf16).div_(W)` + ncclAllReduce + `buffer.copy_(result)`: three or four launches and an
NCCL call.  Here one launch per bucket reads every rank's fp32 gradients, moves bf16 (or fp32)
over NVLink, accumulates in fp32 in rank order, multiplies by 1/W and writes the fp32 mean back
into the bucket: no div_, no cast kernels, no copy_, no NCCL.

Attachment point: `DistributedDataParallel.register_comm_hook(state, hook)` with
`hook(state, bucket) -> Future[Tensor]`; the future's value must be the bucket buffer holding the
mean.  The kernel is enqueued on a dedicated communication stream so it overlaps the rest of the
backward pass, like the NCCL stream of the default reducer.
"""
import logging
import os
from typing import Optional

import torch

from . import _native as N
from .b200_group import PeerMemoryComm, next_comm_key

logger = logging.getLogger(__name__)

_WIRE = {None: None, "fp32": None, "bf16": N.BFLOAT16, "fp16": N.FLOAT16,
         torch.float32: None, torch.bfloat16: N.BFLOAT16, torch.float16: N.FLOAT16}
_BUCKET = {torch.float32: N.FLOAT32, torch.bfloat16: N.BFLOAT16, torch.float16: N.FLOAT16}


class B200GradState:
    """Hook state: the peer-memory communicator, the wire dtype and the communication stream."""

    def __init__(self, comm: PeerMemoryComm, wire="fp32", algo: int = N.ALGO_AUTO, time_kernels: bool = False):
        if wire not in _WIRE:
            raise ValueError("wire must be one of fp32 / bf16 / fp16")
        self.comm = comm
        self.wire = _WIRE[wire]
        self.algo = algo
        # high priority: the few CTAs of a bucket reduction take SM slots as soon as the backward kernels free any,
        # instead of queueing behind their whole grids (every rank's matching block must be resident to progress)
        self.stream = torch.cuda.Stream(device=comm.device, priority=-1)
        self.launches = 0
        self.bytes = 0
        self.time_kernels = time_kernels
        self.events = []  # (start, end, nbytes) when time_kernels

    def kernel_times_ms(self):
        """(milliseconds, bytes) per hook launch recorded since the last call; synchronises."""
        torch.cuda.synchronize(self.comm.device)
        out = [(s.elapsed_time(e), n) for s, e, n in self.events]
        self.events = []
        return out


def resolve_wire(wire: Optional[str] = None) -> str:
    """The gradient wire type: `wire`, else B200COLL_GRAD_WIRE (set from B200TorchConfig.grad_wire), else fp32."""
    wire = wire or os.environ.get("B200COLL_GRAD_WIRE", "fp32")
    if wire != "fp32":
        logger.warning("B200 gradient reduction uses a %s wire (fp32 accumulate): gradients are rounded to %s on the "
                       "way across NVLink, like torch's %s_compress_hook. Use grad_wire='fp32' for the exact "
                       "default-reducer numerics.", wire, wire, wire)
    return wire


SMALL_BUCKET_BYTES = 1 << 20


def b200_allreduce_hook(state: B200GradState, bucket) -> torch.futures.Future[torch.Tensor]:
    buf = bucket.buffer()
    if buf.dtype not in _BUCKET:
        raise RuntimeError(f"B200 gradient hook supports fp32 / bf16 / fp16 buckets, got {buf.dtype}")
    dtype = _BUCKET[buf.dtype]
    wire = state.wire if (state.wire is not None and buf.dtype == torch.float32) else dtype
    comm = state.comm
    nbytes = buf.numel() * buf.element_size()
    if nbytes <= SMALL_BUCKET_BYTES and not state.time_kernels:
        # Latency-bound buckets (an RLlib learner's few hundred KB): nothing to overlap, so the reduction is enqueued
        # on the stream the gradients were produced on — no stream switch, no extra events — and takes the LL / one-shot
        # kernels with an fp32 wire (a 16-bit wire would only add a cast pass to a message this small).
        comm.allreduce_scaled(buf.data_ptr(), buf.data_ptr(), buf.numel(), dtype, dtype, 1.0 / comm.world_size, state.algo)
        fut = torch.futures.Future(devices=[torch.device("cuda", comm.device)])
        fut.set_result(buf)
        state.launches += 1
        state.bytes += nbytes
        return fut
    s = state.stream
    s.wait_stream(torch.cuda.current_stream(comm.device))  # gradients of this bucket are final
    with torch.cuda.stream(s):
        if state.time_kernels:
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record(s)
        comm.allreduce_scaled(buf.data_ptr(), buf.data_ptr(), buf.numel(), dtype, wire, 1.0 / comm.world_size, state.algo)
        if state.time_kernels:
            e1.record(s)
            state.events.append((e0, e1, nbytes))
        fut = torch.futures.Future(devices=[torch.device("cuda", comm.device)])
        fut.set_result(buf)  # records an event on `s`; DDP's wait() makes the compute stream wait on it
    state.launches += 1
    state.bytes += nbytes
    return fut


def make_grad_state(world_size: Optional[int] = None, rank: Optional[int] = None, device: Optional[int] = None,
                    wire="fp32", store=None, config=None, name: str = "ddp", **kw) -> B200GradState:
    """Build the communicator for the hook from the torch.distributed world (rank / world size and,
    by default, the default process group's store for the rendezvous)."""
    import torch.distributed as dist

    if world_size is None:
        world_size = dist.get_world_size() if dist.is_initialized() else 1
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    if config is None:
        # The reduction runs beside the backward pass: a small grid leaves the SMs to the convolutions
        # (the bucket traffic needs a tiny fraction of NVLink), like NCCL's handful of channels.
        from .b200_group import make_config

        config = make_config(max_blocks=int(os.environ.get("B200COLL_HOOK_MAX_BLOCKS", "64")))
    comm = PeerMemoryComm(world_size, rank, next_comm_key("train/" + name), device, store, config)
    return B200GradState(comm, wire=wire, **kw)


def register(ddp_model, state: Optional[B200GradState] = None, **kw) -> B200GradState:
    """Attach the fused reduction to a DistributedDataParallel module; returns the state."""
    if state is None:
        dev = next(ddp_model.parameters()).device
        state = make_grad_state(device=dev.index, **kw)
    ddp_model.register_comm_hook(state, b200_allreduce_hook)
    return state
