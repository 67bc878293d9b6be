"""Ray Train integration (R3): a TorchConfig-shaped backend config and prepare_model().

Mirrors python/ray/train/torch/config.py (`TorchConfig` :41-70, `_setup_torch_process_group`
:73-128, `_TorchBackend.on_start` :163-212) and python/ray/train/v2/torch/train_loop_utils.py
(`prepare_model` :166-248).  Ray Train's plugin seam is `BackendConfig.backend_cls` ->
`Backend.on_start/on_training_start/on_shutdown` (python/ray/train/backend.py:15-59); the
classes below keep those names and signatures and only rely on the three WorkerGroup methods the
reference backend itself uses (`execute`, `execute_single`, `__len__`), so they plug into Ray
Train when Ray is installed and into any stand-in worker group otherwise (tests, bench.py).

What changes against the reference: torch.distributed is still initialised (DDP needs a process
group for its one-off parameter broadcast), but every per-step gradient reduction goes through
the fused peer-memory kernel registered as DDP's comm hook — NCCL is off the hot path.  With
parallel_strategy="fsdp" the model is wrapped in FullyShardedDataParallel as in the reference and
the gradient reduce-scatter runs in a comm hook on the same kernels (fsdp.py); FSDP1's parameter
all-gathers stay on the process group.
"""
import os
import socket
from dataclasses import dataclass
from datetime import timedelta
from typing import Any, Dict, Optional, Union

import torch
import torch.distributed as dist

from . import ddp_hook


@dataclass
class B200TorchConfig:
    """Drop-in for ray.train.torch.TorchConfig.  `backend` is the c10d backend used for the
    control-plane process group (nccl when GPUs are present); `grad_wire` selects what crosses
    NVLink in the fused gradient reduction: "fp32" (the default: exact torch-DDP default-reducer
    semantics, so switching the import does not change training numerics), or — opt-in, like
    registering torch's bf16_compress_hook — "bf16" / "fp16" (16-bit wire, fp32 accumulate)."""

    backend: Optional[str] = None
    init_method: str = "env"
    timeout_s: int = 1800
    grad_wire: str = "fp32"

    @property
    def backend_cls(self):
        return _B200TorchBackend

    @property
    def train_func_context(self):
        return _DeviceContext


class _DeviceContext:
    def __enter__(self):
        if torch.cuda.is_available():
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))

    def __exit__(self, *exc):
        return False


def _free_address():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return "127.0.0.1", s.getsockname()[1]


def _setup_torch_process_group(backend: str, world_rank: int, world_size: int, init_method: str, timeout_s: int = 1800,
                               grad_wire: str = "fp32"):
    """Connect torch.distributed (reference config.py:73-128) and remember the gradient wire type."""
    if backend == "nccl" and "TORCH_NCCL_ASYNC_ERROR_HANDLING" not in os.environ and "TORCH_NCCL_BLOCKING_WAIT" not in os.environ:
        os.environ["TORCH_NCCL_ASYNC_ERROR_HANDLING"] = "1"
    os.environ["B200COLL_GRAD_WIRE"] = grad_wire
    dist.init_process_group(backend=backend, init_method=init_method, rank=world_rank, world_size=world_size,
                            timeout=timedelta(seconds=timeout_s))


class _B200TorchBackend:
    share_cuda_visible_devices: bool = True  # peers must be able to map each other's HBM

    def on_start(self, worker_group, backend_config: B200TorchConfig):
        backend = backend_config.backend or ("nccl" if torch.cuda.is_available() else "gloo")
        addr, port = worker_group.execute_single(0, _free_address)
        if backend_config.init_method == "env":

            def set_env_vars(addr, port):
                os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = addr, str(port)

            worker_group.execute(set_env_vars, addr=addr, port=port)
            url = "env://"
        elif backend_config.init_method == "tcp":
            url = f"tcp://{addr}:{port}"
        else:
            raise ValueError(f"The provided init_method ({backend_config.init_method}) is not supported. "
                             "Must be either 'env' or 'tcp'.")
        n = len(worker_group)
        futures = [worker_group.execute_single_async(i, _setup_torch_process_group, backend=backend, world_rank=i,
                                                     world_size=n, init_method=url, timeout_s=backend_config.timeout_s,
                                                     grad_wire=backend_config.grad_wire) for i in range(n)]
        worker_group.wait(futures)

    def on_training_start(self, worker_group, backend_config):
        return None

    def on_shutdown(self, worker_group, backend_config):
        def _shutdown():
            if dist.is_initialized():
                dist.destroy_process_group()
            if torch.cuda.is_available():
                torch.cuda.empty_cache()

        worker_group.execute(_shutdown)


def get_device() -> torch.device:
    if torch.cuda.is_available():
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


def prepare_model(model: torch.nn.Module, move_to_device: Union[bool, torch.device] = True,
                  parallel_strategy: Optional[str] = "ddp", parallel_strategy_kwargs: Optional[Dict[str, Any]] = None,
                  grad_wire: Optional[str] = None, wrap_single: bool = False) -> torch.nn.Module:
    """ray.train.torch.prepare_model with the fused gradient reduction attached.

    Same arguments as the reference (v2/torch/train_loop_utils.py:166-248); `grad_wire` overrides
    the backend config's wire type, `wrap_single` wraps in DDP / FSDP even at world size 1 (the
    reference returns the bare model there).  The returned module carries `.b200_grad_state`.  On a CUDA device a
    torchvision ResNet, every torchvision Conv2dNormActivation ending in ReLU6, SiLU or Hardswish (MobileNetV2 / V3,
    EfficientNet), the inverted-residual blocks with their projection batch norm and squeeze-and-excitation, a
    torchvision DenseNet (whose concatenating batch norms then read the feature maps in place), torchvision's
    Inception v3 and GoogLeNet (whose Inception modules' branches then write into their concatenation in place), and
    torchvision's ShuffleNetV2 (whose blocks' branch ends then write the shuffled block output directly), and
    torchvision's VGG (whose stage ends then run batch norm, ReLU and the 2 x 2 max-pool as one site), is first
    rewritten in place by `fused_norm.fuse_model`, and with more than one rank the
    model's `nn.SyncBatchNorm` layers over the world group run on peer memory (`fused_norm.sync_batch_norm`, the
    communicator kept as `.b200_norm_comm`); SyncBatchNorm over a subgroup stays on torch.  The rewritten blocks'
    eval forward under `torch.no_grad()` or `torch.inference_mode()` (validation) runs each batch-norm site as one
    native eval launch with eager torch's bits; SyncBatchNorm does not synchronise in eval, so those run locally.
    """
    parallel_strategy_kwargs = dict(parallel_strategy_kwargs or {})
    device = move_to_device if isinstance(move_to_device, torch.device) else get_device()
    if device.type == "cuda":
        torch.cuda.set_device(device)
    if move_to_device:
        model = model.to(device)
    if device.type == "cuda":
        # batch norm + ReLU (+ residual add) of torchvision ResNets, and batch norm + activation of Conv2dNormActivation
        # blocks, as fused native sites; same bits as eager torch
        from . import fused_norm

        fused_norm.fuse_model(model)
    world_size = dist.get_world_size() if dist.is_initialized() else 1
    norm_comm = _attach_sync_norm(model, device, world_size)
    if parallel_strategy and (world_size > 1 or wrap_single):
        if parallel_strategy not in ("ddp", "fsdp"):
            raise RuntimeError(f"Unknown parallel_strategy {parallel_strategy!r}: the B200 backend supports 'ddp' and 'fsdp'.")
        if device.type != "cuda":
            raise RuntimeError("The B200 backend needs CUDA devices; there is no CPU fallback.")
        wire = ddp_hook.resolve_wire(grad_wire)
        if parallel_strategy == "ddp":
            from torch.nn.parallel import DistributedDataParallel

            kwargs = {"device_ids": [device], "output_device": device, **parallel_strategy_kwargs}
            model = DistributedDataParallel(model, **kwargs)
            model.b200_grad_state = ddp_hook.register(model, wire=wire)
        else:
            # the gradient reduce-scatter (or, for NO_SHARD, allreduce) runs in the comm hook; FSDP1 has no seam
            # for the parameter all-gather, which stays on the torch process group
            from torch.distributed.fsdp import FullyShardedDataParallel

            from . import fsdp

            model = FullyShardedDataParallel(model, **parallel_strategy_kwargs)
            model.b200_grad_state = fsdp.register_fsdp1(model, wire=wire)
    if norm_comm is not None:
        model.b200_norm_comm = norm_comm
    return model


def _attach_sync_norm(model, device, world_size):
    """Run the model's world-group SyncBatchNorm layers on peer memory instead of NCCL (fused_norm.sync_batch_norm);
    returns the communicator, or None where there is nothing to synchronise.  It is a communicator of its own: these
    collectives run on the compute stream, the gradient hook's on its own stream.  The returned module owns it
    (`.b200_norm_comm`), like the hook's communicator it lives until the process ends; a caller that keeps the
    process after training calls `model.b200_norm_comm.destroy()`, after which the model's sync sites raise."""
    if device.type != "cuda" or world_size <= 1:
        return None
    from . import fused_norm

    if not fused_norm.has_world_sync_batch_norm(model):
        return None
    comm = _sync_norm_comm(device)
    fused_norm.sync_batch_norm(model, comm)
    return comm


def _sync_norm_comm(device):
    """The sync batch norm's communicator over the default store.  Its messages are at most W * (2C + 1) floats
    (C <= 2048 for a ResNet: 16 KiB a rank), so a small staging area and a few CTAs per collective suffice."""
    from .b200_group import PeerMemoryComm, make_config, next_comm_key

    config = make_config(staging_bytes=1 << 20, max_blocks=8)
    return PeerMemoryComm(dist.get_world_size(), dist.get_rank(), next_comm_key("train/syncbn"), device.index, None, config)
