"""B200Group: the BaseGroup implementation that replaces the reference's NCCLGroup (R1).

Interface parity (reference python/ray/util/collective/collective_group/):
  * constructor `(world_size, rank, group_name)` and the 8 ops + `destroy_group` + `backend()`
    of BaseGroup (base_collective_group.py:15-84);
  * every op takes the caller's tensors wrapped in lists exactly as `collective.py` passes them
    (:343, :515, :569) and writes results in place, returning None;
  * like NCCLGroup the native communicator is created lazily at the first op
    (nccl_collective_group.py:395-449), so `init_collective_group` itself never blocks on peers;
  * misuse raises RuntimeError, CPU tensors raise RuntimeError
    (single_node_gpu_tests/test_allreduce.py:127-162).

Differences by design (one process per GPU on one NVSwitch box):
  * exactly one tensor per call (the reference's `*_multigpu` multi-GPU-per-process lists are
    rejected with RuntimeError);
  * allgather writes straight into the caller's W tensors and reducescatter reads the W input
    tensors in place — the flat temporary and the W extra device copies of
    nccl_collective_group.py:292-296 / :334-337 do not exist;
  * work is enqueued on the caller's current torch stream (the reference hops to a side stream
    and never joins back, :451-459), so ordinary stream semantics apply.
"""
import ctypes
import logging
import os
import threading
from typing import List, Optional

from . import _native as N
from . import rendezvous
from .types import (AllGatherOptions, AllReduceOptions, Backend, BarrierOptions, BroadcastOptions, DagReduceOp,
                    RecvOptions, ReduceOp, ReduceOptions, ReduceScatterOptions, SendOptions)

logger = logging.getLogger(__name__)

# ray.util.collective ReduceOp -> ncclRedOp_t (reference nccl_util.py:22-27)
_REDUCE_OP_MAP = {ReduceOp.SUM: N.SUM, ReduceOp.PRODUCT: N.PROD, ReduceOp.MIN: N.MIN, ReduceOp.MAX: N.MAX}
_incarnations = {}
_incarnations_lock = threading.Lock()


def native_reduce_op(op, is_bool: bool = False) -> int:
    """ncclRedOp_t for a reduce op.  Bool tensors travel as bytes, so SUM becomes MAX (a logical OR
    that keeps every byte 0 or 1) and AVG is refused, as torch's NCCL backend does; PROD, MIN and
    MAX are already logical AND / AND / OR on 0/1 bytes."""
    if isinstance(op, ReduceOp):
        nat = _REDUCE_OP_MAP[op]
    elif isinstance(op, DagReduceOp):
        nat = op.value
    else:
        # ray's own enums when running inside ray: match by name
        name = getattr(op, "name", None)
        if name not in ("SUM", "PRODUCT", "MIN", "MAX", "AVG"):
            raise RuntimeError("B200 backend does not support reduce op: '{}'.".format(op))
        nat = {"SUM": N.SUM, "PRODUCT": N.PROD, "MIN": N.MIN, "MAX": N.MAX, "AVG": N.AVG}[name]
    if is_bool:
        if nat == N.AVG:
            raise RuntimeError("AVG is not defined for bool tensors.")
        if nat == N.SUM:
            return N.MAX
    return nat


def _torch_dtype_map():
    import torch

    return {
        torch.bool: N.UINT8, torch.uint8: N.UINT8, torch.int8: N.INT8, torch.int32: N.INT32, torch.int64: N.INT64,
        torch.float16: N.FLOAT16, torch.float32: N.FLOAT32, torch.float64: N.FLOAT64, torch.bfloat16: N.BFLOAT16,
        torch.uint32: N.UINT32, torch.uint64: N.UINT64,
    }


_TORCH_DTYPES = None
_TYPESTR = {"|i1": N.INT8, "|u1": N.UINT8, "<i4": N.INT32, "<u4": N.UINT32, "<i8": N.INT64, "<u8": N.UINT64,
            "<f2": N.FLOAT16, "<f4": N.FLOAT32, "<f8": N.FLOAT64, "|b1": N.UINT8}


class TensorView:
    """Pointer-level view of a GPU tensor (torch.Tensor or any __cuda_array_interface__ object)."""

    __slots__ = ("ptr", "numel", "dtype", "shape", "device", "itemsize", "is_bool")

    def __init__(self, t):
        global _TORCH_DTYPES
        try:
            import torch
        except ImportError:  # pragma: no cover
            torch = None
        if torch is not None and isinstance(t, torch.Tensor):
            if not t.is_cuda:
                raise RuntimeError("Torch tensor must be on GPU when using B200 collectives.")
            if not t.is_contiguous():
                raise RuntimeError("B200 collectives require contiguous tensors.")
            if _TORCH_DTYPES is None:
                _TORCH_DTYPES = _torch_dtype_map()
            if t.dtype not in _TORCH_DTYPES:
                raise RuntimeError("Unsupported tensor dtype: {}".format(t.dtype))
            self.ptr = t.data_ptr()
            self.numel = t.numel()
            self.dtype = _TORCH_DTYPES[t.dtype]
            self.is_bool = t.dtype == torch.bool
            self.shape = list(t.shape)
            self.device = t.device.index
            self.itemsize = t.element_size()
            return
        cai = getattr(t, "__cuda_array_interface__", None)
        if cai is not None:
            if cai.get("strides") is not None:
                raise RuntimeError("B200 collectives require contiguous arrays.")
            if cai["typestr"] not in _TYPESTR:
                raise RuntimeError("Unsupported array dtype: {}".format(cai["typestr"]))
            self.ptr = cai["data"][0]
            self.shape = list(cai["shape"])
            n = 1
            for s in self.shape:
                n *= s
            self.numel = n
            self.dtype = _TYPESTR[cai["typestr"]]
            self.is_bool = cai["typestr"] == "|b1"
            self.itemsize = int(cai["typestr"][2:])
            dev = getattr(getattr(t, "device", None), "id", None)
            self.device = dev if isinstance(dev, int) else None
            return
        raise RuntimeError(
            "Unsupported tensor type. Got: {}. Supported GPU tensor types are: torch.Tensor (cuda), "
            "cupy.ndarray.".format(type(t)))


def make_config(**overrides):
    """Library defaults overridden by B200COLL_* environment variables, then by keyword arguments.

    Follows the reference's ENV idiom for tunables (util/collective/const.py:24-33).
    """
    cfg = N.default_config()
    env = {
        "B200COLL_STAGING_MB": ("staging_bytes", lambda v: int(v) << 20),
        "B200COLL_SYMMETRIC_MB": ("symmetric_bytes", lambda v: int(v) << 20),
        "B200COLL_MAX_BLOCKS": ("max_blocks", int),
        "B200COLL_ONESHOT_MAX_BYTES": ("oneshot_max_bytes", int),
        "B200COLL_NVLS_MIN_BYTES": ("nvls_min_bytes", int),
        "B200COLL_NVLS_PIPE_MIN_BYTES": ("nvls_pipe_min_bytes", int),
        "B200COLL_GRANULE_BYTES": ("granule_bytes", int),
        "B200COLL_LL_MAX_BYTES": ("ll_max_bytes", int),
        "B200COLL_BCAST_ROUNDS_MIN_BYTES": ("bcast_rounds_min_bytes", int),
        "B200COLL_NVLS_BLOCKS": ("nvls_blocks", int),
        "B200COLL_NVLS_LANES": ("nvls_lanes", int),
        "B200COLL_LANE_GRANULE_BYTES": ("lane_granule_bytes", int),
        "B200COLL_NVLS_LANES_MIN_BYTES": ("nvls_lanes_min_bytes", int),
        "B200COLL_NVLS_STREAMS_MIN_BYTES": ("nvls_streams_min_bytes", int),
        "B200COLL_NVLS_STREAMS_PIECE_BYTES": ("nvls_streams_piece_bytes", int),
        "B200COLL_TIMEOUT_MS": ("timeout_ms", int),
        "B200COLL_P2P_SLOT_BYTES": ("p2p_slot_bytes", int),
        "B200COLL_P2P_SLOTS": ("p2p_slots", int),
    }
    for name, (field, conv) in env.items():
        if name in os.environ:
            setattr(cfg, field, conv(os.environ[name]))
    mode = os.environ.get("B200COLL_SHARE", "vmm").lower()
    if mode not in ("vmm", "ipc"):
        raise ValueError("B200COLL_SHARE must be 'vmm' or 'ipc'")
    cfg.share_mode = N.SHARE_VMM_FD if mode == "vmm" else N.SHARE_LEGACY_IPC
    for k, v in overrides.items():
        setattr(cfg, k, v)
    return cfg


class PeerMemoryComm:
    """Owns one native communicator; shared by B200Group, B200Communicator and the DDP hook."""

    def __init__(self, world_size: int, rank: int, key: str, device: Optional[int] = None,
                 store: Optional[rendezvous.Store] = None, config=None, timeout_s: Optional[float] = None):
        import torch

        if not torch.cuda.is_available():
            raise RuntimeError("B200 backend requires a CUDA device; there is no CPU fallback.")
        self.lib = N.load()
        self.world_size, self.rank, self.key = world_size, rank, key
        self.device = torch.cuda.current_device() if device is None else int(device)
        self.config = config if config is not None else make_config()
        self.store = store if store is not None else rendezvous.default_store()
        if timeout_s is None:
            timeout_s = float(os.environ.get("B200COLL_RENDEZVOUS_TIMEOUT_S", "180"))
        want_mc = os.environ.get("B200COLL_MULTICAST", "1") != "0"
        handle = ctypes.c_void_p()
        N.check(self.lib.b200c_comm_create(rank, world_size, self.device, ctypes.byref(self.config), ctypes.byref(handle)))
        self.handle = handle
        try:
            self.multicast, self.epoch = rendezvous.establish(handle, self.store, key, rank, world_size, self.config.share_mode,
                                                              want_mc, timeout_s)
        except BaseException:
            self.lib.b200c_comm_destroy(handle)
            self.handle = None
            raise
        self._last_stream = None

    # -- stream discipline: ops of one communicator must execute in issue order ------------------
    def stream(self):
        """Current torch stream.  If the caller switched streams since the previous op, the new stream
        first waits for everything queued on the old one, so the double-buffered staging stays
        ordered.  Costs nothing while the caller stays on one stream."""
        import torch

        cur = torch.cuda.current_stream(self.device)
        last = self._last_stream
        if last is None:
            self._last_stream = cur
        elif last != cur:
            ev = torch.cuda.Event()
            ev.record(last)
            cur.wait_event(ev)
            self._last_stream = cur
        return cur

    def check(self):
        N.check(self.lib.b200c_comm_check(self.handle))

    def abort(self):
        if self.handle is not None:
            self.lib.b200c_comm_abort(self.handle)

    def destroy(self):
        if self.handle is not None:
            h, self.handle = self.handle, None
            self.lib.b200c_comm_destroy(h)  # the rendezvous keys were already deleted when establish() finished

    def symmetric_tensor(self, shape, dtype, byte_offset: int = 0):
        """A torch tensor aliasing this rank's symmetric region at `byte_offset`.  The same offset
        names the same logical buffer on every rank; collectives on such a tensor run zero-copy
        (NVLS reduces and broadcasts it in place)."""
        import torch

        base = self.lib.b200c_comm_symmetric_base(self._h())
        total = int(self.lib.b200c_comm_symmetric_bytes(self._h()))
        numel = 1
        for d in (shape if isinstance(shape, (tuple, list)) else (shape,)):
            numel *= int(d)
        nbytes = numel * torch.empty((), dtype=dtype).element_size()
        if not base or byte_offset % 16 or byte_offset + nbytes > total:
            raise RuntimeError(f"symmetric region too small or offset unaligned: need {byte_offset}+{nbytes} of {total} bytes "
                               "(set B200COLL_SYMMETRIC_MB / config.symmetric_bytes)")

        class _Holder:
            __cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (base + byte_offset, False), "version": 2}

        raw = torch.as_tensor(_Holder(), device=torch.device("cuda", self.device))
        return raw.view(dtype).view(shape)

    def symmetric_pool(self):
        """A torch.cuda.MemPool backed by this communicator's symmetric region: tensors allocated under
        `torch.cuda.use_mem_pool(pool)` — including DistributedDataParallel's gradient buckets when the model is
        wrapped inside the context — are peer-mapped and multicast-bound, so in-place collectives on them run
        zero-copy.  Every rank must allocate the same sequence of sizes inside the pool (offsets are matched
        across ranks; a divergence is reported as a mismatch by the collective, not silently reduced).
        One communicator per process can back the pool at a time."""
        import torch

        if int(self.lib.b200c_comm_symmetric_bytes(self._h())) == 0:
            raise RuntimeError("the communicator has no symmetric region: set config.symmetric_bytes / B200COLL_SYMMETRIC_MB")
        N.check(self.lib.b200c_pool_bind(self._h()))
        if getattr(self, "_pool", None) is None:
            alloc = torch.cuda.memory.CUDAPluggableAllocator(N.library_path(), "b200c_pool_malloc", "b200c_pool_free")
            self._pool_allocator = alloc
            self._pool = torch.cuda.MemPool(alloc.allocator())
        return self._pool

    def _h(self):
        if self.handle is None:
            raise RuntimeError("B200 communicator has been destroyed.")
        return self.handle

    # -- thin typed wrappers (pointers, counts, enums; one ctypes call each) ----------------------
    def allreduce(self, send_ptr, recv_ptr, count, dtype, op, algo=N.ALGO_AUTO):
        s = self.stream()
        N.check(self.lib.b200c_allreduce(self._h(), send_ptr, recv_ptr, count, dtype, op, algo, s.cuda_stream))

    def allreduce_scaled(self, send_ptr, recv_ptr, count, dtype, wire_dtype, scale, algo=N.ALGO_AUTO):
        s = self.stream()
        N.check(self.lib.b200c_allreduce_scaled(self._h(), send_ptr, recv_ptr, count, dtype, wire_dtype, scale, algo,
                                                s.cuda_stream))

    def reduce(self, send_ptr, recv_ptr, count, dtype, op, root):
        s = self.stream()
        N.check(self.lib.b200c_reduce(self._h(), send_ptr, recv_ptr, count, dtype, op, root, s.cuda_stream))

    def broadcast(self, ptr, count, dtype, root):
        s = self.stream()
        N.check(self.lib.b200c_broadcast(self._h(), ptr, count, dtype, root, s.cuda_stream))

    def allgather(self, send_ptr, recv_ptrs: List[int], count, dtype):
        s = self.stream()
        arr = (ctypes.c_void_p * len(recv_ptrs))(*recv_ptrs)
        N.check(self.lib.b200c_allgather(self._h(), send_ptr, arr, count, dtype, s.cuda_stream))

    def reducescatter(self, send_ptrs: List[int], recv_ptr, count, dtype, op):
        s = self.stream()
        arr = (ctypes.c_void_p * len(send_ptrs))(*send_ptrs)
        N.check(self.lib.b200c_reducescatter(self._h(), arr, recv_ptr, count, dtype, op, s.cuda_stream))

    def reducescatter_scaled(self, send_ptrs: List[int], recv_ptr, count, dtype, wire_dtype, scale):
        s = self.stream()
        arr = (ctypes.c_void_p * len(send_ptrs))(*send_ptrs)
        N.check(self.lib.b200c_reducescatter_scaled(self._h(), arr, recv_ptr, count, dtype, wire_dtype, scale, s.cuda_stream))

    def send(self, ptr, nbytes, peer, stream=None):
        s = self.stream() if stream is None else stream
        N.check(self.lib.b200c_send(self._h(), ptr, nbytes, peer, s.cuda_stream))

    def recv(self, ptr, nbytes, peer, stream=None):
        s = self.stream() if stream is None else stream
        N.check(self.lib.b200c_recv(self._h(), ptr, nbytes, peer, s.cuda_stream))

    def send_multi(self, ptr, nbytes, peers: List[int], stream=None):
        """One payload to several readers (one multicast store stream when the NVSwitch object is bound)."""
        s = self.stream() if stream is None else stream
        arr = (ctypes.c_int * len(peers))(*peers)
        N.check(self.lib.b200c_send_multi(self._h(), ptr, nbytes, arr, len(peers), s.cuda_stream))

    def recv_multi(self, ptr, nbytes, src, stream=None):
        s = self.stream() if stream is None else stream
        N.check(self.lib.b200c_recv_multi(self._h(), ptr, nbytes, src, s.cuda_stream))

    def barrier(self):
        s = self.stream()
        N.check(self.lib.b200c_barrier(self._h(), s.cuda_stream))
        return s


def next_comm_key(group_name: str) -> str:
    """Key of the n-th incarnation of a group name in this process.  Only for callers whose ranks are
    all created and re-created in lock step inside one job (the gloo test oracle, bench.py); the
    B200 group itself uses `group_key`, which carries no process-local state."""
    with _incarnations_lock:
        n = _incarnations.get(group_name, 0)
        _incarnations[group_name] = n + 1
    return f"b200coll/{group_name}/{n}"


def group_key(group_name: str) -> str:
    """Rendezvous prefix of a named group.  Incarnations are told apart by the random epoch rank 0
    publishes at every creation (rendezvous._agree_on_epoch), not by a per-process counter, so groups
    may be destroyed and re-created under the same name (single_node_cpu_tests/test_allreduce.py:37-59)
    and a single restarted actor still meets its surviving peers."""
    return f"b200coll/{group_name}"


class B200Group:
    """Collective group over peer-mapped HBM.  Duck-types the reference's BaseGroup."""

    def __init__(self, world_size: int, rank: int, group_name: str, store: Optional[rendezvous.Store] = None,
                 device: Optional[int] = None, config=None):
        if world_size > N.MAX_RANKS:
            raise RuntimeError(
                "B200 backend spans one NVSwitch domain: world_size {} > {} (cross-node groups are out of scope; "
                "use the reference's NCCL/gloo backends for those).".format(world_size, N.MAX_RANKS))
        self._world_size, self._rank, self._group_name = world_size, rank, group_name
        self._store, self._device, self._config = store, device, config
        self._comm: Optional[PeerMemoryComm] = None
        self._destroyed = False
        self._key = group_key(group_name)

    # -- BaseGroup surface ----------------------------------------------------------------------
    @property
    def rank(self):
        return self._rank

    @property
    def world_size(self):
        return self._world_size

    @property
    def group_name(self):
        return self._group_name

    @classmethod
    def backend(cls):
        return Backend.B200

    def destroy_group(self):
        self._destroyed = True
        if self._comm is not None:
            self._comm.destroy()
            self._comm = None

    def check(self, synchronize: bool = False):
        """Raise if a kernel of this group recorded a failure (peer timeout, abort, argument mismatch).
        Collectives are asynchronous like NCCL's: a device-side failure is otherwise only seen by the
        next call.  `synchronize=True` first waits for the work queued so far."""
        if self._comm is None:
            return
        if synchronize:
            import torch

            torch.cuda.current_stream(self._comm.device).synchronize()
            if self._comm._last_stream is not None:
                self._comm._last_stream.synchronize()
        self._comm.check()

    def comm(self, device: Optional[int] = None) -> PeerMemoryComm:
        """The lazily-created communicator (first op decides the device, like the reference's
        per-device-list communicator cache)."""
        if self._destroyed:
            raise RuntimeError("The collective group '{}' has been destroyed.".format(self._group_name))
        if self._comm is None:
            dev = self._device if self._device is not None else device
            self._comm = PeerMemoryComm(self._world_size, self._rank, self._key, dev, self._store, self._config)
        elif device is not None and device != self._comm.device:
            raise RuntimeError("Tensor is on cuda:{} but group '{}' is bound to cuda:{} (one GPU per process).".format(
                device, self._group_name, self._comm.device))
        return self._comm

    @staticmethod
    def _single(tensors, what="tensors") -> TensorView:
        if not tensors or not isinstance(tensors, list):
            raise RuntimeError("'{}' must be a nonempty list.".format(what))
        if len(tensors) != 1:
            raise RuntimeError(
                "B200 backend runs one process per GPU: expected a single tensor, got {} "
                "(the multi-GPU-per-process *_multigpu calls are not supported).".format(len(tensors)))
        return TensorView(tensors[0])

    def _list(self, tensor_lists, like: TensorView) -> List[TensorView]:
        if not tensor_lists or not isinstance(tensor_lists, list) or len(tensor_lists) != 1:
            raise RuntimeError("The second argument 'tensor_lists' expects a list holding one tensor list.")
        lst = tensor_lists[0]
        if not isinstance(lst, list) or len(lst) != self._world_size:
            raise RuntimeError("The tensor list must hold exactly world_size ({}) tensors.".format(self._world_size))
        views = [TensorView(t) for t in lst]
        for v in views:
            # exact dtype and shape match, as _check_inputs_compatibility_for_scatter_gather enforces
            # (nccl_collective_group.py:710-751)
            if v.dtype != like.dtype:
                raise RuntimeError("All tensor operands to scatter/gather must have the same dtype.")
            if v.shape != like.shape:
                raise RuntimeError("All tensor operands to scatter/gather must have the same shape. "
                                   "Got '{}' and '{}'.".format(v.shape, like.shape))
        return views

    def allreduce(self, tensors, allreduce_options=AllReduceOptions()):
        v = self._single(tensors)
        op = native_reduce_op(allreduce_options.reduceOp, v.is_bool)
        self.comm(v.device).allreduce(v.ptr, v.ptr, v.numel, v.dtype, op)

    def barrier(self, barrier_options=BarrierOptions()):
        c = self.comm()
        c.barrier().synchronize()
        c.check()

    def reduce(self, tensors, reduce_options=ReduceOptions()):
        v = self._single(tensors)
        op = native_reduce_op(reduce_options.reduceOp, v.is_bool)
        self.comm(v.device).reduce(v.ptr, v.ptr, v.numel, v.dtype, op, reduce_options.root_rank)

    def broadcast(self, tensors, broadcast_options=BroadcastOptions()):
        v = self._single(tensors)
        self.comm(v.device).broadcast(v.ptr, v.numel, v.dtype, broadcast_options.root_rank)

    def allgather(self, tensor_lists, tensors, allgather_options=AllGatherOptions()):
        v = self._single(tensors)
        outs = self._list(tensor_lists, v)
        self.comm(v.device).allgather(v.ptr, [o.ptr for o in outs], v.numel, v.dtype)

    def reducescatter(self, tensors, tensor_lists, reducescatter_options=ReduceScatterOptions()):
        v = self._single(tensors)
        ins = self._list(tensor_lists, v)
        op = native_reduce_op(reducescatter_options.reduceOp, v.is_bool)
        self.comm(v.device).reducescatter([i.ptr for i in ins], v.ptr, v.numel, v.dtype, op)

    def send(self, tensors, send_options=SendOptions()):
        v = self._single(tensors)
        if send_options.dst_rank == self._rank:
            raise RuntimeError("Send and recv happens on the same process.")
        n = send_options.n_elements if send_options.n_elements > 0 else v.numel
        self.comm(v.device).send(v.ptr, n * v.itemsize, send_options.dst_rank)

    def recv(self, tensors, recv_options=RecvOptions()):
        v = self._single(tensors)
        if recv_options.src_rank == self._rank:
            raise RuntimeError("Send and recv happens on the same process.")
        n = recv_options.n_elements if recv_options.n_elements > 0 else v.numel
        self.comm(v.device).recv(v.ptr, n * v.itemsize, recv_options.src_rank)
