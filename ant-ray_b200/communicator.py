"""B200Communicator: the compiled-graph accelerator communicator (R2), replacing _NcclGroup.

`Communicator` restates the 15-method contract of
python/ray/experimental/channel/communicator.py:18-199; inside a Ray installation the real ABC is
used instead so that `isinstance` checks in the DAG compiler hold.  `B200Communicator` keeps the
constructor the registry calls — `Cls(world_size, comm_id, rank, actor_handles, cuda_stream,
use_communication_streams)` (torch_tensor_accelerator_channel.py:673-680) — and the behaviour of
python/ray/experimental/channel/nccl_group.py:21-374:
  * send() returns once the kernel is enqueued (:149-184);
  * recv() allocates through the caller's allocator and enqueues the receive; the reference then
    blocks the host until the data has landed (:186-241) — here the caller's stream waits instead
    and a failure is raised as RayChannelError by the next call / check() / destroy()
    (section 8(f) N4; B200COLL_BLOCKING_ERRORS=1 brings the blocking behaviour back);
  * allgather/allreduce/reducescatter are out of place and raise RayChannelError when the group was
    closed or a peer disagreed on the shape/dtype (:243-333; the reference relies on an NCCL timeout
    there, test_torch_tensor_dag.py:1544-1588 — here the kernels compare op signatures and fail in
    microseconds), again without a host synchronisation unless blocking errors are requested;
  * destroy() sets `_closed` first, then aborts the in-flight kernels (:347-365).
Register it with `register_accelerator_context("cuda", B200Communicator)`
(accelerator_context.py:222-233) or pass an instance as `transport=`.
"""
import os
import uuid
from abc import ABC, abstractmethod
from typing import Callable, Optional, Tuple

from . import _native as N
from .b200_group import PeerMemoryComm, TensorView, native_reduce_op
from .header_ring import HeaderRing, HeaderTimeout, ring_path
from .types import DagReduceOp as ReduceOp

try:  # inside Ray: be a real subclass so the DAG compiler's isinstance checks pass
    from ray.exceptions import RayChannelError
    from ray.experimental.channel.communicator import Communicator
except ImportError:

    class RayChannelError(RuntimeError):
        """Raised when a channel / communicator is closed or failed (ray.exceptions.RayChannelError)."""

    class Communicator(ABC):
        """Contract of ray.experimental.channel.Communicator (communicator.py:18-199)."""

        @abstractmethod
        def initialize(self, rank: int) -> None: ...

        @abstractmethod
        def get_actor_handles(self) -> list: ...

        @abstractmethod
        def get_rank(self, actor) -> int: ...

        @abstractmethod
        def get_self_rank(self) -> Optional[int]: ...

        def get_world_size(self) -> int:
            raise NotImplementedError

        @abstractmethod
        def send(self, value, peer_rank: int) -> None: ...

        @abstractmethod
        def recv(self, shape, dtype, peer_rank: int, allocator=None): ...

        @property
        @abstractmethod
        def recv_stream(self): ...

        @property
        @abstractmethod
        def send_stream(self): ...

        @abstractmethod
        def allgather(self, send_buf, recv_buf) -> None: ...

        @abstractmethod
        def allreduce(self, send_buf, recv_buf, op) -> None: ...

        @abstractmethod
        def reducescatter(self, send_buf, recv_buf, op) -> None: ...

        @abstractmethod
        def destroy(self) -> None: ...

        @abstractmethod
        def get_transport_name(self) -> str: ...

        @classmethod
        @abstractmethod
        def generate_communicator_id(cls) -> str: ...


TorchTensorAllocator = Callable[[Tuple[int], "torch.dtype"], "torch.Tensor"]


def _actor_key(a):
    return getattr(a, "_ray_actor_id", a)


class B200Communicator(Communicator):
    """One actor's endpoint of a peer-memory group.  Not thread-safe (like _NcclGroup).

    Beyond the 15-method contract (all kept) it offers what the reference marks as TODO:
      * no host synchronisation in `recv` and in the collectives (nccl_group.py:215, 237, 266
        "TODO: Avoid CUDA synchronization"): the call returns once the kernel is enqueued and the
        caller's current stream has been made to wait for it, so the buffer is valid for everything
        the caller enqueues next; a failure on the device (closed group, dead peer, shape mismatch)
        is recorded in the communicator's status block and raised as RayChannelError by the next call,
        by `check()` and by `destroy()`.  `B200COLL_BLOCKING_ERRORS=1` (or `blocking_errors=True`)
        restores the reference's blocking behaviour, where the failing call itself raises;
      * `send_multi` / `recv_multi`: one payload to several readers through one multicast store
        stream (torch_tensor_accelerator_channel.py:586-590 "can replace with a broadcast");
      * `send_with_header` / `recv_with_header`: the shape and dtype travel in a binary record next to
        the cell ring instead of a pickled message on a second channel (:574-578, :592-608).
    """

    inline_metadata = True   # TensorListChannel: this communicator carries tensor headers itself
    multi_reader = True      # ... and can deliver one payload to several readers

    def __init__(self, world_size: int, comm_id: str, rank: Optional[int], actor_handles: list,
                 cuda_stream: Optional["torch.cuda.Stream"], use_communication_streams: bool = False,
                 store=None, config=None, blocking_errors: Optional[bool] = None):
        self._world_size = world_size
        self._rank = rank
        self._actor_handles = actor_handles
        self._use_communication_streams = use_communication_streams
        self._comm: Optional[PeerMemoryComm] = None
        self._cuda_stream = self._send_stream = self._recv_stream = None
        self._closed = False
        self._hdr_out, self._hdr_in = {}, {}
        if blocking_errors is None:
            blocking_errors = os.environ.get("B200COLL_BLOCKING_ERRORS", "0") == "1"
        self._blocking_errors = blocking_errors
        if rank is not None:
            import torch

            assert cuda_stream is not None, "B200 actor must specify cuda_stream"
            assert torch.cuda.is_available(), "B200 actor has no GPUs assigned"
            device = cuda_stream.device.index if hasattr(cuda_stream, "device") else torch.cuda.current_device()
            # blocks until the same call has been made on every other actor of the group
            self._comm = PeerMemoryComm(world_size, rank, f"b200coll/cgraph/{comm_id}", device, store, config)
            self._cuda_stream = cuda_stream
            if use_communication_streams:
                self._send_stream = torch.cuda.Stream(device=device)
                self._recv_stream = torch.cuda.Stream(device=device)
            else:
                self._send_stream = self._recv_stream = cuda_stream

    # -- membership ---------------------------------------------------------------------------
    def initialize(self, rank: int) -> None:
        pass  # everything happens in the constructor, as in _NcclGroup

    def get_actor_handles(self) -> list:
        return self._actor_handles

    def get_rank(self, actor) -> int:
        keys = [_actor_key(a) for a in self._actor_handles]
        try:
            return keys.index(_actor_key(actor))
        except ValueError:
            raise ValueError("Actor is not in the B200 group.")

    def get_self_rank(self) -> Optional[int]:
        return self._rank

    def get_world_size(self) -> int:
        return self._world_size

    def get_transport_name(self) -> str:
        return "accelerator"

    @classmethod
    def generate_communicator_id(cls) -> str:
        return uuid.uuid4().hex

    # -- helpers ------------------------------------------------------------------------------
    def _check_open(self):
        if self._closed or self._comm is None or self._comm.handle is None:
            raise RayChannelError("B200 group has been destroyed.")

    def _raise_if_failed(self, what: str):
        if self._closed:
            raise RayChannelError(f"B200 group has been destroyed during {what}.")
        try:
            self._comm.check()
        except N.B200CollError as e:
            raise RayChannelError(f"B200 {what} failed: {e}. There may be a shape or dtype mismatch between "
                                  "the tensors of different ranks, or a peer actor died.") from e

    def check(self, synchronize: bool = True) -> None:
        """Raise RayChannelError if any operation issued so far has failed on the device."""
        self._check_open()
        if synchronize:
            for st in {self._cuda_stream, self._send_stream, self._recv_stream}:
                if st is not None:
                    st.synchronize()
        self._raise_if_failed("operation")

    def _after_enqueue(self, stream, what: str):
        """Make the data produced on `stream` valid for whatever the caller enqueues next, without
        blocking the host (deferred mode), or block and report now (blocking mode)."""
        if self._blocking_errors:
            stream.synchronize()
            self._raise_if_failed(what)
            return
        import torch

        cur = torch.cuda.current_stream(self._comm.device)
        if cur != stream:
            ev = torch.cuda.Event()
            ev.record(stream)
            cur.wait_event(ev)

    def _native(self, fn, *args, **kw):
        try:
            return fn(*args, **kw)
        except N.B200CollError as e:
            # an error recorded by an EARLIER asynchronous operation surfaces here (deferred mode)
            raise RayChannelError(f"B200 group failed: {e}. There may be a shape or dtype mismatch between the tensors of "
                                  "different ranks, or a peer actor died.") from e

    # -- p2p ----------------------------------------------------------------------------------
    def send(self, buf, peer_rank: int) -> None:
        self._check_open()
        if self._use_communication_streams:
            # keep the CPU loop from running arbitrarily far ahead of the GPU (nccl_group.py:168-173)
            self._send_stream.synchronize()
        v = TensorView(buf)
        self._native(self._comm.send, v.ptr, v.numel * v.itemsize, peer_rank, stream=self._send_stream)

    def recv(self, shape, dtype, peer_rank: int, allocator: Optional[TorchTensorAllocator] = None):
        self._check_open()
        assert allocator is not None, "B200 group requires a tensor allocator"
        buf = allocator(shape, dtype)
        if self._use_communication_streams:
            self._recv_stream.synchronize()
        v = TensorView(buf)
        self._native(self._comm.recv, v.ptr, v.numel * v.itemsize, peer_rank, stream=self._recv_stream)
        if not self._use_communication_streams:
            # "After this call returns, the receive buffer is safe to read" — for everything enqueued from now on
            self._after_enqueue(self._recv_stream, "recv")
        return buf

    def send_multi(self, buf, peer_ranks) -> None:
        """One payload for several readers; every reader calls recv_multi(src = this rank)."""
        self._check_open()
        if self._use_communication_streams:
            self._send_stream.synchronize()
        v = TensorView(buf)
        self._native(self._comm.send_multi, v.ptr, v.numel * v.itemsize, list(peer_ranks), stream=self._send_stream)

    def recv_multi(self, shape, dtype, peer_rank: int, allocator: Optional[TorchTensorAllocator] = None):
        self._check_open()
        assert allocator is not None, "B200 group requires a tensor allocator"
        buf = allocator(shape, dtype)
        if self._use_communication_streams:
            self._recv_stream.synchronize()
        v = TensorView(buf)
        self._native(self._comm.recv_multi, v.ptr, v.numel * v.itemsize, peer_rank, stream=self._recv_stream)
        if not self._use_communication_streams:
            self._after_enqueue(self._recv_stream, "recv")
        return buf

    # -- tensor headers (shape, dtype) next to the cell ring ------------------------------------
    def _ring(self, table, src, dst, role):
        ring = table.get((src, dst))
        if ring is None:
            ring = table[(src, dst)] = HeaderRing(ring_path(self._comm.key + "/" + self._comm.epoch, src, dst), role)
        return ring

    def send_with_header(self, buf, peer_ranks, index: int = 0, count: int = 1) -> None:
        """Announce (shape, dtype) to every reader, then send the payload (once, if there are several readers)."""
        self._check_open()
        peers = [peer_ranks] if isinstance(peer_ranks, int) else list(peer_ranks)
        for p in peers:
            self._ring(self._hdr_out, self._rank, p, "w").put(tuple(buf.shape), buf.dtype, index, count)
        if len(peers) == 1:
            self.send(buf, peers[0])
        else:
            self.send_multi(buf, peers)

    def recv_with_header(self, peer_rank: int, allocator: Optional[TorchTensorAllocator] = None, timeout: Optional[float] = None,
                         multi: bool = False):
        """Returns (tensor, index, count): the header says what to allocate."""
        self._check_open()
        try:
            shape, dtype, index, count = self._ring(self._hdr_in, peer_rank, self._rank, "r").get(
                60.0 if timeout is None else timeout, cancelled=lambda: self._closed)
        except HeaderTimeout as e:
            if self._closed:
                raise RayChannelError("B200 group has been destroyed.") from e
            raise TimeoutError(str(e)) from e
        if count == 0:
            return None, 0, 0   # an empty tensor list: a header, no payload
        fn = self.recv_multi if multi else self.recv
        return fn(shape, dtype, peer_rank, allocator), index, count

    def announce_empty(self, peer_ranks) -> None:
        """Tell the readers that this message carries no tensors (a header with count 0, no payload)."""
        self._check_open()
        import torch

        for p in ([peer_ranks] if isinstance(peer_ranks, int) else list(peer_ranks)):
            self._ring(self._hdr_out, self._rank, p, "w").put((), torch.uint8, 0, 0)

    # -- collectives --------------------------------------------------------------------------
    def _exec_collective(self, send_buf, recv_buf, what, fn):
        self._check_open()
        assert send_buf.dtype == recv_buf.dtype, (
            "Ray Compiled Graph derived the dtype of recv_buf from send_buf, so send_buf and recv_buf must have the same dtype.")
        import torch

        with torch.cuda.stream(self._cuda_stream):
            self._native(fn)
        self._after_enqueue(self._cuda_stream, what)

    def allgather(self, send_buf, recv_buf) -> None:
        s, r = TensorView(send_buf), TensorView(recv_buf)
        if r.numel != s.numel * self._world_size:
            raise RayChannelError(f"allgather recv_buf has {r.numel} elements, expected {s.numel * self._world_size}")
        step = s.numel * s.itemsize
        self._exec_collective(send_buf, recv_buf, "allgather",
                              lambda: self._comm.allgather(s.ptr, [r.ptr + j * step for j in range(self._world_size)], s.numel, s.dtype))

    def allreduce(self, send_buf, recv_buf, op=ReduceOp.SUM) -> None:
        s, r = TensorView(send_buf), TensorView(recv_buf)
        if r.numel != s.numel:
            raise RayChannelError(f"allreduce recv_buf has {r.numel} elements, expected {s.numel}")
        nat = native_reduce_op(op, s.is_bool)
        self._exec_collective(send_buf, recv_buf, "allreduce",
                              lambda: self._comm.allreduce(s.ptr, r.ptr, s.numel, s.dtype, nat))

    def reducescatter(self, send_buf, recv_buf, op=ReduceOp.SUM) -> None:
        s, r = TensorView(send_buf), TensorView(recv_buf)
        if s.numel != r.numel * self._world_size:
            raise RayChannelError(f"reducescatter send_buf has {s.numel} elements, expected {r.numel * self._world_size}")
        step = r.numel * r.itemsize
        nat = native_reduce_op(op, s.is_bool)
        self._exec_collective(send_buf, recv_buf, "reducescatter",
                              lambda: self._comm.reducescatter([s.ptr + j * step for j in range(self._world_size)], r.ptr, r.numel,
                                                               r.dtype, nat))

    # -- streams / teardown -------------------------------------------------------------------
    @property
    def recv_stream(self):
        import torch

        return torch.cuda.StreamContext(self._recv_stream)

    @property
    def send_stream(self):
        import torch

        return torch.cuda.StreamContext(self._send_stream)

    def destroy(self) -> None:
        if self._closed:
            return
        self._closed = True  # before the abort, so ops released by it see the flag (nccl_group.py:355-363)
        for ring in list(self._hdr_out.values()) + list(self._hdr_in.values()):
            ring.close(unlink=True)
        if self._comm is not None:
            self._comm.abort()
            self._comm.destroy()
