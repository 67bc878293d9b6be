"""Host-side rendezvous for a peer-memory group: exchange arena handles, bind multicast.

Replaces the reference's NCCL unique-id rendezvous (nccl_collective_group.py:29-118: a detached
named actor `NCCLUniqueIDStore` holding 128 bytes, polled every second) and the gloo one
(collective.py:93-110: rank 0 publishes `addr:port` in the GCS internal KV, others poll every
50 ms).  Same idea — a tiny key/value channel that every rank can reach — but what travels is:

  * SHARE_LEGACY_IPC: the 64-byte cudaIpcMemHandle_t, as plain bytes through the store itself
    (north_star: "CUDA-IPC handles exchanged through the object store");
  * SHARE_VMM_FD: a POSIX file descriptor, which cannot be pickled, so the store only carries
    the address of a per-rank Unix socket and the fd goes over it with SCM_RIGHTS.

Stores: Ray's internal KV when running inside Ray, a torch.distributed Store (TCPStore /
the default process group's store) under torchrun / Ray Train, or a directory on a shared
filesystem (FileStore: /dev/shm) for plain processes on one box.
"""
import ctypes
import os
import socket
import struct
import threading
import time
import uuid
from typing import List, Optional

from . import _native as N


class RendezvousTimeout(TimeoutError):
    pass


class Store:
    """Minimal KV interface: set(key, bytes), get(key, timeout_s) -> bytes (blocks), delete(key)."""

    def set(self, key: str, value: bytes) -> None:
        raise NotImplementedError

    def get(self, key: str, timeout_s: float) -> bytes:
        raise NotImplementedError

    def delete(self, key: str) -> None:  # best effort
        pass


class FileStore(Store):
    """Directory-backed store; one file per key, written atomically (write + rename)."""

    def __init__(self, root: str):
        self.root = root
        os.makedirs(root, exist_ok=True)

    def _path(self, key):
        return os.path.join(self.root, key.replace("/", "__"))

    def set(self, key, value):
        path = self._path(key)
        tmp = f"{path}.tmp.{os.getpid()}.{threading.get_ident()}"
        with open(tmp, "wb") as f:
            f.write(value)
        os.replace(tmp, path)

    def get(self, key, timeout_s):
        path = self._path(key)
        deadline = time.monotonic() + timeout_s
        delay = 0.0005
        while True:
            try:
                with open(path, "rb") as f:
                    return f.read()
            except FileNotFoundError:
                pass
            if time.monotonic() > deadline:
                raise RendezvousTimeout(f"timed out after {timeout_s}s waiting for key '{key}' in {self.root}")
            time.sleep(delay)
            delay = min(delay * 2, 0.05)

    def delete(self, key):
        try:
            os.unlink(self._path(key))
        except FileNotFoundError:
            pass


class TorchStore(Store):
    """Adapter over a torch.distributed Store (TCPStore, FileStore, PrefixStore...)."""

    def __init__(self, store):
        self.store = store

    def set(self, key, value):
        self.store.set(key, value)

    def get(self, key, timeout_s):
        from datetime import timedelta

        try:
            self.store.wait([key], timedelta(seconds=timeout_s))
        except Exception as e:  # torch raises RuntimeError / DistStoreError on timeout
            raise RendezvousTimeout(f"timed out after {timeout_s}s waiting for key '{key}': {e}") from e
        return bytes(self.store.get(key))

    def delete(self, key):
        try:
            self.store.delete_key(key)
        except Exception:
            pass


class RayKVStore(Store):
    """Ray GCS internal KV (the channel the reference's gloo rendezvous uses, collective.py:93-110)."""

    def __init__(self):
        import ray.experimental.internal_kv as kv

        self.kv = kv

    def set(self, key, value):
        self.kv._internal_kv_put(key, value, overwrite=True)

    def get(self, key, timeout_s):
        deadline = time.monotonic() + timeout_s
        while True:
            v = self.kv._internal_kv_get(key)
            if v is not None:
                return v
            if time.monotonic() > deadline:
                raise RendezvousTimeout(f"timed out after {timeout_s}s waiting for key '{key}' in Ray internal KV")
            time.sleep(0.005)

    def delete(self, key):
        try:
            self.kv._internal_kv_del(key)
        except Exception:
            pass


def default_store() -> Store:
    """Resolve the store when the caller did not pass one.

    Order: $B200COLL_STORE (file://DIR or tcp://HOST:PORT) > Ray internal KV (inside Ray) >
    torch.distributed default store (torchrun / Ray Train) > error.
    """
    spec = os.environ.get("B200COLL_STORE")
    if spec:
        if spec.startswith("file://"):
            return FileStore(spec[len("file://"):])
        if spec.startswith("tcp://"):
            import torch.distributed as dist

            host, port = spec[len("tcp://"):].rsplit(":", 1)
            is_master = os.environ.get("B200COLL_STORE_MASTER", "0") == "1"
            return TorchStore(dist.TCPStore(host, int(port), is_master=is_master, wait_for_workers=False))
        raise ValueError(f"B200COLL_STORE must be file://DIR or tcp://HOST:PORT, got '{spec}'")
    try:
        import ray

        if ray.is_initialized():
            return RayKVStore()
    except ImportError:
        pass
    try:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            return TorchStore(dist.distributed_c10d._get_default_store())
    except Exception:
        pass
    raise RuntimeError(
        "no rendezvous store: run inside Ray, initialise torch.distributed, or set "
        "B200COLL_STORE=file:///dev/shm/<dir> (single box) / tcp://host:port")


# --------------------------------------------------------------------------------------------
# fd passing (SCM_RIGHTS) over an abstract-namespace Unix socket
# --------------------------------------------------------------------------------------------
_REQ = struct.Struct("<ii")  # (requester rank, kind) kind: 0 = arena export, 1 = multicast fd
_LOCAL_SERVERS = {}  # address -> FdServer of this process (see FdServer.take)
_LOCAL_LOCK = threading.Lock()


class FdServer:
    """Serves this rank's exported fds to its peers.  One short-lived thread per group.

    The socket lives in the abstract namespace (no filesystem permissions), so every request is
    authenticated with SO_PEERCRED: the peer must run under this process's uid and — once the group's
    pids are known (`allow`) — be one of the group's processes; the claimed rank must be in range and
    each (rank, kind) is served once."""

    def __init__(self, world: Optional[int] = None, rank: Optional[int] = None):
        self.sock = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        self.address = "\0b200coll-" + uuid.uuid4().hex
        self.sock.bind(self.address)
        self.sock.listen(64)
        self.sock.settimeout(0.1)
        self.world, self.rank = world, rank
        self.payloads = {}  # kind -> (bytes, fd)
        self.allowed_pids = None  # rank -> pid, set by allow()
        self.served = set()
        self.rejected = 0
        self.lock = threading.Lock()
        self.stop = threading.Event()
        self.thread = threading.Thread(target=self._serve, name="b200coll-fd-server", daemon=True)
        self.thread.start()
        with _LOCAL_LOCK:
            _LOCAL_SERVERS[self.address] = self

    def offer(self, kind: int, data: bytes, fd: int):
        with self.lock:
            self.payloads[kind] = (data, fd)

    def allow(self, pids):
        """pids[r] = process id of rank r (as published through the store)."""
        with self.lock:
            self.allowed_pids = dict(enumerate(pids))

    def _authorised(self, conn, rank: int, kind: int) -> bool:
        try:
            pid, uid, _gid = struct.unpack("3i", conn.getsockopt(socket.SOL_SOCKET, socket.SO_PEERCRED, struct.calcsize("3i")))
        except OSError:
            return False
        if uid != os.getuid():
            return False
        if self.world is not None and not (0 <= rank < self.world and rank != self.rank):
            return False
        deadline = time.monotonic() + 60
        while self.world is not None:  # group servers wait for the pid list; ad-hoc servers (tests) skip it
            with self.lock:
                allowed = self.allowed_pids
            if allowed is not None:
                if allowed.get(rank) != pid:
                    return False
                break
            if time.monotonic() > deadline or self.stop.is_set():
                return False
            time.sleep(0.001)
        with self.lock:
            if (rank, kind) in self.served:
                return False
            self.served.add((rank, kind))
        return True

    def take(self, rank: int, kind: int, timeout_s: float):
        """In-process counterpart of fetch_fd for a peer rank in this very process (a loopback world):
        (payload bytes, a duplicate of the offered fd).  Same rank / served-once rules as the socket path;
        no descriptor has to cross a socket, which not every container runtime allows for CUDA's
        shareable-handle fds."""
        if self.world is not None and not (0 <= rank < self.world and rank != self.rank):
            raise OSError(f"rank {rank} may not fetch from rank {self.rank}")
        deadline = time.monotonic() + timeout_s
        while True:
            with self.lock:
                item = self.payloads.get(kind)
                if item is not None:
                    if (rank, kind) in self.served:
                        raise OSError(f"descriptor {kind} already served to rank {rank}")
                    self.served.add((rank, kind))
                    return item[0], os.dup(item[1])
            if time.monotonic() > deadline or self.stop.is_set():
                raise RendezvousTimeout(f"peer offered no descriptor {kind} within {timeout_s}s")
            time.sleep(0.001)

    def _serve(self):
        while not self.stop.is_set():
            try:
                conn, _ = self.sock.accept()
            except socket.timeout:
                continue
            except OSError:
                return
            try:
                conn.settimeout(30)
                raw = b""
                while len(raw) < _REQ.size:
                    part = conn.recv(_REQ.size - len(raw))
                    if not part:
                        break
                    raw += part
                if len(raw) != _REQ.size:
                    continue
                rank, kind = _REQ.unpack(raw)
                if not self._authorised(conn, rank, kind):
                    self.rejected += 1
                    continue
                deadline = time.monotonic() + 60
                while True:
                    with self.lock:
                        item = self.payloads.get(kind)
                    if item is not None or time.monotonic() > deadline or self.stop.is_set():
                        break
                    time.sleep(0.001)
                if item is None:
                    continue
                data, fd = item
                socket.send_fds(conn, [struct.pack("<I", len(data)) + data], [fd])
            except OSError:
                pass
            finally:
                conn.close()

    def close(self):
        self.stop.set()
        with _LOCAL_LOCK:
            _LOCAL_SERVERS.pop(self.address, None)
        try:
            self.sock.close()
        except OSError:
            pass
        self.thread.join(timeout=2)


def _fetch_from_peer(address, my_rank: int, kind: int, timeout_s: float):
    """fetch_fd, or FdServer.take when the serving rank lives in this process."""
    with _LOCAL_LOCK:
        local = _LOCAL_SERVERS.get(address.decode() if isinstance(address, bytes) else address)
    if local is not None:
        return local.take(my_rank, kind, timeout_s)
    return fetch_fd(address, my_rank, kind, timeout_s)


def fetch_fd(address: str, my_rank: int, kind: int, timeout_s: float):
    """Connect to a peer's FdServer and receive (payload bytes, fd)."""
    if isinstance(address, bytes):
        address = address.decode()
    deadline = time.monotonic() + timeout_s
    while True:
        s = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
        try:
            s.settimeout(max(0.1, deadline - time.monotonic()))
            s.connect(address)
            s.sendall(_REQ.pack(my_rank, kind))
            msg, fds, _, _ = socket.recv_fds(s, 4096, 1)
            if not fds or len(msg) < 4:
                raise OSError("peer closed the connection without sending a descriptor")
            (n,) = struct.unpack("<I", msg[:4])
            data = msg[4:]
            while len(data) < n:
                part = s.recv(n - len(data))
                if not part:
                    raise OSError("short read from peer")
                data += part
            return data[:n], fds[0]
        except (ConnectionRefusedError, FileNotFoundError):
            if time.monotonic() > deadline:
                raise RendezvousTimeout(f"could not reach peer socket within {timeout_s}s")
            time.sleep(0.01)
        finally:
            s.close()


# --------------------------------------------------------------------------------------------
# the rendezvous proper
# --------------------------------------------------------------------------------------------
def _barrier(store: Store, prefix: str, tag: str, rank: int, world: int, timeout_s: float, payload: bytes = b"1") -> List[bytes]:
    """All-gather of small payloads through the store; doubles as a barrier."""
    store.set(f"{prefix}/{tag}/{rank}", payload)
    return [store.get(f"{prefix}/{tag}/{r}", timeout_s) for r in range(world)]


def _proc_start_time(pid: int) -> Optional[str]:
    """Kernel start time (clock ticks since boot) of a live process, None if there is no such process.
    (pid, start time) never repeats on a box, unlike the pid alone."""
    try:
        with open(f"/proc/{pid}/stat", "rb") as f:
            stat = f.read().decode(errors="replace")
        return stat[stat.rindex(")") + 2:].split()[19]
    except (OSError, ValueError, IndexError):
        return None


def _agree_on_epoch(store: Store, prefix: str, rank: int, timeout_s: float) -> str:
    """Give this incarnation of the group a fresh key namespace.

    Stores outlive processes (Ray's internal KV, a /dev/shm directory), so keys of an earlier incarnation
    that crashed — or that was never destroyed — may still be there.  Rank 0 publishes a new random epoch
    together with its (pid, start time); the other ranks accept an epoch only from a publisher that is
    alive right now, so a dead incarnation's epoch is ignored until the live rank 0 overwrites it.  Every
    other rendezvous key lives under the epoch; a successful rendezvous deletes all of them, the epoch
    key included (see establish), so a finished incarnation leaves nothing a later one could pick up.
    Nothing is derived from process-local counters: a single restarted actor agrees with its surviving
    peers as soon as they re-create the group."""
    key = f"{prefix}/epoch"
    if rank == 0:
        epoch = uuid.uuid4().hex
        store.set(key, f"{epoch}:{os.getpid()}:{_proc_start_time(os.getpid())}".encode())
        return epoch
    trust = os.environ.get("B200COLL_TRUST_EPOCH") == "1"  # ranks in different pid namespaces cannot check liveness
    deadline = time.monotonic() + timeout_s
    while True:
        try:
            raw = store.get(key, min(0.25, max(0.01, deadline - time.monotonic())))
            epoch, pid, started = raw.decode().split(":")
            if trust or _proc_start_time(int(pid)) == started:
                return epoch
        except RendezvousTimeout:
            pass
        except ValueError:
            pass  # a foreign or half-written value: wait for rank 0
        if time.monotonic() > deadline:
            raise RendezvousTimeout(f"no live rank 0 published an epoch for '{prefix}' within {timeout_s}s")
        time.sleep(0.005)


_TAGS = ("addr", "ipc", "imported", "mc_created", "mc_added", "mc_bound", "ready", "done")


def establish(comm: int, store: Store, prefix: str, rank: int, world: int, share_mode: int,
              want_multicast: bool, timeout_s: float = 60.0) -> bool:
    """Drive a freshly created native communicator (`b200c_comm_create`) to the ready state.

    Returns (multicast, epoch): whether the NVSwitch multicast object is bound on every rank, and the
    random id of this incarnation of the group (the same string on every rank).
    """
    lib = N.load()
    exp = N.Export()
    N.check(lib.b200c_comm_export(comm, ctypes.byref(exp)))
    if world == 1:
        if exp.fd >= 0:
            os.close(exp.fd)
        N.check(lib.b200c_comm_ready(comm))
        return False, uuid.uuid4().hex
    server: Optional[FdServer] = None
    own_fd = exp.fd
    mc_fd_own = -1
    base = prefix
    epoch = None
    ok_all = False
    try:
        epoch = _agree_on_epoch(store, base, rank, timeout_s)
        prefix = f"{base}/{epoch}"
        if share_mode == N.SHARE_VMM_FD:
            server = FdServer(world, rank)
            server.offer(0, bytes(exp), own_fd)
            hello = _barrier(store, prefix, "addr", rank, world, timeout_s, server.address.encode() + b"|" + str(os.getpid()).encode())
            addrs = [h.rsplit(b"|", 1)[0] for h in hello]
            server.allow([int(h.rsplit(b"|", 1)[1]) for h in hello])
            for peer in range(world):
                if peer == rank:
                    continue
                data, fd = _fetch_from_peer(addrs[peer], rank, 0, timeout_s)
                try:
                    pe = N.Export.from_buffer_copy(data)
                    pe.fd = fd
                    N.check(lib.b200c_comm_import(comm, peer, ctypes.byref(pe)))
                finally:
                    os.close(fd)
        else:
            blobs = _barrier(store, prefix, "ipc", rank, world, timeout_s, bytes(exp))
            for peer in range(world):
                if peer == rank:
                    continue
                pe = N.Export.from_buffer_copy(blobs[peer])
                N.check(lib.b200c_comm_import(comm, peer, ctypes.byref(pe)))
        _barrier(store, prefix, "imported", rank, world, timeout_s)

        have_mc = False
        if want_multicast and share_mode == N.SHARE_VMM_FD:
            ok = True
            try:
                if rank == 0:
                    fd = ctypes.c_int(-1)
                    N.check(lib.b200c_comm_mc_create(comm, ctypes.byref(fd)))
                    mc_fd_own = fd.value
                    server.offer(1, b"mc", mc_fd_own)
            except N.B200CollError:
                ok = False
            flags = _barrier(store, prefix, "mc_created", rank, world, timeout_s, b"1" if ok else b"0")
            ok = flags[0] == b"1"
            if ok and rank != 0:
                try:
                    _, fd = _fetch_from_peer(addrs[0], rank, 1, timeout_s)
                    try:
                        N.check(lib.b200c_comm_mc_import(comm, fd))
                    finally:
                        os.close(fd)
                except (N.B200CollError, OSError, RendezvousTimeout):
                    ok = False
            if ok:
                try:
                    N.check(lib.b200c_comm_mc_add_device(comm))
                except N.B200CollError:
                    ok = False
            flags = _barrier(store, prefix, "mc_added", rank, world, timeout_s, b"1" if ok else b"0")
            ok = all(f == b"1" for f in flags)
            if ok:
                try:
                    N.check(lib.b200c_comm_mc_bind(comm))
                except N.B200CollError:
                    ok = False
            flags = _barrier(store, prefix, "mc_bound", rank, world, timeout_s, b"1" if ok else b"0")
            have_mc = all(f == b"1" for f in flags)
            if not have_mc:
                lib.b200c_comm_mc_disable(comm)
        N.check(lib.b200c_comm_ready(comm))
        _barrier(store, prefix, "ready", rank, world, timeout_s)
        # nobody needs the keys any more once every rank has passed "ready": rank 0 collects a "done" from
        # every rank and deletes the whole epoch, so nothing stale is left for a later incarnation
        store.set(f"{prefix}/done/{rank}", b"1")
        if rank == 0:
            for r in range(world):
                store.get(f"{prefix}/done/{r}", timeout_s)
            cleanup_keys(store, prefix, world)
            store.delete(f"{base}/epoch")
        ok_all = True
        return have_mc, epoch
    finally:
        if not ok_all and rank == 0 and epoch is not None:
            # a failed rendezvous must not leave a live-looking epoch behind
            cleanup_keys(store, f"{base}/{epoch}", world)
            store.delete(f"{base}/epoch")
        if server is not None:
            server.close()
        if own_fd >= 0:
            os.close(own_fd)
        if mc_fd_own >= 0:
            os.close(mc_fd_own)


def cleanup_keys(store: Store, prefix: str, world: int):
    for tag in _TAGS:
        for r in range(world):
            store.delete(f"{prefix}/{tag}/{r}")
