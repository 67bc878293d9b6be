"""Host-side rendezvous plumbing (no GPU): stores, fd passing over SCM_RIGHTS, world_size-2
exchange through real processes."""
import os
import threading

import pytest

from mini_actor import get, spawn

from ant_ray_b200 import rendezvous as R


def test_filestore_set_get_delete(tmp_path):
    s = R.FileStore(str(tmp_path))
    s.set("a/b/0", b"hello")
    assert s.get("a/b/0", 1) == b"hello"
    s.delete("a/b/0")
    with pytest.raises(R.RendezvousTimeout):
        s.get("a/b/0", 0.05)


def test_filestore_get_blocks_until_set(tmp_path):
    s = R.FileStore(str(tmp_path))
    threading.Timer(0.1, lambda: s.set("k", b"v")).start()
    assert s.get("k", 5) == b"v"


def test_torchstore_adapter(tmp_path):
    import torch.distributed as dist

    ts = R.TorchStore(dist.FileStore(str(tmp_path / "f"), 1))
    ts.set("x", b"1")
    assert ts.get("x", 1) == b"1"
    with pytest.raises(R.RendezvousTimeout):
        ts.get("missing", 0.2)


def test_default_store_from_env(tmp_path, monkeypatch):
    monkeypatch.setenv("B200COLL_STORE", f"file://{tmp_path}")
    assert isinstance(R.default_store(), R.FileStore)
    monkeypatch.setenv("B200COLL_STORE", "bogus://x")
    with pytest.raises(ValueError):
        R.default_store()
    monkeypatch.delenv("B200COLL_STORE")
    with pytest.raises(RuntimeError):
        R.default_store()


def test_fd_passing_same_process():
    server = R.FdServer()
    r, w = os.pipe()
    try:
        server.offer(0, b"payload-bytes", r)
        data, fd = R.fetch_fd(server.address, 1, 0, 5)
        assert data == b"payload-bytes"
        os.write(w, b"through the duplicated descriptor")
        assert os.read(fd, 100) == b"through the duplicated descriptor"
        os.close(fd)
    finally:
        server.close()
        os.close(r)
        os.close(w)


class _Peer:
    """One rank of a world_size-2 exchange: publishes a socket address through the store, serves a
    memfd to the other rank and fetches the other rank's memfd (the shape of establish())."""

    def __init__(self, rank, store_dir):
        self.rank, self.store = rank, R.FileStore(store_dir)

    def exchange(self):
        fd = os.memfd_create(f"rank{self.rank}")
        os.write(fd, f"arena of rank {self.rank}".encode())
        server = R.FdServer()
        try:
            server.offer(0, f"export-{self.rank}".encode(), fd)
            addrs = R._barrier(self.store, "t", "addr", self.rank, 2, 30, server.address.encode())
            data, pfd = R.fetch_fd(addrs[1 - self.rank], self.rank, 0, 30)
            os.lseek(pfd, 0, os.SEEK_SET)
            content = os.read(pfd, 100).decode()
            os.close(pfd)
            R._barrier(self.store, "t", "done", self.rank, 2, 30)
            return data.decode(), content
        finally:
            server.close()
            os.close(fd)


def test_fd_exchange_between_two_processes(store_dir):
    actors = [spawn(_Peer, r, store_dir) for r in range(2)]
    try:
        res = get([a.exchange.remote() for a in actors])
        assert res[0] == ("export-1", "arena of rank 1")
        assert res[1] == ("export-0", "arena of rank 0")
    finally:
        for a in actors:
            a.kill()


def test_barrier_times_out_when_a_rank_is_missing(tmp_path):
    with pytest.raises(R.RendezvousTimeout):
        R._barrier(R.FileStore(str(tmp_path)), "p", "x", 0, 2, 0.1)


def test_epoch_of_a_dead_incarnation_is_ignored(tmp_path):
    """Stores outlive processes: an epoch published by a process that no longer exists (crashed job, group
    never destroyed) must not be picked up; the live rank 0's epoch is."""
    import subprocess
    import sys

    store = R.FileStore(str(tmp_path))
    p = subprocess.Popen([sys.executable, "-c", "pass"])
    p.wait()
    store.set("g/epoch", f"stale-epoch:{p.pid}:12345".encode())
    with pytest.raises(R.RendezvousTimeout):
        R._agree_on_epoch(store, "g", 1, 0.3)
    # same pid alive but another start time (pid reuse) is stale too
    store.set("g/epoch", f"stale-epoch:{os.getpid()}:1".encode())
    with pytest.raises(R.RendezvousTimeout):
        R._agree_on_epoch(store, "g", 1, 0.3)
    got = []
    t = threading.Thread(target=lambda: got.append(R._agree_on_epoch(store, "g", 1, 10)))
    t.start()
    fresh = R._agree_on_epoch(store, "g", 0, 10)
    t.join(10)
    assert got == [fresh] and fresh != "stale-epoch"


def test_in_process_fetch_takes_the_descriptor_directly():
    """Ranks in one process (a loopback world) take the offered fd from the serving FdServer (a duplicate), with
    the socket path's rules: rank in range and not the server's own, each (rank, kind) served once."""
    server = R.FdServer(world=3, rank=0)
    r, w = os.pipe()
    try:
        server.offer(0, b"x", r)
        with pytest.raises(OSError):
            R._fetch_from_peer(server.address.encode(), 5, 0, 2)   # rank out of range
        with pytest.raises(OSError):
            R._fetch_from_peer(server.address, 0, 0, 2)            # the server's own rank
        data, fd = R._fetch_from_peer(server.address.encode(), 1, 0, 5)
        assert data == b"x" and fd != r
        os.write(w, b"dup")
        assert os.read(fd, 10) == b"dup"
        os.close(fd)
        with pytest.raises(OSError):
            R._fetch_from_peer(server.address, 1, 0, 2)            # already served
        with pytest.raises(R.RendezvousTimeout):
            server.take(2, 1, 0.05)                                # nothing offered under kind 1
        data, fd = server.take(2, 0, 5)                            # another rank is still served
        os.close(fd)
        assert server.rejected == 0                                # nothing went through the socket
    finally:
        server.close()
        os.close(r)
        os.close(w)
    # a closed server is no longer reachable in-process: the socket path is tried (and nobody listens)
    with pytest.raises(R.RendezvousTimeout):
        R._fetch_from_peer(server.address, 1, 0, 0.2)


def test_fd_server_authenticates_requests():
    """The abstract socket has no file permissions: requests are checked (peer uid, rank in range, pid of
    the published group member, one fd per (rank, kind))."""
    server = R.FdServer(world=2, rank=0)
    r, w = os.pipe()
    try:
        server.offer(0, b"x", r)
        server.allow([os.getpid(), os.getpid()])
        with pytest.raises(OSError):
            R.fetch_fd(server.address, 5, 0, 2)       # rank out of range
        with pytest.raises(OSError):
            R.fetch_fd(server.address, 0, 0, 2)       # the server's own rank
        data, fd = R.fetch_fd(server.address, 1, 0, 5)
        os.close(fd)
        assert data == b"x"
        with pytest.raises(OSError):
            R.fetch_fd(server.address, 1, 0, 2)       # already served
        assert server.rejected == 3
        server2 = R.FdServer(world=2, rank=0)
        try:
            server2.offer(0, b"x", r)
            server2.allow([os.getpid(), 1])           # rank 1 is some other process
            with pytest.raises(OSError):
                R.fetch_fd(server2.address, 1, 0, 2)
        finally:
            server2.close()
    finally:
        server.close()
        os.close(r)
        os.close(w)


def test_ray_internal_kv_store_against_a_stand_in(monkeypatch):
    """RayKVStore (the store default_store() picks inside Ray — the channel the reference's gloo rendezvous uses,
    collective.py:93-110) against an in-process stand-in for ray.experimental.internal_kv: Ray is not installed here."""
    import sys
    import types

    table = {}
    kv = types.ModuleType("ray.experimental.internal_kv")
    kv._internal_kv_put = lambda k, v, overwrite=True: table.__setitem__(k, v)
    kv._internal_kv_get = lambda k: table.get(k)
    kv._internal_kv_del = lambda k: table.pop(k)
    ray = types.ModuleType("ray")
    ray.is_initialized = lambda: True
    ray.experimental = types.ModuleType("ray.experimental")
    ray.experimental.internal_kv = kv
    for name, mod in (("ray", ray), ("ray.experimental", ray.experimental), ("ray.experimental.internal_kv", kv)):
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.delenv("B200COLL_STORE", raising=False)
    s = R.default_store()
    assert isinstance(s, R.RayKVStore)
    s.set("b200coll/g/0/addr/1", b"abc")
    assert s.get("b200coll/g/0/addr/1", 1) == b"abc" and table == {"b200coll/g/0/addr/1": b"abc"}
    threading.Timer(0.05, lambda: s.set("late", b"v")).start()
    assert s.get("late", 5) == b"v"
    s.delete("late")
    s.delete("late")   # deleting a missing key is not an error
    with pytest.raises(R.RendezvousTimeout):
        s.get("late", 0.05)
    # the epoch agreement and a two-rank key exchange run over it like over any other store
    out = {}

    def rank(r):
        out[r] = R._agree_on_epoch(s, "b200coll/kvtest", r, 5)

    ts = [threading.Thread(target=rank, args=(r,)) for r in (0, 1)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert out[0] == out[1] and out[0]
