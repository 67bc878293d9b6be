"""Loopback world: W communicators of ONE process on ONE GPU, each on its own CUDA stream.

The kernels cannot tell the difference: every "peer" arena is a second mapping of memory on the
same device, flags and data travel through local L2/HBM instead of NVLink.  This is how the
single-GPU tiers exercise the real kernels (`__graft_entry__.smoke()`, `pytest -m gpu` on a
one-GPU box, the N=1 bench line).  Because the W kernels of one collective must be co-resident
(each spins on flags the others raise), the per-kernel grid is capped so that W grids fit the
GPU: 2 CTAs of 512 threads per SM (64 registers/thread) -> world * max_blocks <= 2 * SMs.
"""
import threading
from typing import List, Optional

import torch

from . import rendezvous
from .b200_group import PeerMemoryComm, make_config


class _MemStore(rendezvous.Store):
    def __init__(self):
        self.d = {}
        self.cv = threading.Condition()

    def set(self, key, value):
        with self.cv:
            self.d[key] = bytes(value)
            self.cv.notify_all()

    def get(self, key, timeout_s):
        with self.cv:
            if not self.cv.wait_for(lambda: key in self.d, timeout_s):
                raise rendezvous.RendezvousTimeout(f"timed out waiting for '{key}'")
            return self.d[key]

    def delete(self, key):
        with self.cv:
            self.d.pop(key, None)


class LoopbackWorld:
    def __init__(self, world_size: int, device: int = 0, key: str = "loopback", **config_overrides):
        self.world_size, self.device = world_size, device
        sm = torch.cuda.get_device_properties(device).multi_processor_count
        cfg_kw = dict(max_blocks=max(1, min(264, (2 * sm) // world_size - 2)), staging_bytes=32 << 20)
        cfg_kw.update(config_overrides)
        store = _MemStore()
        self.comms: List[Optional[PeerMemoryComm]] = [None] * world_size
        errors = []

        def make(r):
            try:
                with torch.cuda.device(device):
                    self.comms[r] = PeerMemoryComm(world_size, r, key, device, store, make_config(**cfg_kw), timeout_s=60)
            except BaseException as e:  # noqa: BLE001
                errors.append(e)

        import os

        prev = os.environ.get("B200COLL_MULTICAST")
        os.environ["B200COLL_MULTICAST"] = "0"  # a multicast object cannot take the same device twice
        try:
            threads = [threading.Thread(target=make, args=(r,)) for r in range(world_size)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
        finally:
            if prev is None:
                os.environ.pop("B200COLL_MULTICAST", None)
            else:
                os.environ["B200COLL_MULTICAST"] = prev
        if errors:
            self.destroy()
            raise errors[0]
        self.streams = [torch.cuda.Stream(device=device) for _ in range(world_size)]

    def run(self, fn):
        """Call fn(rank, comm) for every rank, each under its own stream, then join the streams."""
        cur = torch.cuda.current_stream(self.device)
        for r in range(self.world_size):
            self.streams[r].wait_stream(cur)
            with torch.cuda.stream(self.streams[r]):
                fn(r, self.comms[r])
        for s in self.streams:
            cur.wait_stream(s)

    def check(self):
        for c in self.comms:
            c.check()

    def destroy(self):
        for c in self.comms:
            if c is not None:
                c.abort()
        for c in self.comms:
            if c is not None:
                c.destroy()
        self.comms = []
