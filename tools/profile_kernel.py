"""Replay-safe single-rank launches of the collective kernels, for Nsight Compute.

    ncu --set full --clock-control none --import-source on -k regex:k_allreduce -c 6 -o prof \
        python tools/profile_kernel.py

Two loopback communicators share cuda:0; rank 0's flags are pre-satisfied
(b200c_debug_fill_flags) so its kernels run alone and survive ncu's kernel replay.  The "peer"
arena is a second mapping on the same GPU, so peer traffic shows up as local HBM/L2 traffic —
the instruction mix, coalescing and stall profile are those of the production kernel.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ant_ray_b200 import _native as N  # noqa: E402
from ant_ray_b200.loopback import LoopbackWorld  # noqa: E402


def main():
    W = int(os.environ.get("PROFILE_WORLD", 2))
    world = LoopbackWorld(W, device=0, key="profile", staging_bytes=128 << 20, max_blocks=264)
    c0 = world.comms[0]
    N.check(c0.lib.b200c_debug_fill_flags(c0.handle, 0x7FFFFFFF))
    n_big = (64 << 20) // 4
    x = torch.randn(n_big, device="cuda")
    g = torch.randn(30 << 18, device="cuda")  # 30 MiB fp32 bucket
    small = torch.randn(16 << 10, device="cuda")
    reps = int(os.environ.get("PROFILE_REPS", 3))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    from ant_ray_b200.b200_group import PeerMemoryComm, make_config  # noqa: E402
    from ant_ray_b200.loopback import _MemStore  # noqa: E402

    solo = PeerMemoryComm(1, 0, "profile-solo", 0, _MemStore(), make_config(staging_bytes=1 << 20))
    gs = [torch.randn(30 << 18, device="cuda") for _ in range(8)]  # rotate 8 x 30 MiB buckets (> L2)
    rot = [0]

    def local_scale():
        b = gs[rot[0] % len(gs)]
        rot[0] += 1
        solo.allreduce_scaled(b.data_ptr(), b.data_ptr(), b.numel(), N.FLOAT32, N.BFLOAT16, 0.5)

    ll = torch.randn(8 << 10, device="cuda")

    def ll_once():
        # LL slots are matched by equality: re-stamp the region with the next op's flag before every launch
        N.check(c0.lib.b200c_debug_fill_flags(c0.handle, 0x7FFFFFFF))
        c0.allreduce(ll.data_ptr(), ll.data_ptr(), ll.numel(), N.FLOAT32, N.SUM, N.ALGO_LL)

    for name, fn in [
        ("local_scale f32/bf16 30MiB (W=1)", local_scale),
        ("LL f32 32KiB", ll_once),
        ("twoshot f32 64MiB", lambda: c0.allreduce(x.data_ptr(), x.data_ptr(), n_big, N.FLOAT32, N.SUM, N.ALGO_TWOSHOT)),
        ("fused grad mean 30MiB bf16 wire", lambda: c0.allreduce_scaled(g.data_ptr(), g.data_ptr(), g.numel(), N.FLOAT32, N.BFLOAT16, 0.5, N.ALGO_TWOSHOT)),
        ("oneshot f32 64KiB", lambda: c0.allreduce(small.data_ptr(), small.data_ptr(), small.numel(), N.FLOAT32, N.SUM, N.ALGO_ONESHOT)),
    ]:
        fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        print(f"{name}: {e0.elapsed_time(e1) / reps * 1e3:.1f} us per launch (single rank, flags pre-satisfied)")
    c0.check()
    solo.destroy()
    world.destroy()


if __name__ == "__main__":
    main()
