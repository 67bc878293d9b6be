"""Replay-safe profiling of the MULTI-GPU kernels (NVLS, multicast broadcast, peer pushes) under Nsight Compute.

    ncu --target-processes application-only --set full --clock-control none --import-source on \
        -k regex:"k_allreduce|k_broadcast|k_send|k_allgather" -c 12 -o prof_multi python tools/profile_multi.py 2

ncu replays a kernel many times in isolation, so a kernel that waits for a concurrently running peer kernel
can never be profiled inside a live group.  Here rank 0 (this process — the only one ncu sees) pre-satisfies
its flags (b200c_debug_fill_flags) and launches alone, while ranks 1..W-1 are helper processes that only
create their communicator (arena mapped on their GPU, bound to the multicast object) and then sleep: rank
0's pushes really cross NVLink into their HBM and its multimem.ld_reduce really pulls from every GPU through
the switch, so nvlrx/nvltx and DRAM counters are those of the production kernel; only the data is meaningless.
"""
import multiprocessing as mp
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def helper(rank, world, store_dir, ready, done):
    os.environ["B200COLL_STORE"] = f"file://{store_dir}"
    import torch

    from ant_ray_b200.b200_group import PeerMemoryComm, make_config

    torch.cuda.set_device(rank)
    comm = PeerMemoryComm(world, rank, "profile-multi", rank, None, make_config(symmetric_bytes=256 << 20, timeout_ms=20000))
    ready.put((rank, bool(comm.multicast)))
    done.wait()
    comm.destroy()


def main():
    world = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    store_dir = tempfile.mkdtemp(prefix="b200prof")
    os.environ["B200COLL_STORE"] = f"file://{store_dir}"
    ctx = mp.get_context("spawn")
    ready, done = ctx.Queue(), ctx.Event()
    procs = [ctx.Process(target=helper, args=(r, world, store_dir, ready, done)) for r in range(1, world)]
    for p in procs:
        p.start()
    import torch

    from ant_ray_b200 import _native as N
    from ant_ray_b200.b200_group import PeerMemoryComm, make_config

    torch.cuda.set_device(0)
    comm = PeerMemoryComm(world, 0, "profile-multi", 0, None, make_config(symmetric_bytes=256 << 20, timeout_ms=20000))
    for _ in procs:
        print("helper ready:", ready.get(timeout=120))
    print("multicast:", comm.multicast)
    lib = comm.lib

    def prefill():
        N.check(lib.b200c_debug_fill_flags(comm.handle, 0x7FFFFFFF))

    n64 = (64 << 20) // 4
    x = torch.randn(n64, device="cuda")
    g = torch.randn(30 << 18, device="cuda")
    sym = comm.symmetric_tensor((n64,), torch.float32)
    small = torch.randn(8 << 10, device="cuda")
    b24 = torch.empty(24 << 20, dtype=torch.uint8, device="cuda")
    cases = [
        ("twoshot f32 64MiB", lambda: comm.allreduce(x.data_ptr(), x.data_ptr(), n64, N.FLOAT32, N.SUM, N.ALGO_TWOSHOT)),
        ("oneshot f32 32KiB", lambda: comm.allreduce(small.data_ptr(), small.data_ptr(), small.numel(), N.FLOAT32, N.SUM, N.ALGO_ONESHOT)),
        ("LL f32 32KiB", lambda: comm.allreduce(small.data_ptr(), small.data_ptr(), small.numel(), N.FLOAT32, N.SUM, N.ALGO_LL)),
        ("broadcast 24MiB (root)", lambda: comm.broadcast(b24.data_ptr(), b24.numel(), N.UINT8, 0)),
        ("send 24MiB", lambda: comm.send(b24.data_ptr(), b24.numel(), 1)),
    ]
    if comm.multicast:
        cases += [
            ("nvls staged f32 64MiB", lambda: comm.allreduce(x.data_ptr(), x.data_ptr(), n64, N.FLOAT32, N.SUM, N.ALGO_NVLS)),
            ("nvls rounds f32 64MiB", lambda: comm.allreduce(x.data_ptr(), x.data_ptr(), n64, N.FLOAT32, N.SUM, N.ALGO_NVLS_PIPE)),
            ("nvls symmetric f32 64MiB", lambda: comm.allreduce(sym.data_ptr(), sym.data_ptr(), n64, N.FLOAT32, N.SUM, N.ALGO_NVLS)),
            ("fused grad mean 30MiB bf16 wire (nvls)", lambda: comm.allreduce_scaled(g.data_ptr(), g.data_ptr(), g.numel(), N.FLOAT32, N.BFLOAT16, 1.0 / world, N.ALGO_NVLS)),
        ]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, fn in cases:
        prefill()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        print(f"{name}: {e0.elapsed_time(e1) * 1e3:.1f} us (rank 0 alone, flags pre-satisfied)")
    done.set()
    for p in procs:
        p.join(30)
    comm.destroy()


if __name__ == "__main__":
    main()
