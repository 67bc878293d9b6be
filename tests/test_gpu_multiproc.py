"""GPU tests with one PROCESS per GPU (need >= 2 GPUs): the real deployment shape.

Ported from the reference's single_node_gpu_tests (python/ray/util/collective/tests/
single_node_gpu_tests/test_{allreduce,allgather,reducescatter,broadcast,reduce,sendrecv}.py) with
torch CUDA tensors in place of cupy arrays, plus seeded-random parity against the CPU oracle and
the NVLS (multimem) path, which needs distinct devices.
"""
import numpy as np
import pytest
import torch

from gpu_common import assert_equal_bits, make_input
from mini_actor import get, spawn
from workers import GPUWorker, create_collective_workers

from ant_ray_b200.types import ReduceOp
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


needs2 = pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")


@pytest.fixture
def workers(store_dir):
    made = []

    def make(n=2, group_name="default"):
        actors = create_collective_workers(n, group_name, "nccl", store_dir, gpu=True)  # "nccl" is the B200 alias
        made.extend(actors)
        return actors

    yield make
    for a in made:
        a.kill()


@needs2
@pytest.mark.parametrize("group_name", ["default", "123?34!"])
def test_allreduce_known_answer(workers, group_name):
    actors = workers(2, group_name)
    results = get([a.do_allreduce.remote(group_name) for a in actors])
    for r in results:
        assert (r == torch.ones(10) * 2).all()


@needs2
@pytest.mark.parametrize("array_size", [2, 2**5, 2**10, 2**15, 2**20])
def test_allreduce_different_array_size(workers, array_size):
    actors = workers()
    get([a.set_buffer.remote(np.ones(array_size, dtype=np.float32)) for a in actors])
    results = get([a.do_allreduce.remote() for a in actors])
    for r in results:
        assert (r == torch.ones(array_size) * 2).all()


@needs2
def test_allreduce_destroy_and_reinit(workers):
    actors = workers()
    assert (get([a.do_allreduce.remote() for a in actors])[0] == 2).all()
    get([a.destroy_group.remote() for a in actors])
    with pytest.raises(RuntimeError):
        get([a.do_allreduce.remote() for a in actors])
    get([a.init_group.remote(2, i, "b200", "default") for i, a in enumerate(actors)])
    results = get([a.do_allreduce.remote() for a in actors])
    for r in results:
        assert (r == torch.ones(10) * 4).all()


@needs2
def test_allreduce_multiple_group_and_ops(workers):
    actors = workers()
    for g in range(1, 3):
        get([a.init_group.remote(2, i, "b200", str(g)) for i, a in enumerate(actors)])
    for i in range(3):
        name = "default" if i == 0 else str(i)
        results = get([a.do_allreduce.remote(name) for a in actors])
        assert (results[0] == torch.ones(10) * (2 ** (i + 1))).all()
    for op, val in {ReduceOp.PRODUCT: 6, ReduceOp.MIN: 2, ReduceOp.MAX: 3}.items():
        get([a.set_buffer.remote(np.ones(10, dtype=np.float32) * (i + 2)) for i, a in enumerate(actors)])
        results = get([a.do_allreduce.remote(op=op) for a in actors])
        for r in results:
            assert (r == torch.ones(10) * val).all()


@needs2
@pytest.mark.parametrize("dtype", [np.uint8, np.float16, np.float32, np.float64])
def test_allreduce_different_dtype(workers, dtype):
    actors = workers()
    get([a.set_buffer.remote(np.ones(10, dtype=dtype)) for a in actors])
    results = get([a.do_allreduce.remote() for a in actors])
    for r in results:
        assert (r.numpy() == np.ones(10, dtype=dtype) * 2).all()


@needs2
def test_allreduce_cpu_tensor_raises(workers):
    """GPU buffer on one rank, CPU torch tensor on the other must raise RuntimeError
    (single_node_gpu_tests/test_allreduce.py:127-162)."""
    actors = workers()
    get(actors[1].set_buffer.remote(torch.ones(10), on_gpu=False))
    with pytest.raises(RuntimeError):
        get(actors[1].do_allreduce.remote())


@needs2
@pytest.mark.parametrize("shape", [10, [2, 2], [5, 5, 5]])
def test_allgather_different_shape(workers, shape):
    actors = workers()
    for i, a in enumerate(actors):
        get(a.set_buffer.remote(np.ones(shape, dtype=np.float32) * (i + 1)))
        get(a.set_list_buffer.remote([np.ones(shape, dtype=np.float32) for _ in range(2)]))
    results = get([a.do_allgather.remote() for a in actors])
    for i in range(2):
        for j in range(2):
            assert (results[i][j] == torch.ones(shape) * (j + 1)).all()


@needs2
def test_allgather_wrong_shape_raises(workers):
    actors = workers()
    get(actors[0].set_list_buffer.remote([np.ones(11, dtype=np.float32) for _ in range(2)]))
    with pytest.raises(RuntimeError):
        get(actors[0].do_allgather.remote())


@needs2
def test_reducescatter_broadcast_reduce(workers):
    actors = workers()
    for r in get([a.do_reducescatter.remote() for a in actors]):
        assert (r == torch.ones(10) * 2).all()
    for src in (0, 1):
        get([a.set_buffer.remote(np.ones(10, dtype=np.float32) * (i + 2)) for i, a in enumerate(actors)])
        for r in get([a.do_broadcast.remote(src_rank=src) for a in actors]):
            assert (r == torch.ones(10) * (src + 2)).all()
    with pytest.raises(ValueError):
        get([a.do_broadcast.remote(src_rank=3) for a in actors])
    get([a.set_buffer.remote(np.ones(10, dtype=np.float32)) for a in actors])
    results = get([a.do_reduce.remote(dst_rank=1) for a in actors])
    assert (results[0] == 1).all() and (results[1] == 2).all()


@needs2
@pytest.mark.parametrize("shape", [[10], [5, 9, 10, 85]])
def test_sendrecv(workers, shape):
    actors = workers()
    get([a.set_buffer.remote(np.ones(shape, dtype=np.float32) * (i + 1)) for i, a in enumerate(actors)])
    results = get([actors[0].do_send.remote(dst_rank=1), actors[1].do_recv.remote(src_rank=0)])
    assert (results[1] == torch.ones(shape)).all()
    with pytest.raises(RuntimeError):
        get(actors[0].do_send.remote(dst_rank=0))


@needs2
def test_barrier(workers):
    actors = workers()
    assert get([a.do_barrier.remote() for a in actors]) == [True, True]


# ---------------------------------------------------------------------------------------------
# seeded-random parity through the pointer-level API, all GPUs of the box, including NVLS
# ---------------------------------------------------------------------------------------------
class RawWorker:
    def __init__(self, rank, world, store_dir):
        import os

        os.environ["B200COLL_STORE"] = f"file://{store_dir}"
        os.environ["B200COLL_BCAST_MULTICAST"] = "1"  # exercise the multicast broadcast even on a 2-GPU box
        torch.cuda.set_device(rank)
        self.rank, self.world = rank, world
        self.comm = None

    def connect(self):
        from ant_ray_b200.b200_group import PeerMemoryComm, make_config

        self.comm = PeerMemoryComm(self.world, self.rank, "raw", self.rank, None,
                                   make_config(staging_bytes=8 << 20, symmetric_bytes=64 << 20, timeout_ms=20000), timeout_s=60)
        return True

    def has_multicast(self):
        return bool(self.comm.multicast)

    def allreduce(self, dtype, n, op, algo, scale_wire=None, symmetric=False):
        from gpu_common import NATIVE
        from ant_ray_b200 import _native as N

        x = make_input(dtype, n, self.rank).cuda()
        if symmetric:
            buf = self.comm.symmetric_tensor((n,), dtype)  # same offset on every rank
            buf.copy_(x)
            self.comm.allreduce(buf.data_ptr(), buf.data_ptr(), n, NATIVE[dtype], op, algo)
            x.copy_(buf)
        elif scale_wire is not None:
            self.comm.allreduce_scaled(x.data_ptr(), x.data_ptr(), n, NATIVE[dtype], NATIVE[scale_wire], 1.0 / self.world, algo)
        else:
            self.comm.allreduce(x.data_ptr(), x.data_ptr(), n, NATIVE[dtype], op, algo)
        torch.cuda.synchronize()
        self.comm.check()
        return x.cpu()

    def streams_then_twoshot(self, n):
        """No host synchronisation between the pipeline and the next staged op."""
        from ant_ray_b200 import _native as N

        x = make_input(torch.float32, n, self.rank).cuda()
        y = make_input(torch.int32, 100_003, self.rank).cuda()
        self.comm.allreduce(x.data_ptr(), x.data_ptr(), n, N.FLOAT32, N.SUM, N.ALGO_NVLS_STREAMS)
        self.comm.allreduce(y.data_ptr(), y.data_ptr(), 100_003, N.INT32, N.SUM, N.ALGO_TWOSHOT)
        torch.cuda.synchronize()
        self.comm.check()
        return x.cpu(), y.cpu()

    def pool_allreduce(self, n):
        """Ordinary torch tensors from the communicator's MemPool are zero-copy: NVLS reduces them in place."""
        from ant_ray_b200 import _native as N

        pool = self.comm.symmetric_pool()
        with torch.cuda.use_mem_pool(pool):
            a = torch.empty(n, device="cuda")
            b = torch.empty(n // 2, device="cuda")
        base = int(self.comm.lib.b200c_comm_symmetric_base(self.comm.handle))
        size = int(self.comm.lib.b200c_comm_symmetric_bytes(self.comm.handle))
        inside = all(base <= t.data_ptr() and t.data_ptr() + t.numel() * 4 <= base + size for t in (a, b))
        offs = (a.data_ptr() - base, b.data_ptr() - base)
        a.copy_(make_input(torch.float32, n, self.rank))
        b.copy_(make_input(torch.float32, n // 2, self.rank + 100))
        before = N.launch_count()
        self.comm.allreduce(a.data_ptr(), a.data_ptr(), n, N.FLOAT32, N.SUM, N.ALGO_NVLS)
        self.comm.allreduce(b.data_ptr(), b.data_ptr(), n // 2, N.FLOAT32, N.SUM, N.ALGO_NVLS)
        torch.cuda.synchronize()
        self.comm.check()
        out = (a.cpu(), b.cpu())
        del a, b
        return inside, offs, N.launch_count() - before, out

    def broadcast(self, nbytes, root):
        from ant_ray_b200 import _native as N

        g = torch.Generator().manual_seed(77 + self.rank)
        x = torch.randint(0, 255, (nbytes,), dtype=torch.uint8, generator=g).cuda()
        self.comm.broadcast(x.data_ptr(), nbytes, N.UINT8, root)
        torch.cuda.synchronize()
        self.comm.check()
        return x.cpu()

    def big_properties(self, n):
        """Size-independent checks at the sweep's largest message (1 GiB): see test_full_size_properties."""
        from ant_ray_b200 import _native as N

        g = torch.Generator(device="cuda").manual_seed(4321 + self.rank)
        x = torch.randint(-2**31, 2**31 - 1, (n,), dtype=torch.int32, device="cuda", generator=g)
        local = int(x.sum(dtype=torch.int64).item())
        self.comm.allreduce(x.data_ptr(), x.data_ptr(), n, N.INT32, N.SUM)
        torch.cuda.synchronize()
        self.comm.check()
        total = int(x.sum(dtype=torch.int64).item())
        edges = torch.cat([x[:4], x[n // 2:n // 2 + 4], x[-4:]]).cpu()
        y = x.clone()
        self.comm.allreduce(y.data_ptr(), y.data_ptr(), n, N.INT32, N.MAX)  # MAX of identical buffers: idempotent
        torch.cuda.synchronize()
        idempotent = bool(torch.equal(x, y))
        del y
        f = torch.full((n,), 1.0, dtype=torch.float32, device="cuda")      # the reference's known-answer fill, full size
        self.comm.allreduce(f.data_ptr(), f.data_ptr(), n, N.FLOAT32, N.SUM)
        torch.cuda.synchronize()
        self.comm.check()
        fill_ok = bool((f == float(self.world)).all().item())
        return local, total, idempotent, fill_ok, edges

    def close(self):
        self.comm.destroy()
        return True


@pytest.fixture(scope="module")
def raw_world(tmp_path_factory):
    n = _ngpu()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    d = str(tmp_path_factory.mktemp("rawstore"))
    actors = [spawn(RawWorker, r, n, d, start_method="spawn") for r in range(n)]
    get([a.connect.remote() for a in actors])
    yield actors, n
    get([a.close.remote() for a in actors])
    for a in actors:
        a.kill()


@pytest.mark.parametrize("dtype", [torch.int32, torch.float32, torch.bfloat16])
@pytest.mark.parametrize("algo_name", ["oneshot", "twoshot", "auto"])
def test_allreduce_parity_all_gpus(raw_world, dtype, algo_name):
    from ant_ray_b200 import _native as N

    actors, W = raw_world
    algo = {"oneshot": N.ALGO_ONESHOT, "twoshot": N.ALGO_TWOSHOT, "auto": N.ALGO_AUTO}[algo_name]
    for n in (10, 100_003, 3_000_001):
        outs = get([a.allreduce.remote(dtype, n, N.SUM, algo) for a in actors])
        want = O.allreduce([make_input(dtype, n, r) for r in range(W)])
        for r in range(W):
            if algo_name == "auto" and dtype != torch.int32:
                # AUTO may pick NVLS on a multicast-capable box: the switch's summation order is not
                # the oracle's, so compare within the north-star tolerance instead of bit-exactly
                tol = 1e-5 if dtype == torch.float32 else 2e-2
                assert torch.allclose(outs[r].float(), want.float(), rtol=tol, atol=tol * 4)
            else:
                assert_equal_bits(outs[r], want, f"{dtype} n={n} {algo_name} rank={r}")
        for r in range(1, W):
            assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_nvls_allreduce(raw_world, dtype):
    """multimem.ld_reduce / multimem.st path: fp32 within 1e-5 relative of the rank-order oracle
    (north_star tolerance); identical bits on every rank."""
    from ant_ray_b200 import _native as N

    actors, W = raw_world
    if not all(get([a.has_multicast.remote() for a in actors])):
        pytest.skip("multicast object not bound on this box")
    for n in (16, 100_003, 3_000_001):
        for symmetric, algo in ((False, N.ALGO_NVLS), (True, N.ALGO_NVLS), (False, N.ALGO_NVLS_PIPE), (False, N.ALGO_NVLS_LANES),
                                (False, N.ALGO_NVLS_STREAMS)):
            if symmetric and (n * torch.empty((), dtype=dtype).element_size()) % 16:
                continue
            outs = get([a.allreduce.remote(dtype, n, N.SUM, algo, None, symmetric) for a in actors])
            want = O.allreduce([make_input(dtype, n, r) for r in range(W)])
            tol = 1e-5 if dtype == torch.float32 else (2e-2 if dtype == torch.bfloat16 else 2e-3)
            assert torch.allclose(outs[0].float(), want.float(), rtol=tol, atol=tol * 4), f"nvls {dtype} n={n} sym={symmetric} algo={algo}"
            for r in range(1, W):
                assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")


def test_symmetric_pool_tensors_are_zero_copy(raw_world):
    """torch.cuda.MemPool over the symmetric region: same offsets on every rank, NVLS in place, right answer."""
    actors, W = raw_world
    if not all(get([a.has_multicast.remote() for a in actors])):
        pytest.skip("multicast object not bound on this box")
    n = 1_000_000
    res = get([a.pool_allreduce.remote(n) for a in actors])
    assert all(r[0] for r in res), "pool tensors must live inside the symmetric region"
    assert len({r[1] for r in res}) == 1, "the same allocation sequence must give the same offsets on every rank"
    assert all(r[2] == 2 for r in res)
    want_a = O.allreduce([make_input(torch.float32, n, r) for r in range(W)])
    want_b = O.allreduce([make_input(torch.float32, n // 2, r + 100) for r in range(W)])
    for r in range(W):
        assert torch.allclose(res[r][3][0], want_a, rtol=1e-5, atol=4e-5) and torch.allclose(res[r][3][1], want_b, rtol=1e-5, atol=4e-5)
        assert_equal_bits(res[r][3][0], res[0][3][0], "every rank must hold identical bits")


def test_nvls_pipelined_multi_piece_and_fused(raw_world):
    """Pipelined staged NVLS: a message of several pieces (staging half is 8 MiB here) and the fused
    bf16-wire gradient mean; 20 back-to-back launches exercise the sub-tile flag epochs."""
    from ant_ray_b200 import _native as N

    actors, W = raw_world
    if not all(get([a.has_multicast.remote() for a in actors])):
        pytest.skip("multicast object not bound on this box")
    n = 5_000_011  # 20 MB fp32 -> 3 pieces
    for _ in range(20):
        outs = get([a.allreduce.remote(torch.float32, n, N.SUM, N.ALGO_NVLS_PIPE) for a in actors])
    want = O.allreduce([make_input(torch.float32, n, r) for r in range(W)])
    assert torch.allclose(outs[0], want, rtol=1e-5, atol=4e-5)
    for r in range(1, W):
        assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")
    for algo in (N.ALGO_NVLS_PIPE, N.ALGO_NVLS_LANES, N.ALGO_NVLS_STREAMS):
        outs = get([a.allreduce.remote(torch.float32, n, N.SUM, algo, torch.bfloat16) for a in actors])
        want = O.allreduce_scaled([make_input(torch.float32, n, r) for r in range(W)], torch.bfloat16, 1.0 / W)
        assert torch.allclose(outs[0], want, rtol=2e-2, atol=2e-2)
        for r in range(1, W):
            assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")
    # lane kernel: one launch for a message several times the staging half (8 MiB here), many ring rounds, 20 in a row;
    # multi-stream pipeline: 9 pieces of 4 MiB through 4 staging regions (region reuse), 10 in a row, then a staged
    # op of another kind right behind it (the closing barrier must keep its staging writes away from the last copy-out)
    n = 9_000_017
    want = O.allreduce([make_input(torch.float32, n, r) for r in range(W)])
    for algo, reps in ((N.ALGO_NVLS_LANES, 20), (N.ALGO_NVLS_STREAMS, 10)):
        for _ in range(reps):
            outs = get([a.allreduce.remote(torch.float32, n, N.SUM, algo) for a in actors])
        assert torch.allclose(outs[0], want, rtol=1e-5, atol=4e-5)
        for r in range(1, W):
            assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")
    outs = get([a.streams_then_twoshot.remote(n) for a in actors])
    want_i = O.allreduce([make_input(torch.int32, 100_003, r) for r in range(W)])
    for r in range(W):
        assert torch.allclose(outs[r][0], want, rtol=1e-5, atol=4e-5)
        assert_equal_bits(outs[r][1], want_i, "two-shot right behind the pipeline")


def test_broadcast_all_gpus(raw_world):
    """Large broadcasts go out as ONE multicast store stream from the root when the multicast object
    is bound (unicast pushes otherwise); odd byte counts exercise the sub-vector tail."""
    actors, W = raw_world
    for root in (0, W - 1):
        # 20,000,001 spans several 8 MiB pieces; the 16-byte multiples >= 4 MiB take the round-pipelined paths
        # (scatter + multicast allgather with a multicast object and W > 2, pipelined unicast pushes otherwise)
        for nbytes in (1000, 100_003, 3_000_000, 20_000_001, 6 << 20, (24 << 20) + 4096):
            outs = get([a.broadcast.remote(nbytes, root) for a in actors])
            want = torch.randint(0, 255, (nbytes,), dtype=torch.uint8, generator=torch.Generator().manual_seed(77 + root))
            for r in range(W):
                assert_equal_bits(outs[r], want, f"broadcast {nbytes} B root={root} rank={r}")


def test_full_size_properties(raw_world):
    """The sweep's largest message (1 GiB, 2^28 elements) is too big to check element by element
    against the CPU oracle in seconds, so it is checked through size-independent properties:
      * int32 SUM wraps modulo 2^32, hence  sum_i result[i] == sum_r sum_i x_r[i]  (mod 2^32)
        -- a checksum of checksums computed on the GPUs in int64;
      * every rank ends with identical bits (same checksum, same sampled elements);
      * MAX over already-identical buffers is idempotent;
      * a constant fill of ones sums to exactly W (the reference's known-answer test at full size).
    The message spans >100 staging pieces here (8 MiB staging), so piece boundaries are covered too."""
    actors, W = raw_world
    n = 1 << 28
    res = get([a.big_properties.remote(n) for a in actors], timeout=600)
    locals_, totals = [r[0] for r in res], [r[1] for r in res]
    assert len(set(totals)) == 1, "ranks disagree on the checksum of the result"
    assert (sum(locals_) - totals[0]) % (1 << 32) == 0, "checksum of checksums mismatch"
    for r in range(W):
        assert res[r][2], f"rank {r}: MAX was not idempotent"
        assert res[r][3], f"rank {r}: fill of ones did not sum to W everywhere"
        assert torch.equal(res[r][4], res[0][4])


def test_fused_gradient_mean_all_gpus(raw_world):
    from ant_ray_b200 import _native as N

    actors, W = raw_world
    n = 2_000_003
    for algo in (N.ALGO_TWOSHOT, N.ALGO_AUTO):
        outs = get([a.allreduce.remote(torch.float32, n, N.SUM, algo, torch.bfloat16) for a in actors])
        want = O.allreduce_scaled([make_input(torch.float32, n, r) for r in range(W)], torch.bfloat16, 1.0 / W)
        if algo == N.ALGO_TWOSHOT:
            assert_equal_bits(outs[0], want, "fused bf16-wire mean")
        else:
            assert torch.allclose(outs[0], want, rtol=2e-2, atol=2e-2)
        for r in range(1, W):
            assert_equal_bits(outs[r], outs[0], "every rank must hold identical bits")
