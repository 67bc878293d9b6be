"""ant_ray_b200.fsdp without a GPU: the hook signatures FSDP1 dispatches on, the torch FSDP2 interfaces the
collectives implement, the reduce-op mapping (with a fake communicator) and prepare_model's CPU refusal."""
import inspect

import pytest
import torch
import torch.distributed as dist
from torch.distributed.fsdp._fully_shard._fsdp_api import AllGather, ReduceScatter

from ant_ray_b200 import _native as N
from ant_ray_b200 import ddp_hook, fsdp
from ant_ray_b200 import train as T


class _FakeComm:
    """Records the calls a PeerMemoryComm would forward to the library."""

    def __init__(self, world_size=4, rank=1):
        self.world_size, self.rank = world_size, rank
        self.calls = []

    def reducescatter_scaled(self, *args):
        self.calls.append(("reducescatter_scaled",) + args)

    def allreduce_scaled(self, *args):
        self.calls.append(("allreduce_scaled",) + args)

    def allgather(self, *args):
        self.calls.append(("allgather",) + args)


class _State:
    """The fields of ddp_hook.B200GradState the FSDP adapters use (the real one creates a CUDA stream)."""

    def __init__(self, comm, wire="fp32"):
        self.comm, self.wire, self.algo = comm, ddp_hook._WIRE[wire], N.ALGO_AUTO
        self.launches = self.bytes = 0


class _Group:
    def __init__(self, W, r):
        self.W, self.r = W, r

    def size(self):
        return self.W

    def rank(self):
        return self.r


def test_hook_signatures_are_what_fsdp1_dispatches_on():
    # FSDP1 calls hook(state, grad, output) for the sharded strategies and hook(state, grad) for NO_SHARD
    assert list(inspect.signature(fsdp.b200_reduce_scatter_hook).parameters) == ["state", "grad", "output"]
    assert list(inspect.signature(fsdp.b200_allreduce_hook_no_shard).parameters) == ["state", "grad"]


def test_collectives_implement_the_fsdp2_interfaces():
    assert issubclass(fsdp.B200AllGather, AllGather) and issubclass(fsdp.B200ReduceScatter, ReduceScatter)
    ag, rs = fsdp.B200AllGather(_FakeComm()), fsdp.B200ReduceScatter(_State(_FakeComm()))
    for comm in (ag, rs):
        t = comm.allocate((6,), dtype=torch.bfloat16, device=torch.device("cpu"))
        assert t.shape == (6,) and t.dtype == torch.bfloat16


@pytest.mark.parametrize("dtype,wire,op,native_wire,scale", [
    (torch.float32, "fp32", dist.ReduceOp.AVG, N.FLOAT32, 0.25),
    (torch.float32, "bf16", dist.ReduceOp.AVG, N.BFLOAT16, 0.25),
    (torch.bfloat16, "bf16", dist.ReduceOp.AVG, N.BFLOAT16, 0.25),
    (torch.float16, "bf16", dist.ReduceOp.SUM, N.FLOAT16, 1.0),   # the wire only applies to fp32 gradients
], ids=str)
def test_reduce_scatter_maps_the_op_and_the_wire(dtype, wire, op, native_wire, scale):
    comm = _FakeComm(4, 1)
    rs = fsdp.B200ReduceScatter(_State(comm, wire))
    x = torch.zeros(4 * 10, dtype=dtype)
    out = torch.zeros(10, dtype=dtype)
    assert rs(out, x, _Group(4, 1), op) is None
    (name, ptrs, recv, n, nat, nat_wire, sc), = comm.calls
    esz = x.element_size()
    assert name == "reducescatter_scaled" and ptrs == [x.data_ptr() + j * 10 * esz for j in range(4)]
    assert (recv, n, nat, nat_wire, sc) == (out.data_ptr(), 10, ddp_hook._BUCKET[dtype], native_wire, scale)


def test_reduce_scatter_refuses_other_ops():
    rs = fsdp.B200ReduceScatter(_State(_FakeComm(4, 1)))
    x, out = torch.zeros(40), torch.zeros(10)
    with pytest.raises(ValueError, match="set_gradient_divide_factor"):
        rs(out, x, _Group(4, 1), dist._make_nccl_premul_sum(0.5))
    for op in (dist.ReduceOp.MAX, dist.ReduceOp.PRODUCT):
        with pytest.raises(ValueError):
            rs(out, x, _Group(4, 1), op)
    with pytest.raises(ValueError):   # a group that is not the communicator's
        rs(out, x, _Group(2, 1), dist.ReduceOp.AVG)
    with pytest.raises(RuntimeError):  # input is not world size x output
        rs(out, torch.zeros(39), _Group(4, 1), dist.ReduceOp.AVG)
    with pytest.raises(RuntimeError):
        rs(torch.zeros(10, dtype=torch.int32), torch.zeros(40, dtype=torch.int32), _Group(4, 1), dist.ReduceOp.AVG)


def test_all_gather_is_in_place_bytes():
    comm = _FakeComm(4, 2)
    out = torch.zeros(4 * 6, dtype=torch.float16)
    assert fsdp.B200AllGather(comm)(out, out[12:18], _Group(4, 2)) is None
    (name, send, recv_ptrs, nbytes, dtype), = comm.calls
    assert (name, send, nbytes, dtype) == ("allgather", out[12:18].data_ptr(), 12, N.UINT8)
    assert recv_ptrs == [out.data_ptr() + 12 * j for j in range(4)]
    with pytest.raises(ValueError):
        fsdp.B200AllGather(comm)(out, out[12:18], _Group(4, 1))
    with pytest.raises(RuntimeError):
        fsdp.B200AllGather(comm)(out, out[12:17], _Group(4, 2))


def test_fsdp1_hooks_compute_the_mean():
    comm = _FakeComm(4, 0)
    st = _State(comm, "bf16")
    g, out = torch.zeros(40), torch.zeros(10)
    fsdp.b200_reduce_scatter_hook(st, g, out)
    fsdp.b200_allreduce_hook_no_shard(st, g)
    rs, ar = comm.calls
    assert rs[0] == "reducescatter_scaled" and rs[5:] == (N.BFLOAT16, 0.25)
    assert ar == ("allreduce_scaled", g.data_ptr(), g.data_ptr(), 40, N.FLOAT32, N.BFLOAT16, 0.25, N.ALGO_AUTO)
    assert st.launches == 2


def test_wire_comes_from_the_environment(monkeypatch):
    monkeypatch.setenv("B200COLL_GRAD_WIRE", "bf16")
    assert ddp_hook.resolve_wire(None) == "bf16"
    assert ddp_hook.resolve_wire("fp32") == "fp32"
    monkeypatch.delenv("B200COLL_GRAD_WIRE")
    assert ddp_hook.resolve_wire(None) == "fp32"


def test_fsdp_config_is_small_unless_overridden(monkeypatch):
    monkeypatch.delenv("B200COLL_STAGING_MB", raising=False)
    monkeypatch.delenv("B200COLL_HOOK_MAX_BLOCKS", raising=False)
    monkeypatch.delenv("B200COLL_NVLS_STREAMS_MIN_BYTES", raising=False)
    cfg = fsdp.fsdp_config()
    assert (cfg.staging_bytes, cfg.max_blocks, cfg.nvls_streams_min_bytes) == (fsdp.FSDP_STAGING_BYTES, 64, 0)
    monkeypatch.setenv("B200COLL_STAGING_MB", "128")
    monkeypatch.setenv("B200COLL_NVLS_STREAMS_MIN_BYTES", str(1 << 30))
    cfg = fsdp.fsdp_config()
    assert (cfg.staging_bytes, cfg.nvls_streams_min_bytes) == (128 << 20, 1 << 30)


def test_fsdp1_refuses_a_process_group_other_than_the_world():
    """The communicator spans the torch.distributed world (here: not initialised, one rank); a root wrapped over
    another group must not be reduced over the wrong ranks."""
    from torch.distributed.fsdp import ShardingStrategy

    class _Root:
        process_group = _Group(2, 1)
        sharding_strategy = ShardingStrategy.FULL_SHARD

        def register_comm_hook(self, state, hook):
            raise AssertionError("must not register")

    with pytest.raises(ValueError, match="process group"):
        fsdp.register_fsdp1(_Root())
    # an explicit state must match the group as well
    with pytest.raises(ValueError):
        _Root.process_group = _Group(1, 0)
        fsdp.register_fsdp1(_Root(), state=_State(_FakeComm(4, 1)))


def test_prepare_model_fsdp_has_no_cpu_path():
    if torch.cuda.is_available():
        pytest.skip("checks the no-GPU behaviour")
    m = torch.nn.Linear(4, 4)
    with pytest.raises(RuntimeError):
        T.prepare_model(m, move_to_device=torch.device("cpu"), parallel_strategy="fsdp", wrap_single=True)
    with pytest.raises(RuntimeError):
        T.prepare_model(m, move_to_device=torch.device("cpu"), parallel_strategy="zero3", wrap_single=True)
