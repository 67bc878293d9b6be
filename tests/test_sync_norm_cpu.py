"""Sync batch norm without a GPU: the C-ABI's argument checks and scratch sizes, which sites sync (with a stand-in
communicator), and when prepare_model attaches a batch-norm communicator."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn

from ant_ray_b200 import _native as N
from ant_ray_b200 import fused_norm
from ant_ray_b200 import train as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CL = torch.channels_last


def test_sync_calls_reject_bad_arguments_before_any_launch():
    # As in test_native_abi_mask: made-up pointers that a correct library never dereferences, in a process that sees
    # no CUDA device, so that a lost check fails with a CUDA error or a crash instead of launching.
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_sync_norm_cpu as t; t.sync_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def sync_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def fwd(m=8, c=8, relu=1, scratch=p, comm=None, **null):
        a = {k: None if null.get(k, k in ("id", "mask")) else p
             for k in ("x", "id", "y", "mask", "w", "b", "rm", "rv", "nbt", "sm", "si", "nf")}
        return lib.b200c_bn_sync_forward(comm, a["x"], a["id"], a["y"], a["mask"], relu, a["w"], a["b"], a["rm"], a["rv"],
                                         a["nbt"], a["sm"], a["si"], a["nf"], m, c, 0.1, 1e-5, scratch, None)

    def bwd(m=8, c=8, relu=1, scratch=p, comm=None, **null):
        a = {k: None if null.get(k, k in ("dy2", "mask", "gid")) else p
             for k in ("dy", "dy2", "y", "mask", "x", "gid", "dx", "w", "sm", "si", "nf", "gw", "gb")}
        return lib.b200c_bn_sync_backward(comm, a["dy"], a["dy2"], a["y"], a["mask"], relu, a["x"], a["gid"], a["dx"], a["w"],
                                          a["sm"], a["si"], a["nf"], a["gw"], a["gb"], m, c, scratch, None)

    for call in (fwd, bwd):
        for m, c in ((8, 0), (-1, 8), (8, 131080), (2 ** 16, 2 ** 15), (2 ** 14, 2 ** 17)):   # m * c = 2^31 last
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
            assert "sync batch norm" in N.last_error()
        for c in (4, 12, 100):   # the mask packs 8 channels per byte
            assert call(c=c, mask=False) == N.EINVAL, (call.__name__, c)
            assert "mask" in N.last_error()
        assert call(scratch=None) == N.EINVAL
        # a site without ReLU takes no mask, identity or second gradient
        for name in ("mask", "id") if call is fwd else ("mask", "gid", "dy2"):
            assert call(relu=0, **{name: False}) == N.EINVAL, (call.__name__, name)
            assert "without ReLU" in N.last_error()
        # well-formed arguments, down to an empty rank: only the missing communicator is left
        for m in (8, 0):
            assert call(m=m) == N.EINVAL and "null communicator" in N.last_error(), (call.__name__, m)
    for name in ("x", "y", "w", "b", "rm", "rv", "sm", "si", "nf"):
        assert fwd(**{name: True}) == N.EINVAL, name
        assert "null buffer" in N.last_error()
    for name in ("dy", "x", "dx", "w", "sm", "si", "nf", "gw", "gb"):
        assert bwd(**{name: True}) == N.EINVAL, name
    assert bwd(y=True) == N.EINVAL   # a ReLU site reads y or the mask
    # an empty rank passes no rows
    assert fwd(m=0, x=True, y=True) == N.EINVAL and "null communicator" in N.last_error()
    assert bwd(m=0, dy=True, x=True, dx=True, y=True) == N.EINVAL and "null communicator" in N.last_error()
    assert lib.b200c_launch_count() == before


def test_sync_scratch_bytes_bounds():
    lib = N.load()
    assert [lib.b200c_bn_sync_scratch_bytes(c, 2) for c in (-1, 0, 131073)] == [0, 0, 0]
    assert [lib.b200c_bn_sync_scratch_bytes(64, w) for w in (-1, 0, 9)] == [0, 0, 0]
    for c in (1, 3, 64, 100, 2048, 131072):
        local = lib.b200c_bn_scratch_bytes(c)
        row = (2 * c + 1 + 3) // 4 * 4 * 4
        for w in range(1, 9):
            # the local scratch, then W + 1 rows of [mean | invstd | count] from a 16-byte boundary
            assert lib.b200c_bn_sync_scratch_bytes(c, w) == (local + 15) // 16 * 16 + (w + 1) * row, (c, w)


class StandInComm:
    def __init__(self, world_size):
        self.world_size = world_size


@pytest.fixture
def cpu_rows(monkeypatch):
    # the site tests below run on CPU tensors: accept them where a sync site accepts CUDA tensors (fused_norm's
    # own _activation and _rows, with every tensor taken for a CUDA one)
    class Cuda:
        def __init__(self, t):
            self.t = t

        def __getattr__(self, name):
            return True if name == "is_cuda" else getattr(self.t, name)

    rows, activation = fused_norm._rows, fused_norm._activation
    monkeypatch.setattr(fused_norm, "_activation", lambda t: activation(Cuda(t)))
    monkeypatch.setattr(fused_norm, "_rows", lambda t: rows(Cuda(t)))


def sync_bn(c=64, world=2, **kw):
    bn = nn.SyncBatchNorm(c, **kw)
    return fused_norm.sync_batch_norm(nn.Sequential(bn), StandInComm(world))[0]


def act(n, c=64, hw=7):
    return torch.zeros(n, c, hw, hw, dtype=torch.bfloat16).contiguous(memory_format=CL)


def test_sync_site_does_not_depend_on_the_batch_size(cpu_rows):
    bn = sync_bn()
    assert type(bn) is fused_norm.FusedSyncBatchNorm
    for n in (0, 1, 2, 64):
        assert fused_norm._sync_comm(bn, act(n)) is bn.b200_comm, n
    # one row of one pixel per rank still syncs: torch's SyncBatchNorm allows it at world size > 1
    assert fused_norm._sync_comm(bn, act(1, hw=1)) is bn.b200_comm


@pytest.mark.parametrize("case", ["no_comm", "world_1", "eval", "momentum_none", "untracked", "fp32_input", "nchw"])
def test_sites_that_fall_back(cpu_rows, case):
    bn = sync_bn(world=1 if case == "world_1" else 2, momentum=None if case == "momentum_none" else 0.1,
                 track_running_stats=case != "untracked")
    x = act(4)
    if case == "no_comm":
        bn.b200_comm = None
    elif case == "eval":
        bn.eval()
    elif case == "fp32_input":
        x = x.float()
    elif case == "nchw":
        x = act(4).contiguous()
    # a layout is only seen where there are rows: an empty NCHW input syncs like any empty input
    for n in (0, 4) if case != "nchw" else (4,):
        assert fused_norm._sync_comm(bn, x[:n]) is None, (case, n)


def test_empty_input_from_a_convolution_syncs(cpu_rows):
    # a channels-last convolution over an empty batch returns default strides; its rank must still sync
    conv = nn.Conv2d(3, 64, 3, padding=1).to(torch.bfloat16).to(memory_format=CL)
    with torch.no_grad():
        x = conv(torch.zeros(0, 3, 8, 8, dtype=torch.bfloat16).contiguous(memory_format=CL))
    assert x.stride(1) != 1
    bn = sync_bn()
    assert fused_norm._sync_comm(bn, x) is bn.b200_comm


def test_inputs_past_the_kernels_limits_raise(cpu_rows):
    bn = sync_bn(c=131080)
    with pytest.raises(RuntimeError, match="exceeds"):
        fused_norm._sync_comm(bn, torch.empty(1, 131080, 1, 1, dtype=torch.bfloat16, device="meta").contiguous(memory_format=CL))
    bn = sync_bn(c=64)
    with pytest.raises(RuntimeError, match="exceeds"):
        fused_norm._sync_comm(bn, torch.empty(2 ** 25, 64, 1, 1, dtype=torch.bfloat16, device="meta").contiguous(memory_format=CL))


def test_sync_batch_norm_keeps_the_module_and_skips_subgroups():
    model = nn.Sequential(nn.SyncBatchNorm(8), nn.SyncBatchNorm(8, process_group=object()), nn.BatchNorm2d(8))
    keys = list(model.state_dict())
    params = [id(p) for p in model.parameters()]
    comm = StandInComm(4)
    fused_norm.sync_batch_norm(model, comm)
    assert type(model[0]) is fused_norm.FusedSyncBatchNorm and model[0].b200_comm is comm
    assert type(model[1]) is nn.SyncBatchNorm and type(model[2]) is nn.BatchNorm2d
    assert list(model.state_dict()) == keys and [id(p) for p in model.parameters()] == params


def test_prepare_model_attaches_a_norm_comm_only_for_world_sync_batch_norm(monkeypatch):
    made = []

    def fake_comm(device):
        made.append(device)
        return StandInComm(2)

    monkeypatch.setattr(T, "_sync_norm_comm", fake_comm)
    cuda = torch.device("cuda", 0)
    plain = nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8))
    converted = nn.SyncBatchNorm.convert_sync_batchnorm(nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8)))
    subgroup = nn.Sequential(nn.SyncBatchNorm(8, process_group=object()))
    assert T._attach_sync_norm(plain, cuda, 2) is None
    assert T._attach_sync_norm(converted, cuda, 1) is None
    assert T._attach_sync_norm(converted, torch.device("cpu"), 2) is None
    assert T._attach_sync_norm(subgroup, cuda, 2) is None
    assert not made
    comm = T._attach_sync_norm(converted, cuda, 2)
    assert made == [cuda] and type(converted[1]) is fused_norm.FusedSyncBatchNorm and converted[1].b200_comm is comm


def register_hook(mod, kind):
    if kind == "global":
        return torch.nn.modules.module.register_module_forward_hook(lambda *a: None)
    return getattr(mod, f"register_{kind}_hook")(lambda *a: None)


@pytest.mark.parametrize("kind", ["forward", "forward_pre", "full_backward", "full_backward_pre", "global"])
def test_a_hook_on_any_replaced_module_keeps_the_modules(cpu_rows, kind):
    # one rule at local and sync sites alike: any hook on the batch norm or on a module whose call the kernels replace
    relu, x = nn.ReLU(), act(4)
    for bn in (nn.BatchNorm2d(64), sync_bn()):
        want = fused_norm._LOCAL if type(bn) is nn.BatchNorm2d else bn.b200_comm
        for mod in (bn, relu):
            assert fused_norm._site(bn, x, (relu,)) is want
            h = register_hook(mod, kind)
            assert fused_norm._site(bn, x, (relu,)) is None, (type(bn).__name__, type(mod).__name__)
            h.remove()
    # an entry point without a sync form leaves a sync batch norm to its own module forward
    assert fused_norm._site(sync_bn(), x, (relu,), sync=False) is None
