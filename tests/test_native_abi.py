"""The C-ABI library loads on a machine without a GPU and exports exactly what include/b200coll.h
declares; the Python binding lists the same symbols; pure host-side argument checking works."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

from ant_ray_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200coll.h")


def header_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(b200c_[a-z0-9_]+)\s*\(", src))


def test_library_exports_every_header_symbol():
    lib_path = N.library_path()
    assert os.path.exists(lib_path), "libb200coll.so not built (run __graft_entry__.build())"
    out = subprocess.run(["nm", "-D", "--defined-only", lib_path], capture_output=True, text=True, check=True).stdout
    exported = {line.split()[-1] for line in out.splitlines() if " T " in line}
    declared = header_functions()
    assert declared, "no functions parsed from the header"
    assert declared <= exported, f"declared but not exported: {sorted(declared - exported)}"
    assert {s for s in exported if s.startswith("b200c_")} == declared, "library exports b200c_ symbols the header does not declare"


def test_binding_covers_the_header():
    assert set(N.SYMBOLS) == header_functions()


def test_library_has_no_libcuda_link_dependency():
    out = subprocess.run(["ldd", N.library_path()], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out and "libnccl" not in out


def test_load_and_host_side_calls():
    lib = N.load()
    assert lib.b200c_version() == 200
    assert [lib.b200c_dtype_size(d) for d in range(10)] == [1, 1, 4, 4, 8, 8, 2, 4, 8, 2]
    assert lib.b200c_dtype_size(99) == 0
    cfg = N.default_config()
    assert cfg.struct_size == ctypes.sizeof(N.Config) and cfg.staging_bytes == 256 << 20 and cfg.max_blocks == 264
    assert ctypes.sizeof(N.Export) == 96
    assert lib.b200c_status_string(N.ETIMEOUT).decode() == "timed out waiting for a peer"


def test_errors_are_loud_without_a_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("this checks the no-GPU behaviour")
    lib = N.load()
    h = ctypes.c_void_p()
    rc = lib.b200c_comm_create(0, 2, 0, None, ctypes.byref(h))
    assert rc != N.OK and N.last_error()
    with pytest.raises(N.B200CollError):
        N.device_props(0)
    assert lib.b200c_comm_create(5, 2, 0, None, ctypes.byref(h)) == N.EINVAL  # rank out of range
    assert lib.b200c_comm_create(0, 9, 0, None, ctypes.byref(h)) == N.EINVAL  # beyond one NVSwitch domain
    assert lib.b200c_allreduce(None, None, None, 4, N.FLOAT32, N.SUM, 0, None) == N.EINVAL
    from ant_ray_b200.b200_group import B200Group

    g = B200Group(2, 0, "nogpu")
    with pytest.raises(RuntimeError):
        g.allreduce([torch.ones(4)])          # CPU tensor
    with pytest.raises(RuntimeError):
        g.barrier()                            # no CUDA device -> no silent CPU path
    with pytest.raises(RuntimeError):
        B200Group(16, 0, "too-big")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "ant-ray_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f"{f} imports the oracle"
                assert "liboracle" not in text


def test_bn_scratch_bytes_bounds():
    lib = N.load()
    assert [lib.b200c_bn_scratch_bytes(c) for c in (-1, 0, 131073, 1 << 30)] == [0, 0, 0, 0]
    sizes = [lib.b200c_bn_scratch_bytes(c) for c in range(1, 131073)]
    assert sizes[0] > 0 and all(a <= b for a, b in zip(sizes, sizes[1:]))
    assert min(sizes) >= 4096 * 4   # the semaphore region comes first in every buffer


def test_bn_calls_reject_bad_arguments_before_any_launch():
    # The calls pass a made-up pointer, which a correct library never dereferences because it rejects each call
    # first.  They run in a process that sees no CUDA device, so that a library that lost a check fails with a
    # CUDA error instead of launching kernels on that pointer.
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_native_abi as t; t.bn_argument_checks(); print('ok')"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", out.stdout + out.stderr


def bn_argument_checks():
    lib = N.load()
    p = ctypes.c_void_p(16)   # never dereferenced: each call is rejected first
    before = lib.b200c_launch_count()

    def fwd(m=8, c=4, scratch=p, **null):
        a = {k: None if k in null else p for k in ("x", "id", "y", "w", "b", "rm", "rv", "nbt", "sm", "si")}
        return lib.b200c_bn_forward(a["x"], a["id"], a["y"], a["w"], a["b"], a["rm"], a["rv"], a["nbt"], a["sm"], a["si"],
                                    m, c, 0.1, 1e-5, scratch, None)

    def bwd(m=8, c=4, scratch=p, **null):
        a = {k: None if k in null else p for k in ("dy", "y", "x", "mask", "dx", "w", "sm", "si", "gw", "gb")}
        return lib.b200c_bn_backward(a["dy"], a["y"], a["x"], a["mask"], a["dx"], a["w"], a["sm"], a["si"], a["gw"], a["gb"],
                                     m, c, scratch, None)

    for call in (fwd, bwd):
        for m, c in ((0, 4), (8, 0), (-1, 4), (8, 131073), (2 ** 16, 2 ** 15), (2 ** 14, 2 ** 17)):   # m * c = 2^31 last
            assert call(m=m, c=c) == N.EINVAL, (call.__name__, m, c)
        assert call(scratch=None) == N.EINVAL
    for name in ("x", "y", "w", "b", "rm", "rv", "sm", "si"):
        assert fwd(**{name: 1}) == N.EINVAL, name
    for name in ("dy", "y", "x", "dx", "w", "sm", "si", "gw", "gb"):
        assert bwd(**{name: 1}) == N.EINVAL, name
    assert "batch norm" in N.last_error()
    assert lib.b200c_launch_count() == before
