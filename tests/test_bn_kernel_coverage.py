"""Every batch-norm kernel the library compiles is launched by a test.

KERNELS names each `b200c::bn` kernel as the profiler prints it (template arguments included, without the parameter
list) and the case that launches it.  Each case is one site run through the helpers of the parity tests, so it also
checks its results against torch.  On the CPU, the built library's `b200c::bn` functions must be exactly KERNELS, so a
kernel that exists without a case, or a case for a kernel that no longer exists, fails.  On the GPU, each case runs
once under torch.profiler and must launch every kernel the table gives it."""
import json
import os
import re
import shutil
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

_E = "b200c::bn::k_bn_bwd_elemt<{}, (b200c::bn::GradSrc){}, {}, {}>"
_R = "b200c::bn::k_bn_bwd_reduce<(b200c::bn::GradSrc){}, {}>"
_T = "b200c::bn::k_bn_transform<{}, (b200c::bn::Tail){}>"
# GradSrc: 0 masked (g the reduce kernel wrote), 1 y, 2 mask bits, 3 dy (no ReLU), 4 pool.  Tail: 0 none, 1 ReLU,
# 2 add + ReLU, 3 a second batch norm + add + ReLU.
KERNELS = {
    "b200c::bn::k_bn_stats<1>": "local_relu_c100",
    "b200c::bn::k_bn_stats<4>": "local_relu_c64",
    "b200c::bn::k_bn_stats_dual<1>": "dual_c100",
    "b200c::bn::k_bn_stats_dual<4>": "dual_c64",
    "b200c::bn::k_bn_sync_stats<1>": "sync_relu_c100",
    "b200c::bn::k_bn_sync_stats<4>": "sync_relu_c64",
    "b200c::bn::k_bn_sync_merge": "sync_relu_c64",
    _T.format(1, 0): "sync_plain_c100",
    _T.format(1, 1): "local_relu_c100",
    _T.format(1, 2): "local_tail_c100",
    _T.format(1, 3): "dual_c100",
    _T.format(8, 0): "sync_plain_c64",
    _T.format(8, 1): "local_relu_c64",
    _T.format(8, 2): "local_tail_c64",
    _T.format(8, 3): "dual_c64",
    "b200c::bn::k_bn_pool_fwd<1>": "stem_c100",
    "b200c::bn::k_bn_pool_fwd<8>": "stem_c64",
    _R.format(1, "false"): "local_relu_c100",
    _R.format(2, "false"): "local_relu_c64",
    _R.format(3, "false"): "sync_plain_c64",
    _R.format(4, "false"): "stem_c64",
    _R.format(1, "true"): "dual_c100",
    _R.format(2, "true"): "dual_c64",
    _E.format(1, 0, "false", "false"): "local_tail_c100",
    _E.format(1, 0, "true", "false"): "sync_tail_c100",
    _E.format(1, 1, "false", "false"): "local_relu_c100",
    _E.format(1, 1, "false", "true"): "dual_c100",
    _E.format(1, 1, "true", "false"): "sync_relu_c100",
    _E.format(1, 2, "false", "false"): "local_relu_c64_misaligned",
    _E.format(1, 2, "false", "true"): "dual_c64_misaligned",
    _E.format(1, 2, "true", "false"): "sync_relu_c64_misaligned",
    _E.format(1, 3, "true", "false"): "sync_plain_c100",
    _E.format(8, 0, "false", "false"): "local_tail_c64",
    _E.format(8, 0, "true", "false"): "sync_tail_c64",
    _E.format(8, 1, "false", "false"): "local_relu_c64_reading_y",
    _E.format(8, 1, "false", "true"): "dual_c64_reading_y",
    _E.format(8, 1, "true", "false"): "sync_relu_c64_reading_y",
    _E.format(8, 2, "false", "false"): "local_relu_c64",
    _E.format(8, 2, "false", "true"): "dual_c64",
    _E.format(8, 2, "true", "false"): "sync_relu_c64",
    _E.format(8, 3, "true", "false"): "sync_plain_c64",
}


def kernel_name(signature):
    """`b200c::bn::k_...<template arguments>` of a demangled kernel signature: no return type, no parameter list."""
    name = signature[signature.index("b200c::bn::"):]
    depth = 0
    for i, ch in enumerate(name):
        depth += (ch == "<") - (ch == ">")
        if ch == "(" and depth == 0:
            return name[:i]
    return name


def test_the_table_is_the_library_s_batch_norm_kernels():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    mangled = sorted({f for f in re.findall(r"Function (\S+):", out) if f.startswith("_ZN5b200c2bn")})
    demangled = subprocess.run(["c++filt"], input="\n".join(mangled), check=True, capture_output=True, text=True).stdout
    names = {kernel_name(line) for line in demangled.splitlines()}
    assert len(names) == len(mangled) == len(KERNELS) == 41
    assert names == set(KERNELS), {"without a case": sorted(names - set(KERNELS)), "not in the library": sorted(set(KERNELS) - names)}


def case_runs(world):
    """Each case of KERNELS: one site through the parity tests' helpers; sync cases in the W = 2 `world`."""
    import test_gpu_fused_dual as D
    import test_gpu_fused_norm as L
    import test_gpu_fused_stem as P
    import test_gpu_sync_norm as S

    def dual(n, c, h, w, misalign=False):
        x3, x_ds, dy1, dy2 = D.inputs(n, c, h, w, c)
        D.check_dual(x3, L.misaligned(x_ds) if misalign else x_ds, dy1, dy2, "pair", L.make_bn(c, 1), L.make_bn(c, 2))

    return {
        "local_relu_c64": lambda: L.check_site(8, 64, 16, 16, False),
        "local_relu_c64_misaligned": lambda: L.check_site(8, 64, 16, 16, False, misalign=("x",)),
        "local_relu_c100": lambda: L.check_site(3, 100, 9, 9, False),
        "local_tail_c64": lambda: L.check_site(8, 64, 16, 16, True),
        "local_tail_c100": lambda: L.check_site(3, 100, 9, 9, True),
        "local_relu_c64_reading_y": lambda: L.check_native_site(2048, 64, 1),
        "dual_c64": lambda: dual(8, 64, 16, 16),
        "dual_c64_misaligned": lambda: dual(8, 64, 16, 16, misalign=True),
        "dual_c100": lambda: dual(3, 100, 9, 9),
        "dual_c64_reading_y": lambda: D.check_dual_through_the_c_abi(8, 64, 16, 16),
        "stem_c64": lambda: P.check_stem(*P.gauss_inputs(8, 64, 16, 16, 1), L.make_bn(64, 3)),
        "stem_c100": lambda: P.check_stem(*P.gauss_inputs(3, 100, 9, 9, 2), L.make_bn(100, 3)),
        "sync_relu_c64": lambda: S.check_sites(world, 5, 64, 7, 7, "relu", seed=1),
        "sync_relu_c64_misaligned": lambda: S.check_sites(world, 5, 64, 7, 7, "relu", seed=2, misalign=("x",)),
        "sync_relu_c100": lambda: S.check_sites(world, 5, 100, 7, 7, "relu", seed=3),
        "sync_tail_c64": lambda: S.check_sites(world, 5, 64, 7, 7, "tail", seed=4),
        "sync_tail_c100": lambda: S.check_sites(world, 5, 100, 7, 7, "tail", seed=5),
        "sync_plain_c64": lambda: S.check_sites(world, 5, 64, 7, 7, "plain", seed=6),
        "sync_plain_c100": lambda: S.check_sites(world, 5, 100, 7, 7, "plain", seed=7),
        "sync_relu_c64_reading_y": lambda: S.check_relu_site_reading_y(world, 64),
    }


def trace_cases():
    """Runs every case once under torch.profiler and prints {case: [b200c::bn kernels it launched]} as JSON."""
    from ant_ray_b200.loopback import LoopbackWorld
    import test_gpu_sync_norm as S

    world = LoopbackWorld(2, device=0, key="bn-coverage", staging_bytes=1 << 20, max_blocks=8, timeout_ms=20000)
    S.load_torch_kernels()
    launched = {}
    try:
        for case, run in case_runs(world).items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            launched[case] = sorted({kernel_name(e.name) for e in prof.events()
                                     if e.device_type == torch.autograd.DeviceType.CUDA and "b200c::bn::" in e.name})
    finally:
        world.destroy()
    print(json.dumps(launched))


@pytest.mark.gpu
def test_every_kernel_is_launched_by_its_case():
    # in a process of its own, as test_gpu_fused_stem's trace: its profiler sessions share no process with other tests'
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    code = "import test_bn_kernel_coverage as t; t.trace_cases()"
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    launched = json.loads(out.stdout.strip().splitlines()[-1])
    assert set(launched) == set(KERNELS.values())
    for kernel, case in sorted(KERNELS.items(), key=lambda kv: kv[1]):
        print(f"{kernel:72s} {case}")
    missing = {k: case for k, case in KERNELS.items() if k not in launched[case]}
    assert not missing, f"kernels their case did not launch: {missing}"
    unknown = {k for names in launched.values() for k in names} - set(KERNELS)
    assert not unknown, f"launched kernels missing from KERNELS: {unknown}"
