"""The reduce kernels must keep local memory out of their loops: `cuobjdump -res-usage` and `-sass` of the built library.

Every kernel outside the families below compiles without a stack.  The listed families keep a few loop invariants
in local memory under the 64-register budget of two 512-thread CTAs per SM (sm_90a register allocation); their
stack is capped and every local access must sit outside the innermost loops, i.e. outside the per-vector work.
No GPU needed (the listing is static); skipped when the CUDA binary utilities are not installed."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")

# family (regex on the mangled name) -> stack bytes it may use
ALLOWED_STACK = {
    r"k_allreduce_nvls_(lanes|rounds)I": 32,                  # round-pipelined / lane NVLS: per-round peer state
    r"k_broadcast_rounds": 32,
    r"k_allgather": 24,
    r"k_(allreduce_(oneshot|twoshot)|reduce|reducescatter)I(dd|ll|mm|d|l|m)Li": 24,   # 8-byte elements
    r"k_allreduce_oneshotIfNS_(6bf16|5f16)_tELi0ELi8E": 16,   # fused gradient mean, W = 8
    r"k_allreduce_twoshotI(aa|hh|jj)Li\dELi8E": 8,
    r"k_reducescatterIiLi1ELi8E": 8,
    r"k_allreduce_llIaLi0ELi4E": 8,
    r"k_stage_copyI.*Lb1E": 8,
}
# the only kernels with a local access inside an innermost loop (each one a reload of a loop bound or base pointer)
INNER_LOOP_LOCAL = {
    "_ZN5b200c19k_allreduce_twoshotIaaLi1ELi8EEEvNS_8CollArgsE",   # int8 PROD, W = 8
    "_ZN5b200c19k_allreduce_twoshotIhhLi1ELi8EEEvNS_8CollArgsE",   # uint8 PROD, W = 8
    "_ZN5b200c19k_allreduce_oneshotIfNS_6bf16_tELi0ELi8EEEvNS_8CollArgsE",
    "_ZN5b200c15k_reducescatterIlLi1ELi8EEEvNS_8CollArgsE",       # int64 PROD, W = 8
}


def allowed_stack(kernel):
    return max([cap for pat, cap in ALLOWED_STACK.items() if re.search(pat, kernel)], default=0)


@pytest.fixture(scope="module")
def res_usage():
    if shutil.which("cuobjdump") is None or shutil.which("c++filt") is None:
        pytest.skip("cuobjdump / c++filt not installed")
    if not os.path.exists(LIB):
        pytest.skip("libb200coll.so not built")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
        elif cur and "STACK:" in line:
            usage[cur] = (int(re.search(r"REG:(\d+)", line).group(1)), int(re.search(r"STACK:(\d+)", line).group(1)))
            cur = None
    assert len(usage) > 100, "res-usage listing not parsed"
    return usage


def test_no_kernel_uses_a_stack_except_the_listed_ones(res_usage):
    bad = {k: v for k, v in res_usage.items() if v[1] > allowed_stack(k)}
    assert not bad, f"kernels with more local memory than allowed: {bad}"
    # the fp32 / bf16 / fp16 two-shot reduce kernels (the multi-GPU gradient path) and the LL kernels use none
    two = {k: v for k, v in res_usage.items() if re.search(r"k_allreduce_twoshotI(f|NS_6bf16_t|NS_5f16_t)", k)}
    assert len(two) >= 4 and all(v[1] == 0 for v in two.values()), two
    ll = {k: v for k, v in res_usage.items() if "k_allreduce_llI" in k}
    assert len(ll) >= 40 and sum(v[1] > 0 for v in ll.values()) <= 1, {k: v for k, v in ll.items() if v[1]}


def test_local_memory_stays_outside_innermost_loops(res_usage):
    stacked = {k for k, v in res_usage.items() if v[1] > 0}
    sass = subprocess.run(["cuobjdump", "-sass", LIB], check=True, capture_output=True, text=True).stdout
    bad = {}
    for body in re.split(r"\n\s*Function : ", sass)[1:]:
        name = body.split("\n", 1)[0].strip()
        if name not in stacked:
            continue
        ins = [(int(a, 16), t) for a, t in re.findall(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", body)]
        loops = []  # [target, backward branch]
        for a, t in ins:
            m = re.search(r"\bBRA\b.*?(0x[0-9a-f]+)", t)
            if m and int(m.group(1), 16) <= a:
                loops.append((int(m.group(1), 16), a))
        inner = [lp for lp in loops if not any(o != lp and lp[0] <= o[0] and o[1] <= lp[1] for o in loops)]
        hits = sum(1 for a, t in ins if re.search(r"\b(LDL|STL)\b", t) and any(lo <= a <= hi for lo, hi in inner))
        if hits and name not in INNER_LOOP_LOCAL:
            bad[name] = hits
    assert not bad, f"local memory accesses inside innermost loops: {bad}"


def test_reduce_kernels_exist_per_world_size(res_usage):
    # one kernel per world size 2 / 4 / 8 and one for the others (WT = 0): fp32 SUM two-shot
    for wt in (0, 2, 4, 8):
        assert any(re.search(rf"k_allreduce_twoshotIffLi0ELi{wt}E", k) for k in res_usage), wt
    # two CTAs of 512 threads per SM: at most 64 registers per thread in every kernel launched with a max_blocks grid
    for k, (reg, _) in res_usage.items():
        if re.search(r"k_allreduce_(oneshot|twoshot|nvls)|k_reduce|k_reducescatter|k_allgather|k_broadcast", k):
            assert reg <= 64, (k, reg)
