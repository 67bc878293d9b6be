"""Per-kernel registers / stack / local-memory instruction report of libb200coll.so (no GPU needed).

    python tools/sass_report.py

Reads `cuobjdump -res-usage` (REG, STACK) and `cuobjdump -sass` (LDL/STL count per function, plus the
mnemonics that prove the TMA / mbarrier / multimem paths are in the binary) and prints one line per kernel.
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "ant-ray_b200", "libb200coll.so")


def run(*cmd):
    return subprocess.run(cmd, check=True, capture_output=True, text=True).stdout


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout
    return dict(zip(names, out.splitlines()))


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else LIB
    res = run("cuobjdump", "-res-usage", lib)
    usage = {}
    cur = None
    for line in res.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "REG:" in line:
            reg = int(re.search(r"REG:(\d+)", line).group(1))
            stack = int(re.search(r"STACK:(\d+)", line).group(1))
            usage[cur] = (reg, stack)
            cur = None
    sass = run("cuobjdump", "-sass", lib)
    local = collections.Counter()
    marks = collections.defaultdict(collections.Counter)
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur is None:
            continue
        m = re.search(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
        if not m:
            continue
        op = m.group(1)
        base = op.split(".")[0]
        if base in ("LDL", "STL"):
            local[cur] += 1
        if base in ("UBLKCP", "SYNCS", "LDGMC", "UTMALDG", "UTMASTG") or op.startswith("RED.") and "MC" in op or base == "REDMC" or base == "STGMC":
            marks[cur][base] += 1
    names = demangle(sorted(usage))
    try:
        tree = run("git", "-C", ROOT, "rev-parse", "--short", "HEAD").strip()
    except Exception:
        tree = "?"
    print(f"# {os.path.basename(lib)} (sm_90a), tree {tree}: registers, stack bytes (cuobjdump -res-usage) and LDL/STL "
          "instruction count (cuobjdump -sass) per kernel")
    print("# stack 0 = no local memory at all; produced by tools/sass_report.py")
    print()
    print(" regs  stack  LDL+STL  kernel   [TMA / mbarrier / multimem mnemonics]")
    rows = sorted(usage, key=lambda k: names[k])
    for k in rows:
        reg, stack = usage[k]
        extra = " ".join(f"{m}x{c}" for m, c in sorted(marks[k].items()))
        print(f"{reg:5d} {stack:6d} {local[k]:8d}  {names[k]}" + (f"   [{extra}]" if extra else ""))
    n_clean = sum(1 for k in rows if usage[k][1] == 0 and local[k] == 0)
    print()
    print(f"# {len(rows)} kernels, {n_clean} with no stack and no LDL/STL")
    dirty = [names[k] for k in rows if usage[k][1] or local[k]]
    if dirty:
        print("# kernels with local memory:")
        for d in dirty:
            print("#   " + d)


if __name__ == "__main__":
    main()
