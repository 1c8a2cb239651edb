"""Per-kernel SASS mnemonic counts of libub200.so (cuobjdump -sass): which kernels are wgmma (HGMMA) / TMA,
which — for the peer exchange — carry system-scope release / acquire accesses, and which carry
floating-point RED / ATOM instructions (order-dependent sums: none in the deterministic mode's kernels).

    python tools/sass_summary.py > sass_summary.txt
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "uniter_b200", "lib", "libub200.so")
COLS = [("HGMMA", r"\bHGMMA"), ("UTMALDG", r"\bUTMALDG"), ("UTMASTG", r"\bUTMASTG"),
        ("WARPGROUP", r"\bWARPGROUP"),
        ("MUFU.EX2", r"MUFU\.EX2"), ("MUFU.RCP", r"MUFU\.RCP"), ("MUFU.TANH", r"MUFU\.TANH"),
        ("STG.SYS", r"\bSTG\.E(\.\w+)*\.STRONG\.SYS"), ("LDG.SYS", r"\bLDG\.E(\.\w+)*\.STRONG\.SYS"),
        ("MEMBAR.SYS", r"MEMBAR\.\w+\.SYS"),
        # floating-point reductions / atomics to memory: their order depends on scheduling, so a kernel
        # the deterministic mode launches must have none (integer tickets are fine)
        ("FP.RED/ATOM", r"\b(RED|REDG|ATOM|ATOMG)\.[\w.]*\b(F16x2|BF16x2|F32|F32x\d|F64)\b")]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    demangle = {}
    counts = collections.OrderedDict()
    cur = None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts.setdefault(cur, collections.Counter())["__n"] += 1
            continue
        if cur is None:
            continue
        for name, pat in COLS:
            if re.search(pat, line):
                counts[cur][name] += 1
    names = list(counts)
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    agg = collections.OrderedDict()
    for mangled, dem in zip(names, out):
        base = re.sub(r"<.*", "", re.sub(r"^void ", "", dem))
        base = re.sub(r"\(.*", "", base)
        a = agg.setdefault(base, collections.Counter())
        a.update(counts[mangled])
    print("# SASS summary of uniter_b200/lib/libub200.so (cuobjdump -sass, sm_90a), per kernel template (all instantiations summed)")
    print("# columns: instantiations | " + " | ".join(n for n, _ in COLS))
    for base, c in sorted(agg.items(), key=lambda kv: -(kv[1]["HGMMA"] + kv[1]["UTMALDG"])):
        print("%-40s %4d | " % (base[:40], c["__n"]) + " | ".join("%5d" % c[n] for n, _ in COLS))


if __name__ == "__main__":
    sys.exit(main())
