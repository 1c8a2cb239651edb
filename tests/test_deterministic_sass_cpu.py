"""CPU: the kernels the deterministic mode launches carry no floating-point RED / ATOM instruction (whose
order of arrival, and so the rounding of the sum, depends on scheduling), and none of them spills.
Reads the SASS of the built libub200.so and the ptxas reports the build keeps next to the objects."""
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "uniter_b200", "lib", "libub200.so")
FP_ATOMIC = re.compile(r"\b(RED|REDG|ATOM|ATOMG)\.[\w.]*\b(F16x2|BF16x2|F32|F32x\d|F64)\b")

# Kernels (demangled-name patterns) launched only with the mode on; each must be in the library.
DET_ONLY = [r"colsum_det_kernel<", r"ln_bwd_cols_det_kernel<", r"wcolsum_det_kernel<",
            r"embed_bwd_scatter_det_kernel<", r"sumsq_kernel<true>", r"sumsq_finish_kernel",
            r"attn_bwd_short_kernel<(true|false), false>", r"gemm_kernel<.*, -2>"]
# Kernels of the default mode that sum with float atomics; the deterministic mode never launches them.
DEFAULT_ONLY = [r"colsum_kernel<", r"ln_bwd_kernel<", r"ln_bwd_cols_kernel<", r"wcolsum_kernel<",
                r"embed_bwd_scatter_kernel<", r"sumsq_kernel<false>", r"attn_bwd_short_kernel<(true|false), true>",
                r"attn_bwd_kernel<", r"gemm_kernel<.*, -1>", r"gemm_kernel<.*, 144>"]


def _sass_by_kernel():
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(LIB) or not os.path.exists(tool):
        pytest.skip("needs the built library and cuobjdump")
    sass = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = m.group(1)
            funcs[cur] = []
        elif cur is not None:
            funcs[cur].append(line)
    names = list(funcs)
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return {d: funcs[n] for n, d in zip(names, dem)}


def test_deterministic_kernels_have_no_float_atomics():
    funcs = _sass_by_kernel()
    with_atomics = {name for name, lines in funcs.items() if any(FP_ATOMIC.search(x) for x in lines)}
    assert with_atomics, "the pattern finds the default mode's atomics"
    for pat in DET_ONLY:
        hits = [n for n in funcs if re.search(pat, n)]
        assert hits, pat
        assert not [n for n in hits if n in with_atomics], pat
    # every kernel with float atomics is one the deterministic mode does not launch
    stray = [n for n in with_atomics if not any(re.search(p, n) for p in DEFAULT_ONLY)]
    assert not stray, stray


def test_deterministic_kernels_do_not_spill():
    logs = glob.glob(os.path.join(ROOT, "uniter_b200", "lib", "**", "*.ptxas.log"), recursive=True)
    if not logs:
        pytest.skip("no ptxas report next to the objects")
    text = "\n".join(open(p).read() for p in logs)
    blocks = re.split(r"ptxas info\s*: Compiling entry function '", text)
    seen = 0
    for b in blocks[1:]:
        mangled = b.split("'", 1)[0]
        if not any(k in mangled for k in ("colsum_det", "ln_bwd_cols_det", "wcolsum_det", "scatter_det",
                                          "sumsq_finish", "ln_bwd_rows")):
            continue
        seen += 1
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", mangled
    assert seen >= 5
