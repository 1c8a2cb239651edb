"""CPU: the word-region alignment kernels (csrc/heads.cu, wra_*) carry no floating-point RED / ATOM
instruction and do not spill, so the distance and its gradient come out in the same fixed order in every
library mode.  Reads the SASS of the built libub200.so and the ptxas reports the build keeps next to the
objects."""
import glob
import os
import re

import pytest

from tests.test_deterministic_sass_cpu import FP_ATOMIC, LIB, ROOT, _sass_by_kernel

KERNELS = [r"wra_fwd_kernel<true>", r"wra_fwd_kernel<false>", r"wra_bwd_kernel<true>", r"wra_bwd_kernel<false>"]


def test_wra_kernels_have_no_float_atomics():
    funcs = _sass_by_kernel()
    for pat in KERNELS:
        hits = [n for n in funcs if re.search(pat, n)]
        assert hits, pat
        for n in hits:
            assert not any(FP_ATOMIC.search(x) for x in funcs[n]), n


def test_wra_kernels_do_not_spill():
    logs = glob.glob(os.path.join(ROOT, "uniter_b200", "lib", "**", "heads.o.ptxas.log"), recursive=True)
    if not logs or not os.path.exists(LIB):
        pytest.skip("no ptxas report next to the objects")
    blocks = re.split(r"ptxas info\s*: Compiling entry function '", open(logs[0]).read())
    seen = 0
    for b in blocks[1:]:
        mangled = b.split("'", 1)[0]
        if "wra_" not in mangled:
            continue
        seen += 1
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", mangled
    assert seen == 4
