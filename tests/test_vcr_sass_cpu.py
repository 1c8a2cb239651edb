"""CPU: the LayerNorm instantiations added for the VCR head (rows up to 2048 wide, ReLU on the input) do not
spill, their deterministic forms carry no floating-point RED / ATOM instruction, and the LayerNorm
instantiations that existed before them (H <= 1024, no ReLU: the encoder, the embedding front-end,
LibTransform) compile to the same SASS instruction stream as before.

tests/golden/ln_sass_fingerprints.json holds, per pre-existing instantiation (under its current name),
the sha256 of its SASS instructions (addresses and encodings stripped) as nvcc 12.9 built it before the
wide / ReLU instantiations were added."""
import glob
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

from tests.test_deterministic_sass_cpu import FP_ATOMIC, LIB, ROOT
from tests.test_deterministic_sass_cpu import _sass_by_kernel as _sass_uncached

GOLDEN = os.path.join(ROOT, "tests", "golden", "ln_sass_fingerprints.json")
NEW_ROWS = [r"ln_bwd_rows_kernel<(true|false), (4|6|8), true>", r"ln_bwd_rows_kernel<(true|false), (6|8), false>"]
NEW_COLS = [r"ln_bwd_cols_det_kernel<(true|false), true>", r"ln_bwd_cols_kernel<(true|false), true>"]
NEW_FWD = [r"ln_fwd_kernel<(true|false), 4, true>", r"ln_fwd_kernel<(true|false), (6|8), (true|false)>"]


_CACHE = []


def _sass_by_kernel():
    if not _CACHE:
        _CACHE.append(_sass_uncached())
    return _CACHE[0]


def instruction_stream(lines):
    """The instructions of one kernel's SASS listing, without addresses and encodings."""
    out = []
    for line in lines:
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;\s*/\*", line)
        if m:
            out.append(re.sub(r"\s+", " ", m.group(1)))
    return out


def fingerprint(lines):
    return hashlib.sha256("\n".join(instruction_stream(lines)).encode()).hexdigest()


def _matches(funcs, pats):
    return [n for n in funcs if any(re.search(p, n) for p in pats)]


def test_preexisting_layernorm_instantiations_have_unchanged_sass():
    tool = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if os.path.exists(tool):
        ver = subprocess.run([tool, "--version"], capture_output=True, text=True).stdout
        if "release 12.9" not in ver:
            pytest.skip("the fingerprints are of nvcc 12.9's SASS")
    funcs = _sass_by_kernel()
    want = json.load(open(GOLDEN))["kernels"]
    assert len(want) == 22
    for name, fp in sorted(want.items()):
        key = [n for n in funcs if n.startswith("void ub::" + name + "(")]
        assert len(key) == 1, name
        assert fingerprint(funcs[key[0]]) == fp, name


def test_wide_and_relu_layernorm_instantiations_are_built():
    funcs = _sass_by_kernel()
    assert len(_matches(funcs, NEW_ROWS)) == 10
    assert len(_matches(funcs, NEW_COLS)) == 4
    assert len(_matches(funcs, NEW_FWD)) == 10


def test_deterministic_forms_have_no_float_atomics():
    funcs = _sass_by_kernel()
    det = _matches(funcs, NEW_ROWS + [r"ln_bwd_cols_det_kernel<(true|false), true>"])
    assert len(det) == 12
    for n in det:
        assert not any(FP_ATOMIC.search(x) for x in funcs[n]), n
    # the default mode's column kernel is the one with atomics
    default = _matches(funcs, [r"ln_bwd_cols_kernel<(true|false), true>"])
    assert default and all(any(FP_ATOMIC.search(x) for x in funcs[n]) for n in default)


def test_new_instantiations_do_not_spill():
    logs = glob.glob(os.path.join(ROOT, "uniter_b200", "lib", "**", "rowops.o.ptxas.log"), recursive=True)
    if not logs or not os.path.exists(LIB):
        pytest.skip("no ptxas report next to the objects")
    blocks = re.split(r"ptxas info\s*: Compiling entry function '", open(logs[0]).read())
    names = [b.split("'", 1)[0] for b in blocks[1:]]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    seen = 0
    for d, b in zip(dem, blocks[1:]):
        if not any(re.search(p, d) for p in NEW_ROWS + NEW_COLS + NEW_FWD):
            continue
        seen += 1
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", b)
        assert m and m.group(1) == "0" and m.group(2) == "0", d
    assert seen == 24
