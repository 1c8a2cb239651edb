"""Build libub200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a.

    python -m uniter_b200.build [--force] [--verbose]

Objects are compiled in parallel (one nvcc per .cu) and linked into
``uniter_b200/lib/libub200.so``.  The .so is git-ignored.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
OBJ_DIR = os.path.join(LIB_DIR, "obj")
LIB_PATH = os.path.join(LIB_DIR, "libub200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-std=c++17", "-O3", "-lineinfo",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    # an object depends on its .cu, every header in csrc/ and the public header
    deps = [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))
                     if f.endswith((".h", ".cuh"))]
    deps.append(os.path.join(PKG_DIR, "..", "include", "ub200.h"))
    for d in deps:
        with open(d, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src, force, verbose):
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    stamp = obj + ".sha1"
    dig = _digest(path)
    if not force and os.path.exists(obj) and os.path.exists(stamp):
        with open(stamp) as fh:
            if fh.read().strip() == dig:
                return obj, ""
    cmd = [NVCC] + NVCC_FLAGS + ["-c", path, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, res.stdout, res.stderr))
    with open(stamp, "w") as fh:
        fh.write(dig)
    log = res.stderr if verbose else ""
    with open(obj + ".ptxas.log", "w") as fh:
        fh.write(res.stderr)
    return obj, log


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile_one(s, force, verbose), srcs))
    objs = [o for o, _ in results]
    for _, log in results:
        if log:
            sys.stderr.write(log)
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < newest:
        cmd = [NVCC, "-shared", "-o", LIB_PATH] + objs + [
            "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (res.stdout, res.stderr))
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
