"""ORACLE — TEST INFRASTRUCTURE ONLY.  Imports the UNMODIFIED reference modules staged by
``oracle/make_ref.py`` (or straight from the checkout at $UNITER_REFERENCE) under the package
root ``uniter_ref`` so that they cannot shadow or be shadowed by anything else on sys.path.

The only third-party symbols the reference's model code needs and this image lacks are shimmed:
``apex.normalization.fused_layer_norm.FusedLayerNorm := torch.nn.LayerNorm`` (same parameter names,
same eps argument, biased variance, fp32 statistics — SURVEY.md §8c), and for ``data/*.py`` the
module-level imports of horovod / lmdb / lz4 / msgpack / (cy)toolz, of which only
``cytoolz.partition_all / concat / curry`` and ``toolz.sandbox.unzip`` are executed.
"""
import importlib
import importlib.util
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")


def reference_root():
    """Directory holding model/ optim/ data/ of the reference, or None."""
    if os.path.exists(os.path.join(REF_DIR, "model", "model.py")):
        return REF_DIR
    src = os.environ.get("UNITER_REFERENCE", "/root/reference")
    if os.path.exists(os.path.join(src, "model", "model.py")):
        return src
    return None


def available():
    return reference_root() is not None


def _shim(name, **attrs):
    m = sys.modules.get(name)
    if m is None:
        m = types.ModuleType(name)
        sys.modules[name] = m
    for k, v in attrs.items():
        if not hasattr(m, k):
            setattr(m, k, v)
    return m


def _install_shims():
    try:
        import apex.normalization.fused_layer_norm  # noqa: F401  (a real apex wins)
    except Exception:
        apex = _shim("apex")
        norm = _shim("apex.normalization")
        fln = _shim("apex.normalization.fused_layer_norm", FusedLayerNorm=torch.nn.LayerNorm)
        apex.normalization = norm
        norm.fused_layer_norm = fln

    def partition_all(n, seq):
        seq = list(seq)
        for i in range(0, len(seq), n):
            yield tuple(seq[i:i + n])

    def unzip(seq):
        return tuple(zip(*list(seq)))

    def curry(f):
        return f

    for name, attrs in (
            ("horovod", {}), ("horovod.torch", dict(rank=lambda: 0, size=lambda: 1)),
            ("cytoolz", dict(partition_all=partition_all, curry=curry,
                             concat=lambda x: [b for a in x for b in a])),
            ("toolz", {}), ("toolz.sandbox", dict(unzip=unzip)),
            ("lmdb", {}), ("lz4", {}), ("lz4.frame", dict(compress=None, decompress=None)),
            ("msgpack", {}), ("msgpack_numpy", dict(patch=lambda: None))):
        try:
            importlib.import_module(name)
        except Exception:
            _shim(name, **attrs)
    if "horovod" in sys.modules and not hasattr(sys.modules["horovod"], "torch"):
        sys.modules["horovod"].torch = sys.modules["horovod.torch"]
    if not hasattr(sys.modules["toolz"], "sandbox"):
        sys.modules["toolz"].sandbox = sys.modules["toolz.sandbox"]
    if not hasattr(sys.modules["lz4"], "frame"):
        sys.modules["lz4"].frame = sys.modules["lz4.frame"]


def _package(name, path):
    """Register directory `path` as (namespace-like) package `name` without needing __init__.py."""
    if name in sys.modules:
        return sys.modules[name]
    spec = importlib.machinery.ModuleSpec(name, None, is_package=True)
    spec.submodule_search_locations = [path]
    mod = importlib.util.module_from_spec(spec)
    mod.__path__ = [path]
    sys.modules[name] = mod
    return mod


def load(*modules):
    """load("model.model", "model.pretrain") -> the reference modules (as uniter_ref.model.model ...).
    Raises RuntimeError when the reference is neither staged nor mounted."""
    root = reference_root()
    if root is None:
        raise RuntimeError("reference sources not staged: run `python -m oracle.make_ref` with a "
                           "reference checkout at $UNITER_REFERENCE")
    _install_shims()
    _package("uniter_ref", root)
    out = []
    for m in modules:
        pkg = m.split(".")[0]
        _package("uniter_ref." + pkg, os.path.join(root, pkg))
        out.append(importlib.import_module("uniter_ref." + m))
    return out[0] if len(out) == 1 else tuple(out)


def kind():
    """'reference' when the real reference code is importable here, else 'port'."""
    return "reference" if available() else "port"
