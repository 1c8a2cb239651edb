"""ORACLE — TEST INFRASTRUCTURE ONLY.  Recipe that stages the UNMODIFIED reference sources of the
hot path into the git-ignored ``oracle/_ref/``, so that a tree built where a reference checkout
exists carries them to machines that have none.

    python -m oracle.make_ref            # needs a reference checkout ($UNITER_REFERENCE)

Nothing under ``oracle/_ref/`` is ever committed (.gitignore) and the product (``uniter_b200``)
never imports it; users are ``tests/`` (G6: the reference's own heads over the drop-in encoder),
``bench.py --impl reference`` / ``cpu_baseline`` (kind "reference") and ``smoke()``.

Files staged byte for byte (sha256 recorded in ``oracle/_ref/MANIFEST.json``):
  model/{model,layer,pretrain,vqa,itm,ot}.py   the path + the heads named by BASELINE.json
  optim/{adamw,misc,sched}.py                  optimizer the fused AdamW is pinned against
  data/{sampler,data,itm,vqa,mlm,mrm}.py       host batching restated in uniter_b200.batching
  config/uniter-{base,large}.json              model configs
"""
import hashlib
import json
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(HERE, "_ref")
DEFAULT_SRC = os.environ.get("UNITER_REFERENCE", "/root/reference")

FILES = [
    "model/model.py", "model/layer.py", "model/pretrain.py", "model/vqa.py", "model/itm.py",
    "model/ot.py",
    "optim/__init__.py", "optim/adamw.py", "optim/misc.py", "optim/sched.py",
    "data/sampler.py", "data/data.py", "data/itm.py", "data/vqa.py", "data/mlm.py", "data/mrm.py",
    "config/uniter-base.json", "config/uniter-large.json",
    "config/train-vqa-base-4gpu.json", "config/pretrain-alldata-large-16gpu.json",
    "config/train-itm-coco-base-16gpu-hn.json",
]


def _sha(path):
    h = hashlib.sha256()
    with open(path, "rb") as fh:
        h.update(fh.read())
    return h.hexdigest()


def stage(src=DEFAULT_SRC, force=False):
    """Copy FILES from `src` into oracle/_ref/ (idempotent).  Returns the manifest dict, or None
    when `src` is absent and nothing was staged before."""
    man_path = os.path.join(REF_DIR, "MANIFEST.json")
    if not os.path.isdir(src):
        if os.path.exists(man_path):
            with open(man_path) as fh:
                return json.load(fh)
        return None
    manifest = {"source": src, "files": {}}
    for rel in FILES:
        s = os.path.join(src, rel)
        if not os.path.exists(s):
            continue
        d = os.path.join(REF_DIR, rel)
        os.makedirs(os.path.dirname(d), exist_ok=True)
        if force or not os.path.exists(d) or _sha(d) != _sha(s):
            shutil.copyfile(s, d)
        manifest["files"][rel] = _sha(d)
    with open(man_path, "w") as fh:
        json.dump(manifest, fh, indent=1, sort_keys=True)
    return manifest


if __name__ == "__main__":
    m = stage(force="--force" in sys.argv)
    if m is None:
        print("reference not found at %s and nothing staged" % DEFAULT_SRC)
        sys.exit(1)
    print("staged %d reference files into %s" % (len(m["files"]), REF_DIR))
