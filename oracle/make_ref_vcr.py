"""ORACLE — TEST INFRASTRUCTURE ONLY.  Recipe that stages the UNMODIFIED reference sources of the
visual commonsense reasoning (VCR) fine-tuning task into the git-ignored ``oracle/_ref/``, next to what
``oracle/make_ref.py`` stages, so that a tree built where a reference checkout exists carries them to
machines that have none.

    python -m oracle.make_ref_vcr        # needs a reference checkout ($UNITER_REFERENCE)

Files staged byte for byte (sha256 recorded in ``oracle/_ref/MANIFEST_vcr.json``):
  model/vcr.py                         UniterForVisualCommonsenseReasoning (tests/test_vcr_gpu.py runs it
                                       over the drop-in encoder)
  data/vcr.py                          vcr_collate / vcr_eval_collate, restated in uniter_b200.batching
  config/train-vcr-base-4gpu.json      the task's configuration (tools/vcr_step.py takes the token
                                       budget and max_txt_len from it)
"""
import json
import os
import shutil
import sys

from oracle.make_ref import DEFAULT_SRC, REF_DIR, _sha

FILES = ["model/vcr.py", "data/vcr.py", "config/train-vcr-base-4gpu.json"]


def stage(src=DEFAULT_SRC, force=False):
    """Copy FILES from `src` into oracle/_ref/ (idempotent).  Returns the manifest dict, or None when
    `src` is absent and nothing was staged before."""
    man_path = os.path.join(REF_DIR, "MANIFEST_vcr.json")
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
    os.makedirs(REF_DIR, exist_ok=True)
    with open(man_path, "w") as fh:
        json.dump(manifest, fh, indent=1, sort_keys=True)
    return manifest


if __name__ == "__main__":
    m = stage(force="--force" in sys.argv)
    if m is None:
        print("reference not found at %s and nothing staged" % DEFAULT_SRC)
        sys.exit(1)
    print("staged %d reference files into %s" % (len(m["files"]), REF_DIR))
