"""Generate tests/golden/re_batching.npz by running the UNMODIFIED reference's referring-expression code
(data/re.py, model/re.py) on CPU:

    python tests/golden/make_re_goldens.py          # needs a reference checkout ($UNITER_REFERENCE)

* `train/*`, `eval/*`: re_collate / re_eval_collate on seeded samples (`re_samples`);
* `keys/mlp1`, `keys/mlp2`: the state-dict keys of UniterForReferringExpressionComprehension;
* `neg/<seed>/*`: the negatives sample_neg_ix draws under fixed seeds of the global numpy / random
  generators, and the next draw of each generator afterwards (`re_neg_inputs`, `RE_NEG_SEEDS`).

The reference is imported through the shims of make_goldens.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_goldens import import_reference, import_reference_data  # noqa: E402


def re_samples(seed, n, D=16, eval_items=False):
    """Per-sample tuples as ReDataset / ReEvalDataset.__getitem__ return them (data/re.py:102-143,
    :206-248), seeded; a few obj_masks carry interior ones."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        tl = int(torch.randint(3, 12, (1,), generator=g))
        nbb = int(torch.randint(2, 10, (1,), generator=g))
        ids = torch.randint(1000, 2000, (tl,), generator=g)
        feat, pos = torch.randn(nbb, D, generator=g), torch.rand(nbb, 7, generator=g)
        am = torch.ones(tl + nbb, dtype=torch.long)
        om = torch.zeros(nbb, dtype=torch.uint8)
        if i % 3 == 1:
            om[int(torch.randint(0, nbb, (1,), generator=g))] = 1
        if eval_items:
            boxes = torch.rand(nbb, 4, generator=g).numpy() * 100
            out.append((ids, feat, pos, am, om, boxes[0].copy(), boxes, "s%03d" % i))
        else:
            out.append((ids, feat, pos, am, om, torch.tensor([int(torch.randint(0, nbb, (1,), generator=g))])))
    return out


RE_NEG_SEEDS = (3, 11)


def re_neg_inputs(seed, n=40):
    """Scores / targets / num_bbs for one call of the reference's sample_neg_ix (model/re.py:102-127)."""
    g = torch.Generator().manual_seed(1000 + seed)
    num_bbs = torch.randint(2, 12, (n,), generator=g).tolist()
    S = max(num_bbs)
    scores = torch.randn(n, S, generator=g)
    for i, nbb in enumerate(num_bbs):
        scores[i, nbb:] = -1e4
    targets = torch.tensor([int(torch.randint(0, nbb, (1,), generator=g)) for nbb in num_bbs]).view(n, 1)
    return scores, targets, num_bbs


def run_re_batching(out_path):
    """The reference's own re_collate / re_eval_collate (data/re.py) on seeded samples, the state-dict
    keys of its UniterForReferringExpressionComprehension for mlp 1 and 2, and the negatives its
    sample_neg_ix draws under fixed seeds of the global numpy / random generators."""
    import random
    rm = import_reference()[0]
    import_reference_data()
    import data.re as rre_data
    import model.re as rre
    rec = {}

    def put(prefix, batch):
        for k, v in batch.items():
            if k == "obj_boxes":
                rec[prefix + "/obj_boxes"] = np.concatenate(v, 0)
            else:
                rec["%s/%s" % (prefix, k)] = v.numpy() if torch.is_tensor(v) else np.array(v)

    put("train", rre_data.re_collate(re_samples(61, 7)))
    put("eval", rre_data.re_eval_collate(re_samples(62, 5, eval_items=True)))
    cfg = rm.UniterConfig(2000, hidden_size=32, num_hidden_layers=1, num_attention_heads=2, intermediate_size=64,
                          max_position_embeddings=64)
    for mlp in (1, 2):
        mod = rre.UniterForReferringExpressionComprehension(cfg, 16, loss="rank", mlp=mlp)
        rec["keys/mlp%d" % mlp] = np.array(sorted(mod.state_dict().keys()))
    for seed in RE_NEG_SEEDS:
        scores, targets, num_bbs = re_neg_inputs(seed)
        np.random.seed(seed)
        random.seed(seed)
        neg = mod.sample_neg_ix(scores, targets, num_bbs)
        rec["neg/%d/neg_ix" % seed] = neg.numpy()
        rec["neg/%d/next_np" % seed] = np.array(np.random.uniform(0, 1, 1))
        rec["neg/%d/next_py" % seed] = np.array(random.random())
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path, "%.1f KB" % (os.path.getsize(out_path) / 1024))


if __name__ == "__main__":
    run_re_batching(os.path.join(HERE, "re_batching.npz"))
