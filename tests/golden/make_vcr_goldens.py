"""Generate tests/golden/vcr_batching.npz by running the UNMODIFIED reference's VCR code (data/vcr.py,
model/vcr.py) on CPU:

    python tests/golden/make_vcr_goldens.py         # needs a reference checkout ($UNITER_REFERENCE)

* `train/*`, `eval/*`: vcr_collate / vcr_eval_collate on seeded samples (`vcr_train_samples`,
  `vcr_eval_samples`): questions with 4 answer choices, qa type ids (0 for [CLS] + question, 2 for the
  answer) and qar type ids (3 for the rationale), and one eval question with its 4 + 16 sequences;
* `keys`: the state-dict keys of UniterForVisualCommonsenseReasoning;
* `init/*`: the token-type and word tables after init_type_embedding() and init_word_embedding(81)
  under a fixed torch seed (`INIT_SEED`), starting from the seeded weights of `init_state`.

The reference is imported through the shims of make_goldens.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_goldens import import_reference, import_reference_data  # noqa: E402

CLS, SEP = 101, 102
NUM_SPECIAL_TOKENS = 81              # train_vcr.py
INIT_SEED = 42
INIT_CFG = dict(vocab_size=500, hidden_size=64, num_hidden_layers=1, num_attention_heads=1,
                intermediate_size=64, max_position_embeddings=64, type_vocab_size=2)


def _choice(g, q, a, r, nbb, D, with_target):
    """One sequence as VcrDataset / VcrEvalDataset build it (data/vcr.py:120-160, :218-260): [CLS] q [SEP]
    a [SEP] (type ids 0 / 2), plus r [SEP] with type 3 for a rationale sequence."""
    ids = [CLS] + q + [SEP] + a + [SEP]
    types = [0] + [0] * len(q) + [2] * (len(a) + 2)
    if r is not None:
        ids = ids + r + [SEP]
        types = types[:-1] + [3] * (len(r) + 2)
    feat, pos = torch.randn(nbb, D, generator=g), torch.rand(nbb, 7, generator=g)
    out = (torch.tensor(ids), torch.tensor(types), feat, pos, torch.ones(len(ids) + nbb, dtype=torch.long))
    if with_target:
        out = out + (torch.tensor([int(torch.randint(0, 2, (1,), generator=g))]),)
    return out


def _tokens(g, lo, hi):
    return torch.randint(1000, 1900, (int(torch.randint(lo, hi, (1,), generator=g)),), generator=g).tolist()


def vcr_train_samples(seed, n_questions, D=16):
    """Per-question tuples of 4 choices as VcrDataset.__getitem__ returns them; even questions are qa
    (answer choices), odd ones qar (rationale choices after the right answer)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n_questions):
        q, nbb = _tokens(g, 2, 9), int(torch.randint(2, 12, (1,), generator=g))
        a = _tokens(g, 1, 6)
        choices = []
        for _ in range(4):
            if i % 2 == 0:
                choices.append(_choice(g, q, _tokens(g, 1, 7), None, nbb, D, True))
            else:
                choices.append(_choice(g, q, a, _tokens(g, 1, 9), nbb, D, True))
        out.append(tuple(choices))
    return out


def vcr_eval_samples(seed, n_questions, D=16):
    """(choices, qid, qa_target, qar_target) per question as VcrEvalDataset.__getitem__ returns them:
    question 0 carries all 4 + 16 sequences (split "test"), the others their 4 answer sequences and the 4
    rationale sequences of the right answer (split "val")."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n_questions):
        q, nbb = _tokens(g, 2, 9), int(torch.randint(2, 12, (1,), generator=g))
        answers = [_tokens(g, 1, 6) for _ in range(4)]
        rationales = [_tokens(g, 1, 8) for _ in range(4)]
        qa_t, qar_t = int(torch.randint(0, 4, (1,), generator=g)), int(torch.randint(0, 4, (1,), generator=g))
        choices = [_choice(g, q, a, None, nbb, D, False) for a in answers]
        for k, a in enumerate(answers):
            if i == 0 or k == qa_t:
                choices += [_choice(g, q, a, r, nbb, D, False) for r in rationales]
        out.append((tuple(choices), "q%03d" % i, torch.tensor([qa_t]), torch.tensor([qar_t])))
    return out


def init_state(shapes):
    from uniter_b200.synth import seeded_state
    return seeded_state(shapes, seed=21)


def run_vcr_batching(out_path):
    rm = import_reference()[0]
    import_reference_data()
    import data.vcr as rvcr_data
    import model.vcr as rvcr
    rec = {}

    def put(prefix, batch):
        for k, v in batch.items():
            rec["%s/%s" % (prefix, k)] = v.numpy() if torch.is_tensor(v) else np.array(v)

    put("train", rvcr_data.vcr_collate(vcr_train_samples(81, 6)))
    put("eval", rvcr_data.vcr_eval_collate(vcr_eval_samples(82, 3)))
    cfg = rm.UniterConfig(INIT_CFG["vocab_size"], **{k: v for k, v in INIT_CFG.items() if k != "vocab_size"})
    mod = rvcr.UniterForVisualCommonsenseReasoning(cfg, 16)
    rec["keys"] = np.array(sorted(mod.state_dict().keys()))
    mod.load_state_dict(init_state({k: tuple(v.shape) for k, v in mod.state_dict().items()}), strict=True)
    torch.manual_seed(INIT_SEED)
    mod.init_type_embedding()
    mod.init_word_embedding(NUM_SPECIAL_TOKENS)
    rec["init/token_type"] = mod.uniter.embeddings.token_type_embeddings.weight.detach().numpy()
    rec["init/word"] = mod.uniter.embeddings.word_embeddings.weight.detach().numpy()
    rec["init/word_padding_idx"] = np.array(-1 if mod.uniter.embeddings.word_embeddings.padding_idx is None
                                            else mod.uniter.embeddings.word_embeddings.padding_idx)
    rec["init/next_rand"] = torch.rand(4).numpy()
    np.savez_compressed(out_path, **rec)
    print("wrote", out_path, "%.1f KB" % (os.path.getsize(out_path) / 1024))


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    run_vcr_batching(os.path.join(HERE, "vcr_batching.npz"))
