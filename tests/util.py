"""Shared helpers for the parity tests (test infrastructure; may import oracle/)."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

TINY = dict(vocab_size=2000, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
            intermediate_size=512, max_position_embeddings=64, type_vocab_size=2, img_dim=64)
BASE_L1 = dict(vocab_size=28996, hidden_size=768, num_hidden_layers=1, num_attention_heads=12,
               intermediate_size=3072, max_position_embeddings=512, type_vocab_size=2, img_dim=2048)


LARGE_L1 = dict(vocab_size=28996, hidden_size=1024, num_hidden_layers=1, num_attention_heads=16,
                intermediate_size=4096, max_position_embeddings=512, type_vocab_size=2, img_dim=2048)


def large_batch():
    from uniter_b200.synth import synth_batch
    return synth_batch(2, 0, 0, 0, 0, seed=3, txt_lens=[9, 6], num_bbs=[11, 14])


def load_golden(name):
    """name.npz plus its spill-over files name.part<k>.npz (no golden file exceeds 1 MB)."""
    out = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    k = 1
    while os.path.exists(os.path.join(GOLDEN, "%s.part%d.npz" % (name, k))):
        out.update(np.load(os.path.join(GOLDEN, "%s.part%d.npz" % (name, k))))
        k += 1
    return out


def state_checksum(state):
    acc = 0.0
    for k in sorted(state):
        acc += float(state[k].double().abs().sum()) + 3.0 * float(state[k].double().sum())
    return acc


def make_state(cfg, seed=0):
    from uniter_b200.synth import seeded_state, uniter_state_shapes
    shapes = uniter_state_shapes(cfg["hidden_size"], cfg["num_hidden_layers"], cfg["intermediate_size"],
                                 cfg["vocab_size"], cfg["max_position_embeddings"],
                                 cfg["type_vocab_size"], cfg["img_dim"])
    return seeded_state(shapes, seed=seed)


def tiny_batch():
    from uniter_b200.synth import synth_batch
    return synth_batch(4, 5, 12, 3, 9, seed=11, img_dim=64, vocab_size=2000)


def c1_batch(ragged):
    from uniter_b200.synth import synth_batch
    if ragged:
        return synth_batch(2, 0, 0, 0, 0, seed=0, txt_lens=[20, 14], num_bbs=[36, 30])
    return synth_batch(2, 0, 0, 0, 0, seed=0, txt_lens=[20, 20], num_bbs=[36, 36])


def make_model(cfg, state, dtype, device="cuda"):
    from uniter_b200.model import UniterConfig, UniterModel
    c = UniterConfig(cfg["vocab_size"], hidden_size=cfg["hidden_size"],
                     num_hidden_layers=cfg["num_hidden_layers"],
                     num_attention_heads=cfg["num_attention_heads"],
                     intermediate_size=cfg["intermediate_size"],
                     max_position_embeddings=cfg["max_position_embeddings"],
                     type_vocab_size=cfg["type_vocab_size"])
    m = UniterModel(c, cfg["img_dim"])
    m.load_state_dict(state, strict=True)
    return m.to(device=device, dtype=dtype)


def batch_to(batch, device):
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in batch.items()}


def rounded_state(state, dtype):
    """fp32 copy of the weights pre-rounded to the kernel dtype (oracle side of a parity check)."""
    return {k: v.to(dtype).float() for k, v in state.items()}


def head_state(module, seed, ties=()):
    """Seeded weights for one of our head modules, reproducing what the reference module holds
    after `load_state_dict(seeded_state(reference.state_dict() schema, seed))` in
    tests/golden/make_goldens.py: every key is drawn independently (sha1(key) ^ seed), and a
    parameter that the reference ties under a second name ends up with the value of the key that
    is loaded LAST — `ties` lists (our key, reference alias loaded later)."""
    from uniter_b200.synth import seeded_state
    own = {k: tuple(v.shape) for k, v in module.state_dict().items()}
    shapes = dict(own)
    for ours, alias in ties:
        shapes[alias] = shapes[ours]
    st = seeded_state(shapes, seed=seed)
    for ours, alias in ties:
        st[ours] = st[alias]
        if alias not in own:          # the alias only exists in the reference module
            del st[alias]
    return st


PRETRAIN_TIES = (("uniter.embeddings.word_embeddings.weight", "cls.predictions.decoder.weight"),
                 ("uniter.img_embeddings.img_linear.weight", "feat_regress.weight"))


def heads_batch():
    from uniter_b200.synth import synth_batch
    return synth_batch(3, 5, 9, 4, 8, seed=7, img_dim=64, vocab_size=2000, mlm_prob=0.3)


def tiny_config():
    from uniter_b200.model import UniterConfig
    c = TINY
    return UniterConfig(c["vocab_size"], hidden_size=c["hidden_size"],
                        num_hidden_layers=c["num_hidden_layers"],
                        num_attention_heads=c["num_attention_heads"],
                        intermediate_size=c["intermediate_size"],
                        max_position_embeddings=c["max_position_embeddings"],
                        type_vocab_size=c["type_vocab_size"])
