"""CPU: the VCR task's host side and the error checker of its LayerNorm kernels.

* vcr_collate / vcr_eval_collate against what the reference's data/vcr.py built on the same samples
  (tests/golden/vcr_batching.npz): qa and qar type-id patterns, an eval question with 20 sequences;
* the head's state-dict keys against the reference's;
* init_type_embedding / init_word_embedding against the tables the reference's methods made under the
  same torch seed, bit for bit, and the RNG state they leave behind;
* tests/vcr_check.py: a float32 stand-in of the ReLU + wide LayerNorm kernels passes it, and three
  mutations of the stand-in fail it (a mask on relu(pre) >= 0 instead of pre > 0, statistics over pre
  instead of relu(pre), a bias gradient without the dReLU).
"""
import os
import sys

import numpy as np
import pytest
import torch

from tests import util, vcr_check

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_vcr_goldens  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return util.load_golden("vcr_batching")


def _assert_batch(prefix, batch, g):
    keys = [k[len(prefix) + 1:] for k in g if k.startswith(prefix + "/")]
    assert keys
    for k in keys:
        want = g["%s/%s" % (prefix, k)]
        v = batch[k]
        got = v.numpy() if torch.is_tensor(v) else np.array(v)
        assert got.dtype == want.dtype, (k, got.dtype, want.dtype)
        assert got.shape == want.shape and np.array_equal(got, want), k


def test_vcr_collate_matches_the_reference(golden):
    from uniter_b200.batching import vcr_collate
    batch = vcr_collate(make_vcr_goldens.vcr_train_samples(81, 6))
    _assert_batch("train", batch, golden)
    assert set(np.unique(batch["txt_type_ids"].numpy())) == {0, 2, 3}
    assert batch["targets"].shape == (24, 1)
    B, L = batch["attn_masks"].shape
    lens = [a + b for a, b in zip(batch["txt_lens"], batch["num_bbs"])]
    assert batch["attn_masks"].sum(1).tolist() == lens
    assert batch["cu_seqlens"].tolist() == np.cumsum([0] + lens).tolist()


def test_vcr_eval_collate_matches_the_reference(golden):
    from uniter_b200.batching import vcr_eval_collate
    samples = make_vcr_goldens.vcr_eval_samples(82, 3)
    assert len(samples[0][0]) == 20
    batch = vcr_eval_collate(samples)
    _assert_batch("eval", batch, golden)
    assert batch["input_ids"].size(0) == 20 + 8 + 8


def _config():
    from uniter_b200.model import UniterConfig
    c = make_vcr_goldens.INIT_CFG
    return UniterConfig(c["vocab_size"], **{k: v for k, v in c.items() if k != "vocab_size"})


def test_vcr_state_dict_keys_match_the_reference(golden):
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    mod = UniterForVisualCommonsenseReasoning(_config(), 16)
    assert sorted(mod.state_dict().keys()) == [str(k) for k in golden["keys"]]


def test_vcr_init_methods_match_the_reference_bit_for_bit(golden):
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    mod = UniterForVisualCommonsenseReasoning(_config(), 16)
    mod.load_state_dict(make_vcr_goldens.init_state({k: tuple(v.shape) for k, v in mod.state_dict().items()}),
                        strict=True)
    rng = torch.get_rng_state()
    try:
        torch.manual_seed(make_vcr_goldens.INIT_SEED)
        mod.init_type_embedding()
        mod.init_word_embedding(make_vcr_goldens.NUM_SPECIAL_TOKENS)
        nxt = torch.rand(4)
    finally:
        torch.set_rng_state(rng)
    te = mod.uniter.embeddings
    assert np.array_equal(te.token_type_embeddings.weight.detach().numpy(), golden["init/token_type"])
    assert np.array_equal(te.word_embeddings.weight.detach().numpy(), golden["init/word"])
    assert te.word_embeddings.padding_idx is None and int(golden["init/word_padding_idx"]) == -1
    assert np.array_equal(nxt.numpy(), golden["init/next_rand"])
    assert te.token_type_embeddings.weight.shape == (4, 64)
    assert te.word_embeddings.weight.shape == (500 + 81, 64)
    assert set(dict(mod.named_parameters())) == set(mod.state_dict())


def test_vcr_init_retires_the_gradient_arena():
    """A gradient arena planned before init_* (e.g. by a warm-up step) is invalid afterwards: a fresh
    one includes the new tables, and asking the old one for their views raises instead of aliasing."""
    from uniter_b200.arena import GradArena
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    mod = UniterForVisualCommonsenseReasoning(_config(), 16)
    old = GradArena.attach(mod)
    assert old._still_valid()
    mod.init_type_embedding()
    mod.init_word_embedding(81)
    assert not old._still_valid()
    te = mod.uniter.embeddings
    with pytest.raises(RuntimeError, match="no view"):
        old.view(te.word_embeddings.weight)
    new = GradArena.attach(mod)
    assert new is not old and new._still_valid()
    assert new.view(te.word_embeddings.weight).shape == (581, 64)
    assert new.view(te.token_type_embeddings.weight).shape == (4, 64)
    ep = mod.uniter._ensure_arena()[1]
    assert ep["front_small"]["type"][1] == 4 * 64


# ----------------------------------------------------------------------------- checker
def standin(pre, gamma, beta, dy, mutate=None):
    """The kernels' arithmetic in float32: statistics of relu(pre) (of pre with mutate="stats"), 16-bit
    y / dx / dpre, fp32 column sums."""
    dtype = pre.dtype
    p = pre.float()
    x = p if mutate == "stats" else p.clamp(min=0)
    W = x.size(1)
    mean = x.sum(1, keepdim=True) / W
    rstd = torch.rsqrt(((x - mean) ** 2).sum(1, keepdim=True) / W + 1e-12)
    xh = (x - mean) * rstd
    y = (xh * gamma.float() + beta.float()).to(dtype)
    d = dy.float()
    gd = d * gamma.float()
    s1, s2 = gd.sum(1, keepdim=True) / W, (gd * xh).sum(1, keepdim=True) / W
    dx = rstd * (gd - s1 - xh * s2)
    live = (x >= 0) if mutate == "mask" else (p > 0)
    dpre = (dx * live).to(dtype)
    lin = dx.to(dtype) if mutate == "bias" else dpre
    return dict(y=y, dx=dx.to(dtype), dpre=dpre, dgamma=(d * xh).sum(0), dbeta=d.sum(0), dbias=lin.float().sum(0))


def _run(dtype, rows, W, mutate=None):
    pre, gamma, beta, dy = vcr_check.relu_ln_case(rows, W, dtype, seed=rows + W)
    out = standin(pre, gamma, beta, dy, mutate)
    base = vcr_check.relu_ln_baseline(dy, pre, gamma, beta)
    fails = vcr_check.check_fwd(out["y"], vcr_check.relu_ln_fwd_reference(pre, gamma, beta), base["y"], dtype)
    fails += vcr_check.check_bwd(out, vcr_check.relu_ln_bwd_reference(dy, pre, gamma), base, pre, dtype)
    assert not fails, fails


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows,W", [(3, 1536), (5, 2048), (4, 768)])
def test_float32_standin_passes_the_checker(dtype, rows, W):
    _run(dtype, rows, W)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mutate", ["mask", "stats", "bias"])
def test_checker_catches_a_mutation(dtype, mutate):
    with pytest.raises(AssertionError):
        _run(dtype, 3, 1536, mutate)
