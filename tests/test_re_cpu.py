"""CPU: the referring-expression task's host side and the error checker of its kernels.

* re_collate / re_eval_collate against what the reference's data/re.py built on the same samples
  (tests/golden/re_batching.npz), and `re_index` against the rows model/re.py's _get_image_hidden slices;
* re_neg_plan against the reference's sample_neg_ix under the same seeds of the global generators;
* the head's state-dict keys against the reference's, for mlp 1 and 2;
* tests/re_check.py: a float32 stand-in of the kernel math passes it, and mutations of the stand-in
  (a segment start off by one, a masked score in the log-sum-exp, a non-zero padding row of d_rows, a
  hard negative equal to the target) fail it.
"""
import os
import random
import sys

import numpy as np
import pytest
import torch

from tests import re_check, util

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_re_goldens  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return util.load_golden("re_batching")


def _assert_batch(prefix, batch, g):
    keys = [k[len(prefix) + 1:] for k in g if k.startswith(prefix + "/")]
    assert keys
    for k in keys:
        want = g["%s/%s" % (prefix, k)]
        v = batch[k]
        if k == "obj_boxes":
            v = np.concatenate(v, 0)
        got = v.numpy() if torch.is_tensor(v) else np.array(v)
        assert got.dtype == want.dtype, (k, got.dtype, want.dtype)
        assert got.shape == want.shape and np.array_equal(got, want), k


def _image_hidden_rows(batch):
    """The rows _get_image_hidden (model/re.py:129-157) slices, as flat positions of the padded layout."""
    B, L = batch["attn_masks"].shape
    pos = torch.arange(B * L).view(B, L)
    return torch.cat([pos[b, tl:tl + nbb] for b, (tl, nbb) in enumerate(zip(batch["txt_lens"], batch["num_bbs"]))])


def test_re_collate_matches_the_reference(golden):
    from uniter_b200.batching import re_collate
    batch = re_collate(make_re_goldens.re_samples(61, 7))
    _assert_batch("train", batch, golden)
    assert batch["obj_masks"].dtype == torch.uint8
    idx, seg = batch["re_index"], batch["re_seg"]
    want = _image_hidden_rows(batch)
    B, L = batch["attn_masks"].shape
    assert idx.numel() % 64 == 0 and torch.equal(idx[:want.numel()], want)
    assert (idx[want.numel():] == B * L).all()
    assert seg.dtype == torch.int32 and seg[1].tolist() == batch["num_bbs"]
    assert seg[0].tolist() == np.cumsum([0] + batch["num_bbs"][:-1]).tolist()


def test_re_eval_collate_matches_the_reference(golden):
    from uniter_b200.batching import re_eval_collate
    batch = re_eval_collate(make_re_goldens.re_samples(62, 5, eval_items=True))
    _assert_batch("eval", batch, golden)
    assert torch.equal(batch["re_index"][:sum(batch["num_bbs"])], _image_hidden_rows(batch))


def test_re_collate_rejects_a_target_outside_the_regions():
    from uniter_b200.batching import re_collate
    s = make_re_goldens.re_samples(61, 3)
    s[1] = s[1][:5] + (torch.tensor([s[1][1].size(0)]),)
    with pytest.raises(ValueError):
        re_collate(s)


def test_re_neg_plan_draws_like_the_reference(golden):
    from uniter_b200.heads import re_neg_plan
    np_state, py_state = np.random.get_state(), random.getstate()
    try:
        kinds = set()
        for seed in make_re_goldens.RE_NEG_SEEDS:
            scores, targets, num_bbs = make_re_goldens.re_neg_inputs(seed)
            np.random.seed(seed)
            random.seed(seed)
            plan = re_neg_plan(targets.view(-1).tolist(), num_bbs, 0.3)
            assert np.random.uniform(0, 1, 1)[0] == golden["neg/%d/next_np" % seed][0]
            assert random.random() == float(golden["neg/%d/next_py" % seed])
            ref = golden["neg/%d/neg_ix" % seed]
            for i, p in enumerate(plan):
                t = int(targets[i])
                if p < 0:
                    order = torch.argsort(scores[i], descending=True).tolist()
                    want = next(k for k in order if k != t)
                    kinds.add("hard")
                else:
                    want = p
                    kinds.add("easy")
                    assert p != t and 0 <= p < num_bbs[i]
                assert ref[i] == want, (seed, i)
        assert kinds == {"hard", "easy"}
    finally:
        np.random.set_state(np_state)
        random.setstate(py_state)


@pytest.mark.parametrize("mlp", [1, 2])
def test_re_state_dict_keys_match_the_reference(golden, mlp):
    from uniter_b200.heads import UniterForReferringExpressionComprehension
    from uniter_b200.model import UniterConfig
    cfg = UniterConfig(2000, hidden_size=64, num_hidden_layers=1, num_attention_heads=1, intermediate_size=64,
                       max_position_embeddings=64)
    mod = UniterForReferringExpressionComprehension(cfg, 16, loss="rank", mlp=mlp)
    assert sorted(mod.state_dict().keys()) == [str(k) for k in golden["keys/mlp%d" % mlp]]


# ----------------------------------------------------------------------------- checker
def standin(rows, w, b, seg, om, targets, plan, mode, margin, dloss, mutate=None):
    """The kernels' arithmetic in float32 (16-bit scores and d_rows, fp32 sums)."""
    dtype = rows.dtype
    B, S = om.shape
    masked = torch.tensor(-1e4).to(dtype).float()
    starts = seg[0] + (1 if mutate == "segment" else 0)
    live = re_check.live_mask(seg, om)
    scores = torch.full((B, S), float(masked))
    raw = torch.full((B, S), float(masked))
    for i in range(B):
        for k in range(int(seg[1, i])):
            s = (rows[int(starts[i]) + k].float() @ w.float() + b.float()[0]).to(dtype).float()
            raw[i, k] = s
            if live[i, k]:
                scores[i, k] = s
    out = {"scores": scores.to(dtype)}
    if mode == 0:
        return out
    lse_in = raw if mutate == "leak" else scores
    t = targets.view(-1)
    loss = torch.zeros(B)
    ds = torch.zeros(B, S)
    neg = torch.full((B,), -1, dtype=torch.int32)
    for i in range(B):
        ti, ni = int(t[i]), int(seg[1, i])
        if mode == re_check.CLS:
            lse = torch.logsumexp(lse_in[i], 0)
            loss[i] = lse - scores[i, ti]
            p = torch.exp(scores[i] - lse)
            p[ti] -= 1
            ds[i] = torch.where(live[i], p * dloss[i], torch.zeros(S))
        else:
            if int(plan[i]) >= 0:
                n = int(plan[i])
            elif mutate == "neg_target":
                n = max(range(ni), key=lambda k: (bool(live[i, k]), float(scores[i, k]), -k))
            else:
                n = re_check.hard_negative(scores[i].tolist(), live[i].tolist(), ti, ni)
            neg[i] = n
            if n < 0:
                continue
            sn, sp = torch.sigmoid(scores[i, n]), torch.sigmoid(scores[i, ti])
            h = margin + sn - sp
            loss[i] = h.clamp(min=0)
            if h >= 0:
                ds[i, n] += sn * (1 - sn) * dloss[i]
                ds[i, ti] += -sp * (1 - sp) * dloss[i]
    d_rows = torch.zeros(rows.shape)
    hid = re_check.padded(rows, seg, S).float()
    for i in range(B):
        st, ni = int(seg[0, i]), int(seg[1, i])
        d_rows[st:st + ni] = ds[i, :ni, None] * w.float()[None, :]
    if mutate == "padding":
        d_rows[-1] = 1e-3
    out.update(loss=loss, neg=neg if mode == re_check.RANK else None, d_rows=d_rows.to(dtype),
               dw=(ds[:, :, None] * hid).sum((0, 1)), db=ds.sum().reshape(1))
    return out


def _case(dtype, mode):
    """Five samples of 1, 2, 7, 4 and 3 regions with gaps and trailing padding rows; sample 2 has a
    masked interior region with the highest raw score; sample 3's target is its best region."""
    g = torch.Generator().manual_seed(7)
    H, lens = 64, [1, 2, 7, 4, 3]
    starts, r = [], 1
    for n in lens:
        starts.append(r)
        r += n + 1
    R = r + 5
    w = (torch.randn(H, generator=g) / 8).to(dtype)
    b = torch.tensor([0.1]).to(dtype)
    rows = torch.randn(R, H, generator=g).to(dtype)
    rows[starts[2] + 3] = (w.float() * 40).to(dtype)             # the masked region's raw score is the largest
    rows[starts[3] + 2] = (w.float() * 30).to(dtype)             # sample 3's best region is its target
    seg = torch.tensor([starts, lens], dtype=torch.int32)
    om = torch.zeros(5, max(lens), dtype=torch.uint8)
    for i, n in enumerate(lens):
        om[i, n:] = 1
    om[2, 3] = 1
    targets = torch.tensor([0, 1, 5, 2, 0])
    plan = torch.tensor([-1, -1, 4, -1, 2]) if mode == re_check.RANK else None
    dloss = torch.rand(5, generator=g) + 0.5
    return rows, w, b, seg, om, targets, plan, dloss


def _run(dtype, mode, mutate=None):
    rows, w, b, seg, om, targets, plan, dloss = _case(dtype, mode)
    if mode == re_check.RANK:
        targets = targets.clone()
        targets[0] = 0
    out = standin(rows, w, b, seg, om, targets, plan, mode, 0.2, dloss, mutate)
    ref = re_check.reference(rows, w, b, seg, om, out["scores"], targets, plan, mode, 0.2, dloss)
    if mode == re_check.RANK:
        base_neg = ref["neg"].clamp(min=0)
    else:
        base_neg = None
    keep = seg[1] >= (2 if mode == re_check.RANK else 1)
    base = None
    if bool(keep.all()):
        base = re_check.baseline(rows, w, b, seg, om, targets, base_neg, mode, 0.2, dloss)
    re_check.check(out, ref, dtype, base)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mode", [re_check.CLS, re_check.RANK])
def test_float32_standin_passes_the_checker(dtype, mode):
    _run(dtype, mode)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("mutate,mode", [("segment", re_check.CLS), ("leak", re_check.CLS),
                                         ("padding", re_check.CLS), ("neg_target", re_check.RANK)])
def test_checker_catches_a_mutation(dtype, mutate, mode):
    with pytest.raises(AssertionError):
        _run(dtype, mode, mutate)
