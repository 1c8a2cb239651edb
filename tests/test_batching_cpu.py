"""CPU: host-side batching (SURVEY.md §8f-3) against outputs of the reference's own
TokenBucketSampler (data/sampler.py) and collate functions (data/vqa.py, data/mlm.py) stored in
tests/golden/batching.npz by tests/golden/make_goldens.py — bit-exact (integer / copy logic)."""
import random

import numpy as np
import torch

from tests import util
from tests.golden.make_goldens import batching_samples
from uniter_b200 import batching


def _unflatten(flat, lens):
    out, o = [], 0
    for n in lens:
        out.append([int(x) for x in flat[o:o + n]])
        o += n
    return out


def test_token_bucket_sampler_reproduces_reference_batches():
    g = util.load_golden("batching")
    lens = [int(x) for x in g["lens"]]
    random.seed(5)
    got = list(iter(batching.TokenBucketSampler(lens, bucket_size=128, batch_size=1024)))
    assert got == _unflatten(g["batches_flat"], g["batches_len"])
    random.seed(6)
    got = list(iter(batching.TokenBucketSampler(lens, bucket_size=64, batch_size=800, droplast=True,
                                                size_multiple=4)))
    assert got == _unflatten(g["batches2_flat"], g["batches2_len"])
    # invariants of data/sampler.py:42-52: padded size under the budget, multiples of size_multiple
    for b in got:
        assert len(b) % 4 == 0
        assert max(lens[i] for i in b) * len(b) <= 800
    # an injected generator gives the same partition as the global one with the same seed
    alt = list(iter(batching.TokenBucketSampler(lens, 64, 800, True, 4, rng=random.Random(6))))
    assert alt == got


def test_sampler_rejects_impossible_budget():
    import pytest
    with pytest.raises(ValueError):
        list(iter(batching.TokenBucketSampler([100] * 16, 16, 500)))


def test_collates_match_reference_bit_exactly():
    g = util.load_golden("batching")
    for name, fn, lab in (("vqa", batching.vqa_collate, False), ("mlm", batching.mlm_collate, True)):
        b = fn(batching_samples(31, 6, lab))
        keys = [k[len(name) + 1:] for k in g if k.startswith(name + "/")]
        assert len(keys) >= 7
        for k in keys:
            ref = g["%s/%s" % (name, k)]
            assert b[k].dtype == torch.from_numpy(ref).dtype, k
            assert np.array_equal(b[k].numpy(), ref), (name, k)
        # host-known bookkeeping added for the packed GPU path
        lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
        assert b["attn_masks"].sum(1).tolist() == lens
        assert b["cu_seqlens"].dtype == torch.int32
        assert b["cu_seqlens"].tolist() == [0] + list(np.cumsum(lens))
        if lab:
            mask = b["txt_labels"] != -1
            assert torch.equal(b["mlm_targets"], b["txt_labels"][mask])
            L = b["attn_masks"].size(1)
            flat_mask = torch.zeros(b["attn_masks"].numel(), dtype=torch.bool)
            flat_mask[b["mlm_index"]] = True
            assert torch.equal(flat_mask.view(-1, L)[:, :mask.size(1)], mask)


def test_empty_and_single_sample_edges():
    one = batching_samples(3, 1, True)
    b = batching.mlm_collate(one)
    assert b["input_ids"].shape[0] == 1 and b["gather_index"].shape == b["attn_masks"].shape
    assert b["cu_seqlens"].tolist() == [0, one[0][0].numel() + one[0][1].size(0)]
    # a sampler over zero samples yields no batches
    assert list(iter(batching.TokenBucketSampler([], 8, 64))) == []


def test_itm_rank_and_mrm_batch_builders_match_reference_bit_exactly():
    """data/itm.py:240-374 (itm_rank_collate, the two hard-negative datasets incl. the stale-`tl`
    gather_index of :356-361, itm_rank_hn_collate) and data/mrm.py:76-227 (mrfr / mrc collates)
    against outputs of the reference's own code (tests/golden/itm_batching.npz)."""
    from tests.golden.make_goldens import itm_world, mrm_samples, rank_samples
    g = util.load_golden("itm_batching")

    def check(prefix, batch):
        keys = [k[len(prefix) + 1:] for k in g if k.startswith(prefix + "/")]
        assert len(keys) >= 6, prefix
        for k in keys:
            ref = g["%s/%s" % (prefix, k)]
            got = batch[k]
            if torch.is_tensor(got):
                assert got.dtype == torch.from_numpy(ref).dtype, (prefix, k)
                assert np.array_equal(got.numpy(), ref), (prefix, k)
            else:
                assert np.array_equal(np.array(got), ref), (prefix, k)

    check("rank", batching.itm_rank_collate(rank_samples(41, 3, 3)))
    txt_db, img_db, ids = itm_world()
    for name, cls in (("hn_t", batching.ItmRankDatasetHardNegFromText),
                      ("hn_i", batching.ItmRankDatasetHardNegFromImage)):
        ds = cls(txt_db, img_db, ids, txt_db.txt2img, txt_db.img2txts, neg_sample_size=4)
        for i in (0, 7):
            random.seed(100 + i)
            b = batching.itm_rank_hn_collate([ds[i]])
            check("%s%d" % (name, i), b)
            lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
            assert b["attn_masks"].sum(1).tolist() == lens            # host bookkeeping for the packed path
    check("mrfr", batching.mrfr_collate(mrm_samples(51, 5, False)))
    mb = batching.mrc_collate(mrm_samples(52, 5, True))
    check("mrc", mb)
    # mrm_index = flat positions of the masked regions, in the reference's row order
    L = mb["attn_masks"].size(1)
    flat = torch.zeros(mb["attn_masks"].numel(), dtype=torch.bool)
    flat[mb["mrm_index"]] = True
    assert torch.equal(flat.view(-1, L), mb["img_mask_tgt"].bool())
    assert mb["label_targets"].size(0) == mb["mrm_index"].numel()
