"""CPU: the word-region alignment task's host side and the error checker of its kernels.

* itm_ot_collate against what the reference's data/itm.py built on the same samples (tests/golden/wra.npz),
  bit for bit, and the text / region split taken from txt_lens against the slots ot_scatter assigns;
* tests/wra_check.py's float64 IPOT against the reference's optimal_transport_dist run in float64;
* the checker: a float32 stand-in of the kernels passes it, and mutations of the stand-in (a transposed
  plan, 49 iterations, eps 1e-6, a non-zero gradient on a row outside every pair, dist not rounded to
  16 bits) each fail it.
"""
import os
import sys

import numpy as np
import pytest
import torch

from tests import util, wra_check

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_wra_goldens  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    return util.load_golden("wra")


def test_itm_ot_collate_matches_the_reference(golden):
    from uniter_b200.batching import itm_ot_collate
    batch = itm_ot_collate(make_wra_goldens.wra_samples(81, 6))
    keys = [k[len("batch/"):] for k in golden if k.startswith("batch/")]
    assert keys
    for k in keys:
        want = golden["batch/" + k]
        v = batch["ot_inputs"][k[len("ot_inputs/"):]] if k.startswith("ot_inputs/") else batch[k]
        got = v.numpy() if torch.is_tensor(v) else np.array(v)
        assert got.dtype == want.dtype, (k, got.dtype, want.dtype)
        assert got.shape == want.shape and np.array_equal(got, want), k
    assert batch["ot_inputs"]["txt_pad"].dtype == torch.uint8
    assert batch["ot_txt_lens"].dtype == torch.int32 and batch["ot_txt_lens"].tolist() == batch["txt_lens"]
    t = batch["targets"]
    assert torch.equal(batch["ot_pos_index"], (t == 1).nonzero().view(-1))
    assert torch.equal(batch["ot_neg_index"], (t == 0).nonzero().view(-1))


def test_txt_lens_split_selects_the_ot_scatter_positions():
    """model/pretrain.py:170-183 scatters position j of pair b to text slot j (j < tl) or image slot j - tl;
    the packed split takes the first txt_lens[b] valid positions as text and the next num_bbs[b] as regions."""
    from uniter_b200.batching import itm_ot_collate
    batch = itm_ot_collate(make_wra_goldens.wra_samples(83, 9))
    sc = batch["ot_inputs"]["ot_scatter"]
    max_tl = batch["input_ids"].size(1)
    for b, (tl, nbb) in enumerate(zip(batch["txt_lens"], batch["num_bbs"])):
        valid = batch["attn_masks"][b].nonzero().view(-1)
        assert valid.tolist() == list(range(tl + nbb))                       # prefix mask
        assert sc[b, valid[:tl]].tolist() == list(range(tl))                 # text slots 0 .. tl-1
        assert (sc[b, valid[tl:]] - max_tl).tolist() == list(range(nbb))    # image slots 0 .. nbb-1
        # text slots past tl and image slots past nbb are padding in the reference's pads
        assert batch["ot_inputs"]["txt_pad"][b].tolist() == [0] * tl + [1] * (max_tl - tl)
        assert batch["ot_inputs"]["img_pad"][b, :nbb].sum() == 0


def _packed_from_padded(txt, img, tl, nb):
    rows, cu = [], [0]
    for b in range(txt.size(0)):
        rows += [txt[b, :tl[b]], img[b, :nb[b]]]
        cu.append(cu[-1] + tl[b] + nb[b])
    return torch.cat(rows), cu


@pytest.mark.parametrize("case", ["a", "b"])
def test_float64_ipot_matches_the_reference(golden, case):
    g = {k: torch.from_numpy(golden["ot/%s/%s" % (case, k)]) for k in
         ("txt", "img", "txt_pad", "img_pad", "g", "dist", "d_txt", "d_img")}
    tl = (~g["txt_pad"]).sum(1).tolist()
    nb = (~g["img_pad"]).sum(1).tolist()
    packed, cu = _packed_from_padded(g["txt"], g["img"], tl, nb)
    ref = wra_check.reference(packed, cu, tl, g["g"])
    assert (ref["dist"] - g["dist"]).abs().max().item() <= 1e-10
    for b in range(len(tl)):
        s = cu[b]
        assert (ref["d_packed"][s:s + tl[b]] - g["d_txt"][b, :tl[b]]).abs().max().item() <= 1e-10
        assert (ref["d_packed"][s + tl[b]:s + tl[b] + nb[b]] - g["d_img"][b, :nb[b]]).abs().max().item() <= 1e-10
        assert g["d_txt"][b, tl[b]:].abs().sum() == 0 and g["d_img"][b, nb[b]:].abs().sum() == 0


# ----------------------------------------------------------------------------- the checker
def standin(packed, cu, txt_lens, g, iters=50, eps=1e-5, transpose=False, round16=True, dummy_grad=False):
    """float32 model of the kernels: dist [B] and d_packed [T, H] in packed.dtype."""
    dt = packed.dtype
    rows = packed.float()
    d = torch.zeros_like(rows)
    dist = []
    for b, (s, m, n) in enumerate(wra_check.pairs(cu, txt_lens)):
        x, y = rows[s:s + m], rows[s + m:s + m + n]
        nx, ny = x.norm(dim=1, keepdim=True), y.norm(dim=1, keepdim=True)
        sx, sy = nx.clamp_min(eps), ny.clamp_min(eps)
        xh, yh = x / sx, y / sy
        C = 1 - xh @ yh.t()
        T = wra_check.ipot(C, iters)                              # [n, m]
        if transpose:
            T = T.reshape(m, n).t()
        dist.append((C * T.t()).sum())
        dC = float(g[b]) * T.t()
        for lo, r, dh, sr, nr in ((s, x, -dC @ yh, sx, nx), (s + m, y, -dC.t() @ xh, sy, ny)):
            coef = torch.where(nr >= eps, (dh * r).sum(1, keepdim=True) / sr ** 3, torch.zeros_like(nr))
            d[lo:lo + r.size(0)] = dh / sr - coef * r
    dist = torch.stack(dist)
    if round16:
        dist = dist.to(dt).float()
    if dummy_grad:
        d[cu[-1]:] = 1e-3
    return {"dist": dist, "d_packed": d.to(dt)}


def _case(dtype, seed=3, H=32):
    """Pairs whose rows come from a few directions (costs spread over [0, 2], a slowly converging plan),
    one text row of norm < 1e-5, one pair with a single region, and 5 rows of a padding sequence."""
    gen = torch.Generator().manual_seed(seed)
    dirs = torch.randn(4, H, generator=gen)
    geo = [(5, 7), (3, 1), (6, 9), (1, 4)]
    rows, cu, tl = [], [0], []
    for m, n in geo:
        k = torch.randint(0, 4, (m + n,), generator=gen)
        rows.append(dirs[k] * (0.5 + torch.rand(m + n, 1, generator=gen)) + 0.3 * torch.randn(m + n, H, generator=gen))
        cu.append(cu[-1] + m + n)
        tl.append(m)
    rows[0][1] = 2.0 ** -22
    packed = torch.cat(rows + [torch.randn(5, H, generator=gen)]).to(dtype)
    g = torch.tensor([1.0, -0.5, 2.0, 0.25]).to(dtype).float()
    return packed, cu, tl, g


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_checker_accepts_the_float32_standin(dtype):
    packed, cu, tl, g = _case(dtype)
    ref = wra_check.reference(packed, cu, tl, g)
    base = wra_check.baseline(packed, cu, tl, g)
    wra_check.check(standin(packed, cu, tl, g), ref, dtype, base)


@pytest.mark.parametrize("mutation", [dict(transpose=True), dict(iters=49), dict(eps=1e-6), dict(dummy_grad=True),
                                      dict(round16=False)], ids=["transposed_plan", "49_iterations", "eps_1e-6",
                                                                 "padding_row_gradient", "dist_not_rounded"])
def test_checker_rejects_mutations(mutation):
    dtype = torch.float16
    packed, cu, tl, g = _case(dtype)
    ref = wra_check.reference(packed, cu, tl, g)
    base = wra_check.baseline(packed, cu, tl, g)
    with pytest.raises(AssertionError):
        wra_check.check(standin(packed, cu, tl, g, **mutation), ref, dtype, base)
