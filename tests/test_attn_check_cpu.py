"""CPU: the host mirror of the dropout generator and the attention checker of tests/attn_check.py.

The mirror is pinned to the Random123 known-answer vectors of Philox-4x32-10 and to a plain
Python loop.  The checker must accept a float32 stand-in for a kernel result and reject each
single-item mutation of it that a scheduling, masking or accumulation bug would produce."""
import copy
import math

import numpy as np
import pytest
import torch

from oracle import philox
from tests import attn_check as ac


def _philox_loop(c, k):
    c, k = list(c), list(k)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return c


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    assert tuple(int(w) for w in philox.philox4x32(*ctr, *key)) == want
    assert tuple(_philox_loop(ctr, key)) == want


def test_rand16_matches_plain_loop():
    rng = np.random.default_rng(0)
    seed, stream = (1 << 40) + 12345, (7 << 33) + 99
    e = np.concatenate([np.arange(64), rng.integers(0, 1 << 50, 200)]).astype(np.uint64)
    got = philox.rand16(seed, stream, e)
    for i, ei in enumerate(e.tolist()):
        g = ei >> 3
        w = _philox_loop((g & 0xFFFFFFFF, g >> 32, stream & 0xFFFFFFFF, stream >> 32),
                         (seed & 0xFFFFFFFF, seed >> 32))[(ei & 7) >> 1]
        assert int(got[i]) == ((w >> 16) if ei & 1 else (w & 0xFFFF)), i


def test_dropout_params_and_device_offset():
    thr, inv = philox.dropout_params(0.1)
    assert thr == 6554 and inv == float(np.float32(65536.0) / np.float32(65536 - 6554))
    assert philox.dropout_params(1e-9)[0] == 1 and philox.dropout_params(0.99999999)[0] == 65535
    assert philox.stream_with_offset(5, 3) == 5 + (3 << 20)
    assert philox.stream_with_offset((1 << 64) - 1, 1) == (1 << 20) - 1
    # attention element index ((b * nheads + h) * 512 + q) * 512 + key
    m = philox.attn_keep(3, 9, 0.3, 12, 5, np.arange(12), 70, 90)
    b, h, q, k = 5, 7, 33, 81
    assert m[h, q, k] == (philox.rand16(3, 9, ((b * 12 + h) * 512 + q) * 512 + k) >= philox.dropout_params(0.3)[0])
    assert abs(m.mean() - 0.7) < 0.01


def _case(lens, heads, dtype, p, seed=0):
    g = torch.Generator().manual_seed(seed)
    T, H = sum(lens), heads * ac.D
    qkv = torch.randn(T, 3 * H, generator=g).to(dtype)
    dctx = torch.randn(T, H, generator=g).to(dtype)
    dbias0 = torch.randn(3 * H, generator=g)
    thr_inv = philox.dropout_params(p)[1] if p else 1.0
    keep = ac.keep_masks(lens, heads, p, 17, 4, "cpu")
    ref = ac.attention_reference(qkv, dctx, lens, heads, keep, thr_inv, dbias0, p_dtype=dtype)
    base = ac.attention_baseline(qkv, dctx, lens, heads, keep, thr_inv)
    f32 = ac.attention_reference(qkv, dctx, lens, heads, keep, thr_inv, dbias0, dtype=torch.float32)
    stand_in = dict(ctx=f32["ctx"].to(dtype), lse=f32["lse"], dqkv=f32["dqkv"].to(dtype), dbias=f32["dbias"])
    return qkv, dctx, dbias0, keep, thr_inv, ref, base, stand_in


def _item(qkv, dctx, lens, heads, b, h, keep, inv_keep):
    """float64 P, Pd, dS, q, k, dO of one (sequence, head)."""
    o, S = sum(lens[:b]), lens[b]
    q, k, v = [t[h] for t in ac._split(qkv.double(), o, S, heads)]
    do = dctx.double()[o:o + S, h * ac.D:(h + 1) * ac.D]
    P = torch.softmax(q @ k.t() * ac.SCALE, -1)
    m = keep[b][h].double() * inv_keep if keep is not None else 1.0
    dP = (do @ v.t()) * m
    dS = P * (dP - (dP * P).sum(-1, keepdim=True))
    return P, P * m, dS, q, k, do


CPU_CASES = [([5, 0, 37, 64, 65, 100, 1], 3, torch.bfloat16, 0.0),
             ([5, 0, 37, 64, 65, 100, 1], 3, torch.float16, 0.1),
             ([128, 2, 70, 0], 2, torch.bfloat16, 0.1),
             ([128, 2, 70, 0], 2, torch.float16, 0.0)]


@pytest.mark.parametrize("lens,heads,dtype,p", CPU_CASES)
def test_checker_accepts_stand_in_and_rejects_mutations(lens, heads, dtype, p):
    qkv, dctx, dbias0, keep, inv, ref, base, good = _case(lens, heads, dtype, p)
    fails, _ = ac.check_attention(good, ref, base, lens, heads, dtype, dbias0)
    assert not fails, fails
    H = heads * ac.D
    b = max(range(len(lens)), key=lambda i: lens[i])          # the longest item: hardest to see one row in
    o, S = sum(lens[:b]), lens[b]
    rows = slice(o, o + S)
    h, h2 = heads - 1, 0
    cols = [slice(j * H + h * ac.D, j * H + (h + 1) * ac.D) for j in range(3)]
    cols2 = [slice(j * H + h2 * ac.D, j * H + (h2 + 1) * ac.D) for j in range(3)]
    P, Pd, dS, q, k, do = _item(qkv, dctx, lens, heads, b, h, keep, inv)

    def expect_fail(mut, names, what):
        fails, _ = ac.check_attention(mut, ref, base, lens, heads, dtype, dbias0)
        for n in names:
            assert any(f.startswith(n + ":") for f in fails), "%s not caught in %s: %s" % (what, n, fails)

    m = copy.deepcopy(good)                                    # item (b, h) holds head h2's results
    m["ctx"][rows, h * ac.D:(h + 1) * ac.D] = good["ctx"][rows, h2 * ac.D:(h2 + 1) * ac.D]
    m["lse"][h, rows] = good["lse"][h2, rows]
    for c, c2 in zip(cols, cols2):
        m["dqkv"][rows, c] = good["dqkv"][rows, c2]
    expect_fail(m, ["ctx", "lse", "dq", "dk", "dv"], "swapped head")

    m = copy.deepcopy(good)                                    # item (b, h) never written
    m["ctx"][rows, h * ac.D:(h + 1) * ac.D] = float("nan")
    m["lse"][h, rows] = float("nan")
    for c in cols:
        m["dqkv"][rows, c] = float("nan")
    expect_fail(m, ["ctx", "lse", "dq", "dk", "dv"], "unwritten item")

    q0 = S // 2                                                # query row q0 missing from dV / from dK
    m = copy.deepcopy(good)
    m["dqkv"][rows, cols[2]] = (good["dqkv"][rows, cols[2]].double() - torch.outer(Pd[q0], do[q0])).to(dtype)
    expect_fail(m, ["dv"], "query row missing from dV")
    m = copy.deepcopy(good)
    m["dqkv"][rows, cols[1]] = (good["dqkv"][rows, cols[1]].double()
                                - ac.SCALE * torch.outer(dS[q0], q[q0])).to(dtype)
    expect_fail(m, ["dk"], "query row missing from dK")

    k0 = S // 3                                                # key row k0 missing from dQ
    m = copy.deepcopy(good)
    m["dqkv"][rows, cols[0]] = (good["dqkv"][rows, cols[0]].double()
                                - ac.SCALE * torch.outer(dS[:, k0], k[k0])).to(dtype)
    expect_fail(m, ["dq"], "key row missing from dQ")

    m = copy.deepcopy(good)                                    # one row's lse off by ln 2
    m["lse"][h, o + q0] += math.log(2.0)
    expect_fail(m, ["lse"], "lse off by ln 2")

    # the bias gradient missing, or counting twice, the smallest non-empty item
    bs = min((i for i in range(len(lens)) if lens[i]), key=lambda i: lens[i])
    rs = slice(sum(lens[:bs]), sum(lens[:bs]) + lens[bs])
    contrib = torch.zeros(3 * H)
    for c in cols:
        contrib[c] = good["dqkv"][rs, c].float().sum(0)
    for sign, what in ((-1, "item missing from dbias"), (1, "item counted twice in dbias")):
        m = copy.deepcopy(good)
        m["dbias"] = good["dbias"] + sign * contrib
        expect_fail(m, ["dbias"], what)


def test_bias_check_resolves_one_item_at_pretraining_scale():
    """C2 lengths (T = 3451, 12 heads): one missing or doubled item of the QKV bias gradient, the
    smallest of every head, stays far above the bound."""
    from uniter_b200.synth import synth_batch
    bt = synth_batch(64, 12, 28, 26, 46, 1234, img_dim=8, vocab_size=2000)
    lens = [t + n for t, n in zip(bt["txt_lens"], bt["num_bbs"])]
    assert sum(lens) == 3451
    heads, dtype = 12, torch.bfloat16
    qkv, dctx, dbias0, keep, inv, ref, base, good = _case(lens, heads, dtype, 0.1, seed=3)
    fails, stats = ac.check_attention(good, ref, base, lens, heads, dtype, dbias0)
    assert not fails, fails
    H = heads * ac.D
    bs = min(range(len(lens)), key=lambda i: lens[i])
    rs = slice(sum(lens[:bs]), sum(lens[:bs]) + lens[bs])
    for h in range(heads):
        m = copy.deepcopy(good)
        for j in range(3):
            c = slice(j * H + h * ac.D, j * H + (h + 1) * ac.D)
            m["dbias"][c] -= good["dqkv"][rs, c].float().sum(0)
        fails, _ = ac.check_attention(m, ref, base, lens, heads, dtype, dbias0)
        assert any(f.startswith("dbias:") for f in fails), (h, fails)
