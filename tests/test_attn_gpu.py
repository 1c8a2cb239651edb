"""GPU: fused varlen attention (ops.attn_fwd / attn_bwd) against a float64 reference.

Every output (ctx, lse, dQ, dK, dV and the accumulated QKV-bias gradient) is compared with a
float64 reference of model/layer.py:80-100 computed per (sequence, head), with the eager 16-bit
torch computation as the yardstick (tests/attn_check.py), elementwise and per (sequence, head).
With dropout, the reference applies the mask of the host mirror of the kernels' Philox generator
(oracle/philox.py), so the masks are compared exactly as well.  Outputs are written into NaN-filled
buffers, so an element that is never written fails.

max_seqlen <= 128 runs the persistent short kernels (grid min(2 x SMs, B x heads), items ordered
head-major and balanced by cost); longer runs the multi-block kernels with the fp32 dQ accumulator."""
import numpy as np
import pytest
import torch

from oracle import philox
from tests import attn_check as ac

pytestmark = pytest.mark.gpu

SEED, STREAM = 1234567, 42


def _c2_lens():
    from uniter_b200.synth import synth_batch
    b = synth_batch(64, 12, 28, 26, 46, 1234, img_dim=8, vocab_size=2000)
    return [t + n for t, n in zip(b["txt_lens"], b["num_bbs"])]


def _large_lens():
    """UNITER-large batch: 64 lengths in [1, 128] including the block edges."""
    g = np.random.default_rng(16)
    lens = g.integers(1, 129, 64).tolist()
    lens[3:9] = [1, 63, 64, 65, 127, 128]
    return lens


def _lens_b(n, seed):
    return np.random.default_rng(seed).integers(1, 129, n).tolist()


def _inputs(lens, heads, dtype, regime="randn", seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    T, H = sum(lens), heads * ac.D
    qkv = torch.randn(T, 3 * H, device="cuda", generator=g)
    if regime == "sharp":       # score std ~ 20: softmax close to one-hot
        qkv[:, :H] *= 20.0
    elif regime == "flat":      # all scores 0: uniform softmax
        qkv[:, :H] = 0.0
    dctx = torch.randn(T, H, device="cuda", generator=g)
    dbias0 = torch.randn(3 * H, device="cuda", generator=g)
    return qkv.to(dtype), dctx.to(dtype), dbias0


def _run(qkv, dctx, lens, heads, p=0.0, max_seqlen=None, dbias0=None, stream=STREAM, rng_dev=None):
    """Kernel forward and backward into NaN-filled outputs."""
    from uniter_b200 import ops
    T, H = dctx.shape
    cu = ac.cu_seqlens(lens, "cuda")
    ms = max_seqlen or max(max(lens), 1)
    nan = float("nan")
    ctx = torch.full((T, H), nan, device="cuda", dtype=qkv.dtype)
    lse = torch.full((heads, T), nan, device="cuda")
    dqkv = torch.full_like(qkv, nan)
    dev = None if rng_dev is None else rng_dev.data_ptr()
    ops.attn_fwd(qkv, cu, ms, heads, dropout_p=p, rng_seed=SEED, rng_stream=stream, rng_offset_dev=dev,
                 ctx=ctx, lse=lse)
    dbias = None if dbias0 is None else dbias0.clone()
    ops.attn_bwd(qkv, ctx, lse, dctx, cu, ms, heads, dropout_p=p, rng_seed=SEED, rng_stream=stream,
                 dbias=dbias, rng_offset_dev=dev, dqkv=dqkv)
    torch.cuda.synchronize()
    return dict(ctx=ctx, lse=lse, dqkv=dqkv, dbias=dbias)


def _reference(qkv, dctx, lens, heads, p, dbias0, stream=STREAM):
    keep = ac.keep_masks(lens, heads, p, SEED, stream, "cuda")
    inv = philox.dropout_params(p)[1] if p else 1.0
    ref = ac.attention_reference(qkv, dctx, lens, heads, keep, inv, dbias0, p_dtype=qkv.dtype)
    base = ac.attention_baseline(qkv, dctx, lens, heads, keep, inv)
    return ref, base


def _check(lens, heads, dtype, p=0.0, regime="randn", max_seqlen=None, label=""):
    qkv, dctx, dbias0 = _inputs(lens, heads, dtype, regime, seed=sum(lens) + heads)
    ref, base = _reference(qkv, dctx, lens, heads, p, dbias0)
    out = _run(qkv, dctx, lens, heads, p, max_seqlen, dbias0)
    fails, stats = ac.check_attention(out, ref, base, lens, heads, dtype, dbias0)
    print("\n[attn %s B=%d heads=%d T=%d %s p=%g %s max_seqlen=%s] %s" % (
        label, len(lens), heads, sum(lens), str(dtype)[6:], p, regime, max_seqlen, ac.format_stats(stats)))
    assert not fails, "\n".join(fails)
    return out, ref


DTYPES = [torch.bfloat16, torch.float16]

# the original kernel cases: short (<= 128) and long (> 128) paths, 2 and 12 heads
CASES = [
    [56, 56], [56, 44], [1], [7, 128, 64, 1, 33], [129], [300, 5, 17], [512, 256],
    [74, 38, 61, 50, 45, 66, 53, 70],
]


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 2e-2), (torch.float16, 4e-3)])
@pytest.mark.parametrize("lens", CASES)
@pytest.mark.parametrize("heads", [2, 12])
def test_attention_fwd_bwd(dtype, tol, lens, heads):
    """The checker's bounds, and also this test's original whole-tensor bounds (max error against
    tol times the largest reference value)."""
    out, ref = _check(lens, heads, dtype)
    H = heads * ac.D
    err = (out["ctx"].double() - ref["ctx"]).abs().max().item()
    assert err <= tol * max(1.0, ref["ctx"].abs().max().item()), "fwd err %.3e" % err
    g = ref["dqkv"]
    eb = (out["dbias"].double() - ref["dbias"]).abs().max().item()
    assert eb <= 2 * tol * max(1.0, g.abs().sum(0).max().item()), "dbias err %.3e" % eb
    for name, sl in (("dq", slice(0, H)), ("dk", slice(H, 2 * H)), ("dv", slice(2 * H, 3 * H))):
        e = (out["dqkv"][:, sl].double() - g[:, sl]).abs().max().item()
        assert e <= 2 * tol * max(1.0, g[:, sl].abs().max().item()), "%s err %.3e" % (name, e)


# (name, lens, heads): the pre-training path.  C2 gives the 264 CTAs of an H100 SXM 768 items; the
# 16-head batch 1024 (several per CTA, so the prefetch into the second slot and the per-head bias
# flush run many times per CTA)
SHORT = {
    "c2": (_c2_lens, 12),
    "c2_dummy_empty": (lambda: _c2_lens() + [0], 12),        # graph mode: B + 1 sequences
    "c2_dummy_127": (lambda: _c2_lens() + [127], 12),
    "large16": (_large_lens, 16),
    "empty_edges": (lambda: [0, 0, 50, 0, 70, 128, 1, 0, 65, 0], 12),
    "b32": (lambda: _lens_b(32, 32), 12),
    "b33": (lambda: _lens_b(33, 33), 12),
    "b1": (lambda: [100], 12),
}
LONG = {
    "long_mix12": (lambda: [512, 1, 128, 129, 256, 0, 383], 12),
    "long_mix16": (lambda: [512, 1, 128, 129, 256, 0, 383], 16),
}
DROPOUT = ["c2", "c2_dummy_127", "large16", "empty_edges", "b33", "long_mix12"]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(SHORT) + list(LONG))
def test_attention_matches_reference(name, dtype):
    make, heads = {**SHORT, **LONG}[name]
    _check(make(), heads, dtype, label=name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", DROPOUT)
def test_attention_dropout_matches_reference(name, dtype):
    make, heads = {**SHORT, **LONG}[name]
    _check(make(), heads, dtype, p=0.1, label=name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("regime", ["sharp", "flat"])
@pytest.mark.parametrize("name", ["c2", "long_mix12"])
def test_attention_score_regimes(name, regime, dtype):
    make, heads = {**SHORT, **LONG}[name]
    _check(make(), heads, dtype, regime=regime, label=name)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_attention_long_path_agrees_with_short_path(dtype, p):
    """C2 through the long kernels (max_seqlen = 129) and the short ones: both within the
    checker's bounds of the same reference (the mask is keyed on (b, h, q, key) on both paths)."""
    lens = _c2_lens()
    _check(lens, 12, dtype, p=p, label="c2 short")
    _check(lens, 12, dtype, p=p, max_seqlen=129, label="c2 long")


# ---------------------------------------------------------------- exact invariances
INVARIANCE = {
    # (lens, indices that keep length and content, max_seqlen)
    "short": ([50, 0, 128, 7, 64, 65, 1, 100] * 5 + [33], [2, 5, 8, 11, 19, 26, 33, 40], 128),
    "long": ([300, 17, 0, 129, 512, 64, 200, 383], [0, 1, 3, 4, 6], 512),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("path", ["short", "long"])
def test_attention_item_independent_of_neighbours(path, p, dtype):
    """A sequence that keeps its index and length gives bit-identical ctx, lse and dqkv whatever the
    other sequences hold: their lengths (which shift its offset), content and magnitude (up to
    +-1e4).  Each item's arithmetic reads only its own rows, so no tolerance applies: a mask leak,
    a TMA tail, or a slot / prefetch / schedule bug (an item depending on which CTA ran it or on
    what ran before it) shows up as a bit difference.  dQ of sequences longer than 128 is excluded:
    it is summed with fp32 atomics in no fixed order.  dqkv must also not depend on whether the
    bias gradient is accumulated."""
    lens, fixed, ms = INVARIANCE[path]
    heads, H = 12, 12 * ac.D
    g = np.random.default_rng(5)
    lens2 = [S if i in fixed else int(g.integers(0, ms + 1)) for i, S in enumerate(lens)]
    qkv, dctx, dbias0 = _inputs(lens, heads, dtype, seed=1)
    qkv2 = (torch.rand(sum(lens2), 3 * H, device="cuda") * 2e4 - 1e4).to(dtype)
    dctx2 = (torch.rand(sum(lens2), H, device="cuda") * 2e4 - 1e4).to(dtype)
    o1, o2 = np.cumsum([0] + lens), np.cumsum([0] + lens2)
    for i in fixed:
        qkv2[o2[i]:o2[i + 1]] = qkv[o1[i]:o1[i + 1]]
        dctx2[o2[i]:o2[i + 1]] = dctx[o1[i]:o1[i + 1]]
    a = _run(qkv, dctx, lens, heads, p, ms, dbias0)
    a_nobias = _run(qkv, dctx, lens, heads, p, ms, None)
    a_again = _run(qkv, dctx, lens, heads, p, ms, dbias0)
    b = _run(qkv2, dctx2, lens2, heads, p, ms, dbias0)

    def bits(dqkv):             # dQ of sequences longer than 128 zeroed
        x = dqkv.view(torch.int16).clone()
        for i, S in enumerate(lens):
            if S > 128:
                x[o1[i]:o1[i + 1], :H] = 0
        return x
    assert torch.equal(bits(a["dqkv"]), bits(a_nobias["dqkv"])), "dqkv depends on dbias"
    assert torch.equal(bits(a["dqkv"]), bits(a_again["dqkv"])), "dqkv not deterministic"
    assert torch.equal(a["ctx"].view(torch.int16), a_again["ctx"].view(torch.int16))
    assert torch.equal(a["lse"], a_again["lse"])
    for i in fixed:
        r1, r2 = slice(o1[i], o1[i + 1]), slice(o2[i], o2[i + 1])
        assert torch.equal(a["ctx"][r1].view(torch.int16), b["ctx"][r2].view(torch.int16)), ("ctx", i)
        assert torch.equal(a["lse"][:, r1], b["lse"][:, r2]), ("lse", i)
        c0 = H if lens[i] > 128 else 0
        assert torch.equal(a["dqkv"][r1, c0:].view(torch.int16), b["dqkv"][r2, c0:].view(torch.int16)), ("dqkv", i)


# ---------------------------------------------------------------- the device's dropout mask
def _read_keep_mask(lens, heads, dtype, p, stream, rng_dev=None):
    """Keep mask [b][heads, S, S] of the forward kernel: q = k = 0 gives a uniform softmax, V one-hot
    over the 64-key window w (V[key, key - 64 w] = 1) makes ctx[q, 64 h + d] non-zero iff
    key 64 w + d of row q is kept."""
    from uniter_b200 import ops
    T, H = sum(lens), heads * ac.D
    cu = ac.cu_seqlens(lens, "cuda")
    ms = max(lens)
    masks = [torch.zeros(heads, S, S, dtype=torch.bool, device="cuda") for S in lens]
    o = np.cumsum([0] + lens)
    for w in range((ms + 63) // 64):
        qkv = torch.zeros(T, 3 * H, device="cuda", dtype=dtype)
        for b, S in enumerate(lens):
            for key in range(64 * w, min(S, 64 * w + 64)):
                qkv[o[b] + key, 2 * H + (key - 64 * w)::ac.D] = 1.0
        ctx, _ = ops.attn_fwd(qkv, cu, ms, heads, dropout_p=p, rng_seed=SEED, rng_stream=stream,
                              rng_offset_dev=None if rng_dev is None else rng_dev.data_ptr())
        for b, S in enumerate(lens):
            n = min(S, 64 * w + 64) - 64 * w
            if n > 0:
                c = ctx[o[b]:o[b + 1]].view(S, heads, ac.D)[:, :, :n]
                masks[b][:, :, 64 * w:64 * w + n] = (c != 0).transpose(0, 1)
    return masks


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("path,lens", [("short", [100, 65, 128, 77, 3]), ("long", [300, 129, 512, 77])])
def test_attention_dropout_mask_equals_host_mirror(path, lens, dtype):
    """The forward's keep mask, read out of ctx, equals the host mirror bit for bit: with a host
    stream, and with a device-side stream offset (what graph replay uses), which must act as
    stream + (counter << 20).  It is deterministic, changes with the stream and keeps 1 - p."""
    heads, p = 12, 0.1
    host = _read_keep_mask(lens, heads, dtype, p, STREAM)
    want = ac.keep_masks(lens, heads, p, SEED, STREAM, "cuda")
    for b in range(len(lens)):
        assert torch.equal(host[b], want[b]), ("host stream", b)
    counter = torch.tensor([3], device="cuda", dtype=torch.int64)
    dev = _read_keep_mask(lens, heads, dtype, p, 5, rng_dev=counter)
    want_dev = ac.keep_masks(lens, heads, p, SEED, philox.stream_with_offset(5, 3), "cuda")
    for b in range(len(lens)):
        assert torch.equal(dev[b], want_dev[b]), ("device offset", b)
        assert not torch.equal(dev[b], host[b])
    again = _read_keep_mask(lens, heads, dtype, p, STREAM)
    assert all(torch.equal(x, y) for x, y in zip(host, again))
    kept = sum(int(m.sum()) for m in host) / sum(m.numel() for m in host)
    assert abs(kept - (1 - p)) < 0.005, kept


def test_attention_dropout_statistics_and_determinism():
    from uniter_b200 import ops
    torch.manual_seed(0)
    lens, heads = [64] * 16, 4
    T, H = sum(lens), 64 * heads
    qkv = torch.zeros(T, 3 * H, device="cuda").bfloat16()
    qkv[:, 2 * H:] = 1.0          # V = 1, uniform attention -> ctx = (#kept / 64) / keep
    cu = torch.arange(0, T + 1, 64, device="cuda", dtype=torch.int32)
    a, _ = ops.attn_fwd(qkv, cu, 64, heads, dropout_p=0.1, rng_seed=3, rng_stream=5)
    b, _ = ops.attn_fwd(qkv, cu, 64, heads, dropout_p=0.1, rng_seed=3, rng_stream=5)
    c, _ = ops.attn_fwd(qkv, cu, 64, heads, dropout_p=0.1, rng_seed=3, rng_stream=6)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    # every ctx element of a row is the same number; its mean over rows must be ~1
    m = a.float()[:, ::64].mean().item()
    assert abs(m - 1.0) < 0.01, m
    assert a.float().std().item() > 0.01


def test_attention_backward_with_dropout_matches_finite_masked_reference():
    """With dropout the backward must use the forward's mask: check dV against P_drop^T dO built
    from the forward output itself (V = I trick makes ctx reveal P_drop)."""
    from uniter_b200 import ops
    torch.manual_seed(1)
    S, heads = 64, 1
    H = 64
    qkv = torch.randn(S, 3 * H, device="cuda").bfloat16()
    qkv[:, 2 * H:] = torch.eye(64, device="cuda").bfloat16()      # V = I  -> ctx = P_drop
    cu = torch.tensor([0, S], device="cuda", dtype=torch.int32)
    ctx, lse = ops.attn_fwd(qkv, cu, S, heads, dropout_p=0.2, rng_seed=11, rng_stream=2)
    pdrop = ctx.float()
    dctx = torch.randn(S, H, device="cuda").bfloat16()
    dqkv = ops.attn_bwd(qkv, ctx, lse, dctx, cu, S, heads, dropout_p=0.2, rng_seed=11, rng_stream=2)
    dv_ref = pdrop.t() @ dctx.float()
    assert (dqkv[:, 2 * H:].float() - dv_ref).abs().max().item() < 0.05
