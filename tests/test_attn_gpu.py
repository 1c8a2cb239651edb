"""GPU: fused varlen attention (wgmma) vs torch fp32 reference of model/layer.py:80-100."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(qkv, lens, heads):
    """fp32 per-sequence attention with autograd (inputs already rounded to 16 bit)."""
    T, H3 = qkv.shape
    H = H3 // 3
    d = H // heads
    outs = []
    o = 0
    for S in lens:
        blk = qkv[o:o + S]
        q = blk[:, :H].view(S, heads, d).transpose(0, 1)
        k = blk[:, H:2 * H].view(S, heads, d).transpose(0, 1)
        v = blk[:, 2 * H:].view(S, heads, d).transpose(0, 1)
        p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(d), -1)
        outs.append((p @ v).transpose(0, 1).reshape(S, H))
        o += S
    return torch.cat(outs, 0)


CASES = [
    [56, 56], [56, 44], [1], [7, 128, 64, 1, 33], [129], [300, 5, 17], [512, 256],
    [74, 38, 61, 50, 45, 66, 53, 70],
]


@pytest.mark.parametrize("dtype,tol", [(torch.bfloat16, 2e-2), (torch.float16, 4e-3)])
@pytest.mark.parametrize("lens", CASES)
@pytest.mark.parametrize("heads", [2, 12])
def test_attention_fwd_bwd(dtype, tol, lens, heads):
    from uniter_b200 import ops
    torch.manual_seed(sum(lens) + heads)
    T, H = sum(lens), 64 * heads
    qkv = torch.randn(T, 3 * H, device="cuda").to(dtype)
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device="cuda", dtype=torch.int32)
    ctx, lse = ops.attn_fwd(qkv, cu, max(lens), heads)
    q32 = qkv.float().requires_grad_(True)
    ref = _ref(q32, lens, heads)
    err = (ctx.float() - ref).abs().max().item()
    assert err <= tol * max(1.0, ref.abs().max().item()), "fwd err %.3e" % err
    dctx = torch.randn(T, H, device="cuda").to(dtype)
    ref.backward(dctx.float())
    dbias = torch.full((3 * H,), 0.5, device="cuda")       # accumulated into: starts non-zero
    dqkv = ops.attn_bwd(qkv, ctx, lse, dctx, cu, max(lens), heads, dbias=dbias)
    gref = q32.grad
    # fused QKV bias gradient = column sums of dqkv over the valid rows only
    bref = gref.sum(0) + 0.5
    eb = (dbias - bref).abs().max().item()
    assert eb <= 2 * tol * max(1.0, gref.abs().sum(0).max().item()), "dbias err %.3e (lens=%s)" % (eb, lens)
    for name, sl in (("dq", slice(0, H)), ("dk", slice(H, 2 * H)), ("dv", slice(2 * H, 3 * H))):
        e = (dqkv[:, sl].float() - gref[:, sl]).abs().max().item()
        lim = 2 * tol * max(1.0, gref[:, sl].abs().max().item())
        assert e <= lim, "%s err %.3e > %.3e (lens=%s)" % (name, e, lim, lens)


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
