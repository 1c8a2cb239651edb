"""Reference, baseline and error checker for the varlen attention kernels (ops.attn_fwd / attn_bwd).

* `attention_reference`: per (sequence, head), in float64 (or another dtype) from the 16-bit inputs:
  ctx, lse (natural log over the valid keys, before dropout), dqkv and the accumulated QKV-bias
  gradient, with the dropout mask applied as keep * P * inv_keep.  Also `mag`, the magnitude that
  rounding errors of dqkv scale with: |dV|, and for dQ and dK the same products with the
  cancellation dS = P o (dP - delta) taken out, scale (P o M) |K| and its transpose with |Q|, where
  M = |dP| + |delta| + rowsum(|dO| o |O|).  The last term is there because a kernel forms delta
  from its rounded 16-bit output (delta = rowsum(dO o O)), so its dS carries an error of order
  u rowsum(|dO| o |O|) that does not cancel: with one key (S = 1) dQ and dK are exactly 0 in the
  reference and the baseline, and of that order in the kernel.  With `p_dtype`, also
  `colsum_p16`: the column sums of dqkv with P rounded to p_dtype, as kernel and baseline round
  it; a flat softmax makes that rounding the same for every row of a sequence, so it adds up in
  the bias gradient instead of averaging out.
* `attention_baseline`: the same in eager torch in the kernel dtype under the same mask, which is
  what the reference model computes under mixed precision (16-bit scores, softmax, dropout and
  products); lse, an fp32 output, in fp32 torch.
* `check_attention`: compares a result with the reference, using the baseline's error as the
  yardstick; returns the list of failures and per-tensor error statistics.

Pure torch, on any device: the GPU tests run it on the kernels' output, the CPU tests on a float32
stand-in and on mutations of it.
"""
import math

import numpy as np
import torch

from oracle import philox

D = 64                      # head dim
SCALE = 1.0 / math.sqrt(D)
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}   # unit roundoff of the 16-bit types
PARTS = ("dq", "dk", "dv")

SLICE_MULT = 2.0            # the bounds of check_attention
ELEM_MULT = 1.25
BIAS_MULT = 4.0
LSE_TOL = 1e-5              # lse is fp32: its atol, rtol and slice floor


def cu_seqlens(lens, device):
    return torch.tensor([0] + np.cumsum(lens).tolist(), device=device, dtype=torch.int32)


def keep_masks(lens, heads, p, seed, stream, device):
    """Per sequence, the bool keep mask [heads, S, S] of the host mirror of the kernels' dropout;
    None at p = 0."""
    if p == 0:
        return None
    hs = np.arange(heads)
    return [torch.from_numpy(philox.attn_keep(seed, stream, p, heads, b, hs, S)).to(device)
            for b, S in enumerate(lens)]


def _split(x, o, S, heads):
    """q, k, v [heads, S, D] of rows [o, o + S) of packed qkv."""
    t = x[o:o + S].view(S, 3, heads, D).permute(1, 2, 0, 3)
    return t[0], t[1], t[2]


def attention_reference(qkv, dctx, lens, heads, keep=None, inv_keep=1.0, dbias0=None, dtype=torch.float64,
                        p_dtype=None):
    """ctx [T, H], lse [heads, T], dqkv [T, 3H] and dbias [3H] = dbias0 + column sums of dqkv, all in
    `dtype`, computed per (sequence, head) from the given inputs (and mag, colsum_p16: see above)."""
    T, H3 = qkv.shape
    H = H3 // 3
    x, g = qkv.to(dtype), dctx.to(dtype)
    ctx = torch.zeros(T, H, dtype=dtype, device=qkv.device)
    lse = torch.zeros(heads, T, dtype=dtype, device=qkv.device)
    dqkv = torch.zeros(T, H3, dtype=dtype, device=qkv.device)
    mag = torch.zeros(T, H3, dtype=dtype, device=qkv.device)
    colsum_p16 = torch.zeros(H3, dtype=dtype, device=qkv.device)
    o = 0
    for b, S in enumerate(lens):
        if S == 0:
            continue
        q, k, v = _split(x, o, S, heads)
        do = g[o:o + S].view(S, heads, D).transpose(0, 1)
        s = q @ k.transpose(-1, -2) * SCALE
        l = torch.logsumexp(s, -1)
        P = torch.exp(s - l[..., None])
        m = keep[b].to(dtype) * inv_keep if keep is not None else 1.0
        dP = (do @ v.transpose(-1, -2)) * m

        def grads(P):
            Pd = P * m
            delta = (dP * P).sum(-1, keepdim=True)
            dS = P * (dP - delta)
            d = torch.stack([dS @ k * SCALE, dS.transpose(-1, -2) @ q * SCALE, Pd.transpose(-1, -2) @ do])
            return Pd @ v, delta, d.permute(2, 0, 1, 3).reshape(S, H3)
        out, delta, dqkv[o:o + S] = grads(P)
        ctx[o:o + S] = out.transpose(0, 1).reshape(S, H)
        lse[:, o:o + S] = l
        A = P * (dP.abs() + delta.abs() + (do.abs() * out.abs()).sum(-1, keepdim=True))
        d = torch.stack([A @ k.abs() * SCALE, A.transpose(-1, -2) @ q.abs() * SCALE])
        mag[o:o + S, :2 * H] = d.permute(2, 0, 1, 3).reshape(S, 2 * H)
        mag[o:o + S, 2 * H:] = dqkv[o:o + S, 2 * H:].abs()
        if p_dtype is not None:
            colsum_p16 += grads(P.to(p_dtype).to(dtype))[2].sum(0)
        o += S
    dbias = dqkv.sum(0)
    if dbias0 is not None:
        dbias = dbias + dbias0.to(dtype)
    return dict(ctx=ctx, lse=lse, dqkv=dqkv, dbias=dbias, mag=mag, colsum_p16=colsum_p16 if p_dtype else None)


def attention_baseline(qkv, dctx, lens, heads, keep=None, inv_keep=1.0):
    """ctx, lse, dqkv of eager torch: scores, softmax, dropout and both products in qkv.dtype, the
    backward by autograd through them; lse in fp32 from the 16-bit inputs."""
    T, H3 = qkv.shape
    H = H3 // 3
    x = qkv.detach().clone().requires_grad_(True)
    outs, lses = [], []
    o = 0
    for b, S in enumerate(lens):
        if S == 0:
            continue
        q, k, v = _split(x, o, S, heads)
        P = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(D), -1)
        if keep is not None:
            P = (P.float() * (keep[b].float() * inv_keep)).to(qkv.dtype)
        outs.append((P @ v).transpose(0, 1).reshape(S, H))
        qf, kf, _ = _split(qkv.detach().float(), o, S, heads)
        lses.append(torch.logsumexp(qf @ kf.transpose(-1, -2) * SCALE, -1))
        o += S
    ctx = torch.cat(outs, 0)
    ctx.backward(dctx)
    return dict(ctx=ctx.detach(), lse=torch.cat(lses, 1), dqkv=x.grad)


def _views(r, heads):
    """(name, [T, heads, n] view) of every checked tensor of a result dict."""
    T = r["ctx"].shape[0]
    H = heads * D
    out = [("ctx", r["ctx"].view(T, heads, D)), ("lse", r["lse"].t().reshape(T, heads, 1))]
    for i, name in enumerate(PARTS):
        out.append((name, r["dqkv"][:, i * H:(i + 1) * H].reshape(T, heads, D)))
    return out


def check_attention(out, ref, base, lens, heads, dtype, dbias0=None):
    """Failures (list of strings; empty = pass) and error statistics of result `out` (dict with ctx,
    lse, dqkv and, optionally, dbias) against `ref` (attention_reference), with `base`
    (attention_baseline) as the yardstick.  NaN anywhere in `out` fails.

    With m = |ref| (ctx, lse) or ref["mag"] (dQ, dK, dV), per tensor:
      elementwise          |err| <= max(atol + rtol m, ELEM_MULT x the baseline's max |err|)
      per (seq, head)      ||err|| <= SLICE_MULT ||baseline err|| + u ||m|| + atol sqrt(n)
      bias gradient        |err| <= BIAS_MULT u sqrt(sum_rows m^2) + ELEM_MULT e_sys + floor
    per column, e_sys being the larger error of the baseline's column sums and of colsum_p16."""
    u = UNIT[dtype]
    dev = ref["ctx"].device
    seq = torch.repeat_interleave(torch.arange(len(lens), device=dev),
                                  torch.tensor(lens, device=dev))
    ok_b = torch.tensor(lens, device=dev) > 0
    B = len(lens)
    fails, stats = [], {}
    rv, bv = dict(_views(ref, heads)), dict(_views(base, heads))
    mv = dict(_views(dict(ref, dqkv=ref["mag"]), heads))
    dqkv_scale = ref["dqkv"].abs().max().item()
    for name, kv in _views(out, heads):
        r = rv[name].double()
        k = kv.to(dev).double()
        bs = bv[name].double()
        if name == "lse":
            atol, rtol, floor_rel = LSE_TOL, LSE_TOL, LSE_TOL
            m = r.abs()
        else:
            scale = dqkv_scale if name in PARTS else r.abs().max().item()
            atol, rtol, floor_rel = 0.01 * u * scale, 2 * u, u
            m = mv[name].double() if name in PARTS else r.abs()
        e, eb = (k - r).abs(), (bs - r).abs()
        bound = torch.clamp(atol + rtol * m, min=ELEM_MULT * eb.max().item())
        bad = ~(e <= bound)
        if bad.any():
            t, h, c = [int(i) for i in bad.nonzero()[0]]
            fails.append("%s: %d elements out of bounds, first (row %d, head %d, col %d): got %r, ref %r, "
                         "bound %.3e" % (name, int(bad.sum()), t, h, c, k[t, h, c].item(), r[t, h, c].item(),
                                         bound[t, h, c].item()))

        # normwise error of every (sequence, head) slice
        def seg(x):
            return torch.zeros(B, heads, dtype=torch.float64, device=dev).index_add_(0, seq, (x ** 2).sum(-1)).sqrt()
        en, ebn, rn = seg(k - r), seg(bs - r), seg(r)
        n = torch.tensor(lens, device=dev, dtype=torch.float64)[:, None] * r.shape[-1]
        lim = SLICE_MULT * ebn + floor_rel * seg(m) + atol * n.sqrt()
        bad = ~(en <= lim) & ok_b[:, None]
        if bad.any():
            b, h = [int(i) for i in bad.nonzero()[0]]
            fails.append("%s: %d (sequence, head) slices out of bounds, first (seq %d, head %d): |err| %.3e > "
                         "%.3e (baseline %.3e, |ref| %.3e)" % (name, int(bad.sum()), b, h, en[b, h].item(),
                                                                lim[b, h].item(), ebn[b, h].item(), rn[b, h].item()))
        stats[name] = dict(max_err=e.max().item(), base_max_err=eb.max().item(),
                           rel_err=((k - r).norm() / r.norm().clamp(min=1e-300)).item(),
                           base_rel_err=((bs - r).norm() / r.norm().clamp(min=1e-300)).item(),
                           worst_slice_ratio=(en / lim.clamp(min=1e-300))[ok_b].max().item())
    if "dbias" in out and out["dbias"] is not None:
        # one missing or doubled item changes a column by its sum over about S rows, ~sqrt(S) times a
        # row's magnitude; the random part of the bound grows only like sqrt(T)
        r = ref["dbias"].double()
        k = out["dbias"].to(dev).double()
        cs = ref["dqkv"].double().sum(0)
        eb = (base["dqkv"].double().sum(0) - cs).abs()
        if ref.get("colsum_p16") is not None:
            eb = torch.maximum(eb, (ref["colsum_p16"].double() - cs).abs())
        lim = (BIAS_MULT * u * ref["mag"].double().pow(2).sum(0).sqrt() + ELEM_MULT * eb
               + 0.01 * u * dqkv_scale * math.sqrt(sum(lens)))
        if dbias0 is not None:
            lim = lim + 1e-6 * dbias0.to(dev).double().abs()
        e = (k - r).abs()
        H = heads * D
        bad = ~(e <= lim)
        if bad.any():
            heads_bad = sorted({(int(c) % H) // D for c in bad.nonzero()[:, 0]})
            c = int(bad.nonzero()[0])
            fails.append("dbias: %d columns out of bounds (heads %s), first col %d: got %r, ref %r, bound %.3e"
                         % (int(bad.sum()), heads_bad, c, k[c].item(), r[c].item(), lim[c].item()))
        stats["dbias"] = dict(max_err=e.max().item(), base_max_err=eb.max().item(),
                              worst_ratio=(e / lim).max().item())
    return fails, stats


def format_stats(stats):
    parts = []
    for name, s in stats.items():
        if name == "dbias":
            parts.append("dbias max %.2e/base %.2e (%.2f of bound)" % (s["max_err"], s["base_max_err"],
                                                                       s["worst_ratio"]))
        else:
            parts.append("%s max %.2e/base %.2e rel %.2e/base %.2e slice %.2f of bound"
                         % (name, s["max_err"], s["base_max_err"], s["rel_err"], s["base_rel_err"],
                            s["worst_slice_ratio"]))
    return "; ".join(parts)
