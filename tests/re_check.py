"""Reference, baseline and error checker for the referring-expression head kernels
(ops.region_score_fwd / region_score_bwd, csrc/heads.cu).

* `reference`: float64 from the same 16-bit inputs.  Scores are the float64 dot products plus bias (to
  be rounded once to the 16-bit type); the losses, the chosen negatives and every gradient are computed
  in float64 from the scores the kernel stored, which are part of the head's contract (re_output's
  16-bit output, model/re.py:69-70).
* `baseline`: the eager 16-bit torch composition the fused head replaces (Linear with N = 1 over the
  zero-padded region rows, masked_fill, cross-entropy or the sigmoid hinge; its autograd backward).
* `check`: scores within 1 ulp of the rounded float64 value (masked positions exactly round16(-1e4)),
  the chosen negatives exactly, padding and masked rows of d_rows exactly zero, and loss / d_rows /
  dweight / dbias elementwise within max(C u sum|terms|, 1.25 x the baseline's error).

Pure torch: the GPU tests run it on the kernels' outputs, the CPU tests on a float32 stand-in and on
mutations of it.
"""
import torch
import torch.nn.functional as F

UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
C_TERMS = 4.0
BASE_MULT = 1.25
CLS, RANK = 1, 2


def round16(x, dtype):
    return x.to(dtype).to(torch.float64)


def padded(rows, seg, S):
    """[B, S, H] float64 of the segment rows, zeros past each segment (model/re.py:129-157)."""
    B = seg.size(1)
    out = torch.zeros(B, S, rows.size(1), dtype=torch.float64, device=rows.device)
    for b in range(B):
        s, n = int(seg[0, b]), int(seg[1, b])
        out[b, :n] = rows[s:s + n].to(torch.float64)
    return out


def live_mask(seg, obj_masks):
    B, S = obj_masks.shape
    k = torch.arange(S, device=obj_masks.device)[None, :]
    return (k < seg[1].to(obj_masks.device).long()[:, None]) & (obj_masks == 0)


def hard_negative(scores, live, t, n_len):
    """Best region != t among the live ones, ties to the lowest index; if none is live, the lowest
    other index."""
    best, arg = None, -1
    for k in range(n_len):
        if k == t or not live[k]:
            continue
        if best is None or scores[k] > best:
            best, arg = scores[k], k
    if arg < 0:
        others = [k for k in range(n_len) if k != t]
        arg = others[0] if others else -1
    return arg


def reference(rows, w, b, seg, obj_masks, scores16, targets=None, plan=None, mode=0, margin=0.0, dloss=None):
    """float64 reference; `scores16` are the kernel's stored scores (for the loss and gradients)."""
    dt = torch.float64
    B, S = obj_masks.shape
    dev = rows.device
    hid = padded(rows, seg, S)
    live = live_mask(seg, obj_masks)
    w64 = w.reshape(-1).to(dt)
    b64 = b.reshape(-1).to(dt)[0] if b is not None else 0.0
    exact = hid @ w64 + b64                                     # [B, S], before rounding / masking
    out = {"exact": exact, "live": live}
    if mode == 0:
        return out
    s = scores16.to(dt)
    t = targets.reshape(-1).long().to(dev)
    loss = torch.zeros(B, dtype=dt, device=dev)
    loss_abs = torch.zeros(B, dtype=dt, device=dev)
    ds = torch.zeros(B, S, dtype=dt, device=dev)
    neg = torch.full((B,), -1, dtype=torch.long, device=dev)
    g = dloss.to(dt) if dloss is not None else torch.ones(B, dtype=dt, device=dev)
    for i in range(B):
        ti, ni = int(t[i]), int(seg[1, i])
        if mode == CLS:
            lse = torch.logsumexp(s[i], 0)
            loss[i] = lse - s[i, ti]
            loss_abs[i] = lse.abs() + s[i, ti].abs()
            p = torch.softmax(s[i], 0)
            p[ti] -= 1.0
            ds[i] = torch.where(live[i], p * g[i], torch.zeros_like(p))
        else:
            pi = int(plan[i])
            if pi >= 0:
                n = pi if pi < ni and pi != ti else -1
            else:
                n = hard_negative(s[i].tolist(), live[i].tolist(), ti, ni)
            neg[i] = n
            if n < 0:
                continue
            sn, sp = torch.sigmoid(s[i, n]), torch.sigmoid(s[i, ti])
            h = margin + sn - sp
            loss[i] = h.clamp(min=0)
            loss_abs[i] = abs(margin) + sn + sp
            if h >= 0:
                if live[i, n]:
                    ds[i, n] = sn * (1 - sn) * g[i]
                if live[i, ti]:
                    ds[i, ti] = -sp * (1 - sp) * g[i]
    d_rows = torch.zeros(rows.shape, dtype=dt, device=dev)
    d_abs = torch.zeros(rows.shape, dtype=dt, device=dev)
    for i in range(B):
        st, ni = int(seg[0, i]), int(seg[1, i])
        d_rows[st:st + ni] = ds[i, :ni, None] * w64[None, :]
        d_abs[st:st + ni] = d_rows[st:st + ni].abs()
    out.update(loss=loss, loss_abs=loss_abs, neg=neg, dscore=ds, d_rows=d_rows, d_rows_abs=d_abs,
               dw=(ds[:, :, None] * hid).sum((0, 1)), dw_abs=(ds[:, :, None] * hid).abs().sum((0, 1)),
               db=ds.sum().reshape(1), db_abs=ds.abs().sum().reshape(1))
    return out


def baseline(rows, w, b, seg, obj_masks, targets, neg, mode, margin, dloss):
    """The eager composition in rows.dtype: loss, d_rows, dw, db (autograd)."""
    B, S = obj_masks.shape
    dtype = rows.dtype
    r = rows.detach().clone().requires_grad_(True)
    w16 = w.detach().reshape(1, -1).clone().requires_grad_(True)
    b16 = b.detach().reshape(1).clone().requires_grad_(True)
    idx = torch.full((B, S), rows.size(0), dtype=torch.long, device=rows.device)
    for i in range(B):
        st, ni = int(seg[0, i]), int(seg[1, i])
        idx[i, :ni] = torch.arange(st, st + ni, device=rows.device)
    hid = torch.cat([r, r.new_zeros(1, r.size(1))])[idx]
    scores = F.linear(hid, w16, b16).squeeze(2).masked_fill(obj_masks.bool(), -1e4)
    t = targets.reshape(-1).long()
    if mode == CLS:
        loss = F.cross_entropy(scores, t, reduction="none")
    else:
        pos = torch.sigmoid(scores.gather(1, t.view(B, 1))).view(-1)
        ng = torch.sigmoid(scores.gather(1, neg.long().view(B, 1))).view(-1)
        loss = torch.clamp(margin + ng - pos, 0)
    loss.backward(dloss.to(loss.dtype))
    return {"loss": loss.detach(), "d_rows": r.grad, "dw": w16.grad.reshape(-1), "db": b16.grad.reshape(1)}


def _ulp_distance(a, b, dtype):
    ia = a.to(dtype).view(torch.int16).to(torch.int32)
    ib = b.to(dtype).view(torch.int16).to(torch.int32)
    # sign-magnitude -> ordered integers
    ia = torch.where(ia < 0, -(ia & 0x7FFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFF), ib)
    return (ia - ib).abs()


def _within(name, got, ref, absterms, base, u, msg):
    got = got.to(torch.float64).reshape(ref.shape)
    err = (got - ref).abs()
    bound = C_TERMS * u * absterms
    if base is not None:
        bound = torch.maximum(bound, BASE_MULT * (base.to(torch.float64).reshape(ref.shape) - ref).abs())
    bad = err > bound
    if bad.any():
        i = int(bad.reshape(-1).nonzero()[0])
        msg.append("%s: %d elements outside the bound, first flat %d: got %.6g want %.6g bound %.3g"
                   % (name, int(bad.sum()), i, float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]),
                      float(bound.reshape(-1)[i])))


def check(out, ref, dtype, base=None, seg=None):
    """Assert `out` (scores [, loss, neg, d_rows, dw, db]) agrees with `ref`.  Returns nothing."""
    u = UNIT[dtype]
    msg = []
    scores = out["scores"].to(torch.float64)
    live = ref["live"]
    want = torch.where(live, round16(ref["exact"], dtype), torch.full_like(ref["exact"], float(torch.tensor(-1e4).to(dtype))))
    ulps = _ulp_distance(scores, want, dtype)
    if (ulps[live] > 1).any():
        msg.append("scores: %d live positions more than 1 ulp off" % int((ulps[live] > 1).sum()))
    if (scores[~live] != want[~live]).any():
        msg.append("scores: %d masked positions are not round16(-1e4)" % int((scores[~live] != want[~live]).sum()))
    if "loss" in out and out["loss"] is not None:
        _within("loss", out["loss"], ref["loss"], ref["loss_abs"], None if base is None else base["loss"], u, msg)
        if out.get("neg") is not None and not torch.equal(out["neg"].long().cpu(), ref["neg"].cpu()):
            msg.append("neg: %s != %s" % (out["neg"].tolist(), ref["neg"].tolist()))
    if "d_rows" in out:
        d = out["d_rows"].to(torch.float64)
        zero = ref["d_rows_abs"] == 0
        if (d[zero] != 0).any():
            msg.append("d_rows: %d elements of padding / masked rows are not zero" % int((d[zero] != 0).sum()))
        for k in ("d_rows", "dw", "db"):
            _within(k, out[k], ref[k], ref[k + "_abs"], None if base is None else base[k], u, msg)
    assert not msg, "; ".join(msg)
