"""Reference, baseline and error checker for the word-region alignment kernels (ops.wra_fwd / wra_bwd,
csrc/heads.cu).

* `reference`: float64 from the same 16-bit packed rows: normalised rows, the cosine cost, 50 IPOT
  iterations (beta 0.5, k = 1), dist = sum C * T^T, and the backward with T held constant
  (dC = g T^T, then the F.normalize backward), with the sums of absolute terms that bound the errors.
* `baseline`: the fp32 torch composition of model/ot.py's math on the padded [B, M, H] / [B, N, H]
  tensors with bool masks (the reference's own code, written out again), and its autograd backward.
* `check`: dist representable in the 16-bit type and within max(1 ulp, 1.25 x the baseline's error) of
  the float64 value; d_packed elementwise within max(C u sum|terms|, 1.25 x the baseline's error), and
  exactly zero on every row no pair owns.

Pure torch: the GPU tests run it on the kernels' outputs, the CPU tests on a float32 stand-in and on
mutations of it.
"""
import torch

UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
C_TERMS = 4.0
BASE_MULT = 1.25
BETA, ITERS, EPS = 0.5, 50, 1e-5


def pairs(cu, txt_lens):
    """(start, m, n) of every pair."""
    cu = [int(v) for v in cu]
    return [(cu[b], int(m), cu[b + 1] - cu[b] - int(m)) for b, m in enumerate(txt_lens)]


def ipot(C, iters=ITERS, beta=BETA):
    """IPOT over one pair's [m, n] cost; returns T [n, m]."""
    m, n = C.shape
    sigma = torch.full((m,), 1.0 / m, dtype=C.dtype)
    T = torch.ones(n, m, dtype=C.dtype)
    A = torch.exp(-C.t() / beta)
    for _ in range(iters):
        Q = A * T
        delta = 1.0 / (n * (Q @ sigma))
        sigma = 1.0 / (m * (delta @ Q))
        T = delta[:, None] * Q * sigma[None, :]
    return T


def reference(packed, cu, txt_lens, g=None):
    """float64 dist [B], d_packed [T, H] for upstream gradients g [B] (default ones), and bounds."""
    dt = torch.float64
    rows = packed.detach().cpu().to(dt)
    B = len(txt_lens)
    g = torch.ones(B, dtype=dt) if g is None else g.detach().cpu().to(dt)
    dist = torch.zeros(B, dtype=dt)
    dist_abs = torch.zeros(B, dtype=dt)
    d = torch.zeros_like(rows)
    d_abs = torch.zeros_like(rows)
    for b, (s, m, n) in enumerate(pairs(cu, txt_lens)):
        x = rows[s:s + m].clone().requires_grad_(True)
        y = rows[s + m:s + m + n].clone().requires_grad_(True)
        sx = x.norm(dim=1, keepdim=True).clamp_min(EPS)
        sy = y.norm(dim=1, keepdim=True).clamp_min(EPS)
        xh, yh = x / sx, y / sy
        C = 1 - xh @ yh.t()
        T = ipot(C.detach())
        db = (C * T.t()).sum()
        db.backward(g[b])
        dist[b] = db.detach()
        dist_abs[b] = (C.detach().abs() * T.t()).sum()
        d[s:s + m], d[s + m:s + m + n] = x.grad, y.grad
        # |terms| of dx^ = -g T^T y^ and the normalize backward dx = dx^/s - (dx^ . x) x / s^3
        with torch.no_grad():
            gx = (g[b].abs() * T.t()) @ yh.abs()
            gy = (g[b].abs() * T) @ xh.abs()
            for lo, r, gr, sr in ((s, x, gx, sx), (s + m, y, gy, sy)):
                d_abs[lo:lo + r.size(0)] = gr / sr + (gr * r.abs()).sum(1, keepdim=True) * r.abs() / sr ** 3
    return {"dist": dist, "dist_abs": dist_abs, "d_packed": d, "d_abs": d_abs}


def baseline(packed, cu, txt_lens, g=None):
    """The fp32 composition on padded tensors with bool masks, as model/pretrain.py:166-193 runs it (the
    scatter into text / image slots written as the packed row split); dist in packed.dtype, d_packed by
    autograd."""
    dev = packed.device
    P = packed.detach().clone().requires_grad_(True)
    geo = pairs(cu, txt_lens)
    B, H = len(geo), packed.size(1)
    M, N = max(m for _, m, _ in geo), max(n for _, _, n in geo)
    zero = P.new_zeros(1, H)
    src = torch.cat([P, zero])
    ti = torch.full((B, M), P.size(0), dtype=torch.long, device=dev)
    ii = torch.full((B, N), P.size(0), dtype=torch.long, device=dev)
    for b, (s, m, n) in enumerate(geo):
        ti[b, :m] = torch.arange(s, s + m, device=dev)
        ii[b, :n] = torch.arange(s + m, s + m + n, device=dev)
    txt, img = src[ti].float(), src[ii].float()
    txt_pad, img_pad = ti == P.size(0), ii == P.size(0)
    cost = 1 - torch.nn.functional.normalize(txt, dim=-1, eps=EPS) @ \
        torch.nn.functional.normalize(img, dim=-1, eps=EPS).transpose(1, 2)
    joint = txt_pad[:, :, None] | img_pad[:, None, :]
    cost = cost.masked_fill(joint, 0)
    tl = (M - txt_pad.sum(1)).float()
    il = (N - img_pad.sum(1)).float()
    with torch.no_grad():
        C = cost.detach()
        sigma = (torch.ones(B, M, device=dev) / tl[:, None]).masked_fill(txt_pad, 0)
        jt = joint.transpose(1, 2)
        T = torch.ones(B, N, M, device=dev).masked_fill(jt, 0)
        A = torch.exp(-C.transpose(1, 2) / BETA).masked_fill(jt, 0)
        xm, ym = (txt_pad.float() * 1e4)[:, None], (img_pad.float() * 1e4)[:, None]
        for _ in range(ITERS):
            Q = A * T
            delta = 1 / (il[:, None, None] * Q.matmul(sigma.view(B, M, 1)).view(B, 1, N) + ym)
            sigma = 1 / (tl[:, None, None] * delta.matmul(Q) + xm)
            T = delta.view(B, N, 1) * Q * sigma
        T = T.masked_fill(jt, 0)
    dist = torch.diagonal(cost.matmul(T), dim1=1, dim2=2).sum(-1).to(packed.dtype)
    gg = torch.ones(B, device=dev, dtype=dist.dtype) if g is None else g.to(dev, dist.dtype)
    dist.backward(gg)
    return {"dist": dist.detach(), "d_packed": P.grad}


def _ulp(x, dtype):
    """Spacing of the 16-bit type at |x| (float64)."""
    u = UNIT[dtype] * 2.0
    e = torch.floor(torch.log2(x.abs().clamp_min(torch.finfo(dtype).tiny)))
    return torch.pow(torch.tensor(2.0, dtype=torch.float64), e) * u


def check(out, ref, dtype, base=None):
    """Assert `out` (dist [B], d_packed [T, H]) agrees with `ref`.  Returns nothing."""
    u = UNIT[dtype]
    msg = []
    dist = out["dist"].detach().cpu().to(torch.float64)
    if not torch.equal(dist, dist.to(dtype).to(torch.float64)):
        msg.append("dist: not rounded to %s" % dtype)
    want = ref["dist"]
    bound = _ulp(want.to(dtype).to(torch.float64), dtype)
    if base is not None:
        bound = torch.maximum(bound, BASE_MULT * (base["dist"].cpu().to(torch.float64) - want).abs())
    bad = (dist - want).abs() > bound
    if bad.any():
        i = int(bad.nonzero()[0])
        msg.append("dist: %d pairs off, first %d: got %.8g want %.8g bound %.3g"
                   % (int(bad.sum()), i, float(dist[i]), float(want[i]), float(bound[i])))
    if "d_packed" in out:
        d = out["d_packed"].detach().cpu().to(torch.float64)
        zero = ref["d_abs"] == 0
        if (d[zero] != 0).any():
            msg.append("d_packed: %d elements outside every pair are not zero" % int((d[zero] != 0).sum()))
        bound = C_TERMS * u * ref["d_abs"]
        if base is not None:
            bound = torch.maximum(bound, BASE_MULT * (base["d_packed"].cpu().to(torch.float64) - ref["d_packed"]).abs())
        bad = (d - ref["d_packed"]).abs() > bound
        if bad.any():
            i = int(bad.reshape(-1).nonzero()[0])
            msg.append("d_packed: %d elements outside the bound, first flat %d: got %.6g want %.6g bound %.3g"
                       % (int(bad.sum()), i, float(d.reshape(-1)[i]), float(ref["d_packed"].reshape(-1)[i]),
                          float(bound.reshape(-1)[i])))
    assert not msg, "; ".join(msg)
