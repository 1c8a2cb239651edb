"""Reference, baseline and error checker for the row-wise kernels: the LayerNorm forward and backward
(ops.layernorm_fwd / layernorm_bwd, csrc/rowops.cu) and the embedding rows (ub200_embed_rows_fwd,
csrc/embed.cu), with their dropout masks replayed on the host.

* `keep_mask`: the keep mask of a row-wise dropout site; element (row, col) draws
  philox.rand16 at index row * ncols + col.
* References, in float64 (or another dtype) from the same 16-bit inputs:
  `ln_fwd_reference`; `ln_bwd_reference`: dx, dx_drop = dx o keep * inv_keep (dropout on dx, the
  Linear branch of a post-LN residual block), dgamma, dbeta and dbias = the column sums of the
  16-bit-rounded Linear-branch gradient, with an optional row kind (inactive rows keep `dx0`) and the
  dropout on dy instead (y = dropout(LN(x)), the embeddings); `embed_rows_reference`: x, u (the sum
  before the last LayerNorm) and ppre (the pos_linear output) of packed embedding rows through
  oracle/encoder_oracle.py's text_embeddings / image_embeddings.
* Baselines: the same in eager torch in the kernel dtype, which is what the reference model computes
  under apex O2 (16-bit tensors, LayerNorm with fp32 statistics): `ln_fwd_baseline`,
  `ln_bwd_baseline`, and `embed_rows_reference(..., dtype=<16-bit>)`.
* `check_rows` / `check_sums` / `check_exact`: compare a result with the reference (see each).

Pure torch, on any device: the GPU tests run it on the kernels' output, the CPU tests on a float32
stand-in and on mutations of it.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import encoder_oracle as orc
from oracle import philox

EPS = 1e-12
UNIT = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}   # unit roundoff of the 16-bit types

ELEM_MULT = 1.25            # the bounds of check_rows
ROW_MULT = 2.0
RTOL_U = 2.0                # rtol = RTOL_U u
ATOL_U = 0.01               # atol = ATOL_U u max|ref|
SUM_TOL = 1e-5              # fp32 column sums: |err| <= SUM_TOL sum |terms|


def keep_mask(seed, stream, p, rows, ncols, device="cpu", counter=None):
    """(bool keep mask [rows, ncols], inv_keep) of a row-wise dropout site at drop probability p > 0;
    `counter`: the device-side stream offset the kernel was also given."""
    thr, inv_keep = philox.dropout_params(p)
    e = np.arange(rows * ncols, dtype=np.uint64)
    r = philox.rand16(seed, philox.stream_with_offset(stream, counter), e)
    return torch.from_numpy((r >= thr).reshape(rows, ncols)).to(device), inv_keep


# ----------------------------------------------------------------------------- LayerNorm
def ln_fwd_reference(x, gamma, beta, dtype=torch.float64):
    return orc.layer_norm(x.to(dtype), gamma.to(dtype), beta.to(dtype), EPS)


def ln_fwd_baseline(x, gamma, beta):
    return F.layer_norm(x, (x.size(-1),), gamma, beta, EPS)


def _active(rows, row_kind, kind, device):
    if row_kind is None:
        return torch.ones(rows, dtype=torch.bool, device=device)
    return row_kind.to(device) == kind


def ln_bwd_reference(dy, x, gamma, keep=None, inv_keep=1.0, on_dy=False, row_kind=None, kind=0, dx0=None,
                     dgamma0=None, dbeta0=None, dbias0=None, dtype=torch.float64):
    """dx, dx_drop (None without a mask or with on_dy), dgamma, dbeta, dbias in `dtype`, plus
    `absg` / `absb` / `absd`, the sums of |terms| of dgamma / dbeta / dbias (initial values excluded).
    Rows whose row_kind differs from `kind` take no part; their dx is dx0 (zeros if None).  dbias is
    dbias0 + the column sums of the Linear-branch gradient (dx_drop, else dx) rounded to dy.dtype."""
    rows, H = x.shape
    dev = x.device
    act = _active(rows, row_kind, kind, dev)[:, None]
    xd, g = x.to(dtype), gamma.to(dtype)
    d = dy.to(dtype)
    if keep is not None and on_dy:
        d = d * keep.to(dtype) * inv_keep
    mu = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xd - mu) ** 2).mean(-1, keepdim=True) + EPS)
    xh = (xd - mu) * rstd
    gd = d * g
    dx = rstd * (gd - gd.mean(-1, keepdim=True) - xh * (gd * xh).mean(-1, keepdim=True))
    base = torch.zeros_like(dx) if dx0 is None else dx0.to(dtype)
    dx = torch.where(act, dx, base)
    dx_drop = dx * keep.to(dtype) * inv_keep if (keep is not None and not on_dy) else None
    lin = (dx_drop if dx_drop is not None else dx).to(dy.dtype).to(dtype) * act
    terms_g, terms_b = d * xh * act, d * act

    def acc(init, t):
        return t.sum(0) + (init.to(dtype) if init is not None else 0)
    return dict(dx=dx, dx_drop=dx_drop, dgamma=acc(dgamma0, terms_g), dbeta=acc(dbeta0, terms_b),
                dbias=acc(dbias0, lin), absg=terms_g.abs().sum(0), absb=terms_b.abs().sum(0),
                absd=lin.abs().sum(0), active=act[:, 0])


def ln_bwd_baseline(dy, x, gamma, keep=None, inv_keep=1.0, on_dy=False):
    """dx, dx_drop of eager torch in the kernel dtype: autograd through F.layer_norm (and the dropout
    after it with on_dy); dx_drop = torch's dropout backward of the 16-bit dx."""
    xg = x.detach().clone().requires_grad_(True)
    y = F.layer_norm(xg, (x.size(-1),), gamma, None, EPS)
    if keep is not None and on_dy:
        y = orc.dropout(y, keep, inv_keep)
    y.backward(dy)
    dx = xg.grad
    dx_drop = orc.dropout(dx, keep, inv_keep) if (keep is not None and not on_dy) else None
    return dict(dx=dx, dx_drop=dx_drop)


# ----------------------------------------------------------------------------- embedding rows
def embed_rows_reference(state, rows, G, box, keep=None, inv_keep=1.0, dtype=torch.float64):
    """x, u, ppre [T, H] in `dtype` of the packed embedding rows that ub200_embed_rows_fwd computes.

    state: the front-end parameters keyed like UniterModel.state_dict(); rows: dict of int tensors
    kind, word_id, pos_id, type_id, img_src [T]; G [T, H]: the img_linear output of each row (the
    kernel's input); box [n, 7]: region boxes as the kernel reads them (rounded to the model dtype).
    Image rows go through image_embeddings with an identity img_linear, so that they start from G."""
    T, H = G.shape
    dev = G.device
    st = {k: v.to(dev, dtype) for k, v in state.items()}
    st["img_embeddings.img_linear.weight"] = torch.eye(H, device=dev, dtype=dtype)
    st["img_embeddings.img_linear.bias"] = torch.zeros(H, device=dev, dtype=dtype)
    out = {k: torch.zeros(T, H, device=dev, dtype=dtype) for k in ("x", "u", "ppre")}
    kind = rows["kind"].to(dev)
    for k in (0, 1):
        sel = (kind == k).nonzero()[:, 0]
        if sel.numel() == 0:
            continue
        taps = {}
        kp = keep[sel][None] if keep is not None else None
        ty = rows["type_id"].to(dev)[sel][None].long()
        if k == 0:
            x = orc.text_embeddings(st, rows["word_id"].to(dev)[sel][None].long(),
                                    rows["pos_id"].to(dev)[sel][None].long(), ty, keep=kp,
                                    inv_keep=inv_keep, taps=taps)
        else:
            b = box.to(dev, dtype)[rows["img_src"].to(dev)[sel].long()][None]
            x = orc.image_embeddings(st, G.to(dtype)[sel][None], b, ty, keep=kp, inv_keep=inv_keep, taps=taps)
            out["ppre"][sel] = taps["ppre"][0]
        out["x"][sel] = x[0]
        out["u"][sel] = taps["u"][0]
    return out


# ----------------------------------------------------------------------------- checks
def check_rows(name, out, ref, base, dtype, rows=None, mag=None):
    """Failures (list of strings) and statistics of a 16-bit result `out` [n, H] against `ref`, with
    `base` (baseline) as the yardstick, over the rows selected by `rows` (bool [n], all if None).
    With m = mag (a stated magnitude) or |ref|, u the unit roundoff of dtype:
      elementwise  |err| <= max(ATOL_U u max|ref| + RTOL_U u m, ELEM_MULT x max |base - ref|)
      per row      ||err|| <= ROW_MULT ||base - ref|| + u ||m|| + atol sqrt(H)
    NaN fails."""
    u = UNIT[dtype]
    r = ref.double()
    k = out.to(r.device).double()
    b = base.to(r.device).double()
    m = (mag.double() if mag is not None else r.abs())
    if rows is not None:
        sel = rows.to(r.device)
        r, k, b, m = r[sel], k[sel], b[sel], m[sel]
    fails = []
    if r.numel() == 0:
        return fails, {}
    atol = ATOL_U * u * r.abs().max().item()
    e, eb = (k - r).abs(), (b - r).abs()
    bound = torch.clamp(atol + RTOL_U * u * m, min=ELEM_MULT * eb.max().item())
    bad = ~(e <= bound)
    if bad.any():
        i, j = [int(v) for v in bad.nonzero()[0]]
        fails.append("%s: %d elements out of bounds, first (row %d, col %d): got %r, ref %r, bound %.3e"
                     % (name, int(bad.sum()), i, j, k[i, j].item(), r[i, j].item(), bound[i, j].item()))
    en, ebn = (k - r).norm(dim=1), (b - r).norm(dim=1)
    lim = ROW_MULT * ebn + u * m.norm(dim=1) + atol * r.shape[1] ** 0.5
    badr = ~(en <= lim)
    if badr.any():
        i = int(badr.nonzero()[0])
        fails.append("%s: %d rows out of bounds, first row %d: |err| %.3e > %.3e (baseline %.3e)"
                     % (name, int(badr.sum()), i, en[i].item(), lim[i].item(), ebn[i].item()))
    return fails, dict(max_err=e.max().item(), base_max_err=eb.max().item(),
                       worst_row_ratio=(en / lim.clamp(min=1e-300)).max().item())


def check_sums(name, out, ref, absterms, init=None, slack=None):
    """An fp32 column sum: |out - ref| <= SUM_TOL (absterms + |init|) + slack, per column (NaN fails).
    `slack` (optional, per column) is an error the reference does not share by construction."""
    r = ref.double()
    k = out.to(r.device).double()
    lim = SUM_TOL * (absterms.double() + (init.to(r.device).double().abs() if init is not None else 0)) + 1e-30
    if slack is not None:
        lim = lim + slack.double()
    e = (k - r).abs()
    bad = ~(e <= lim)
    if bad.any():
        c = int(bad.nonzero()[0])
        return ["%s: %d columns out of bounds, first col %d: got %r, ref %r, bound %.3e"
                % (name, int(bad.sum()), c, k[c].item(), r[c].item(), lim[c].item())]
    return []


def check_exact(name, out, want):
    """Bit-for-bit equality (as values; NaN never equal)."""
    if torch.equal(out, want.to(out.device, out.dtype)):
        return []
    diff = out != want.to(out.device, out.dtype)
    i = diff.nonzero()[0].tolist()
    return ["%s: %d elements differ, first %s: got %r, want %r"
            % (name, int(diff.sum()), i, out[tuple(i)].item(), want[tuple(i)].item())]


def check_ln_bwd(out, ref, base, dtype, dx0=None, dgamma0=None, dbeta0=None, dbias0=None):
    """Failures of a LayerNorm backward result `out` (dict: dx, dx_drop, dgamma, dbeta, dbias; the last
    two may be None) against ln_bwd_reference `ref` and ln_bwd_baseline `base` (on the active rows).
    Inactive rows of dx must hold dx0 (zeros if None) bit for bit.  dbias may differ from the
    reference's by the columns' sums of |round(out's Linear-branch gradient) - round(ref's)|: the
    kernel rounds its own gradient, whose error the elementwise check bounds."""
    act = ref["active"]
    fails = []
    f, _ = check_rows("dx", out["dx"][act], ref["dx"][act], base["dx"], dtype)
    fails += f
    if (~act).any():
        want = dx0[~act.to(dx0.device)] if dx0 is not None else torch.zeros_like(out["dx"][~act])
        fails += check_exact("dx (inactive rows)", out["dx"][~act], want)
    if ref["dx_drop"] is not None:
        f, _ = check_rows("dx_drop", out["dx_drop"][act], ref["dx_drop"][act], base["dx_drop"], dtype)
        fails += f
    fails += check_sums("dgamma", out["dgamma"], ref["dgamma"], ref["absg"], dgamma0)
    fails += check_sums("dbeta", out["dbeta"], ref["dbeta"], ref["absb"], dbeta0)
    if out.get("dbias") is not None:
        lin_out = out["dx_drop"] if ref["dx_drop"] is not None else out["dx"]
        lin_ref = ref["dx_drop"] if ref["dx_drop"] is not None else ref["dx"]
        dev = ref["dx"].device
        slack = (lin_out.to(dev).double() - lin_ref.to(lin_out.dtype).to(dev).double())[act].abs().sum(0)
        fails += check_sums("dbias", out["dbias"], ref["dbias"], ref["absd"], dbias0, slack)
    return fails
