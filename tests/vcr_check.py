"""Reference, baseline and error checker of the ReLU-input LayerNorm (ops.layernorm_fwd / layernorm_bwd
with relu=True, csrc/rowops.cu): y = LayerNorm(relu(pre)), the Linear(H, 2H) -> ReLU -> LayerNorm(2H)
prefix of the VCR head, at widths up to 2048.

* `relu_ln_fwd_reference` / `relu_ln_bwd_reference`: float64 from the same 16-bit `pre`; the backward
  gives dx (the gradient at relu(pre)), dpre = dx o (pre > 0), dgamma, dbeta and dbias = the column
  sums of dpre rounded to the 16-bit type, with the sums of |terms| that bound the fp32 sums.
* `relu_ln_baseline`: eager torch in the kernel dtype (F.relu, F.layer_norm, autograd).
* `check_fwd` / `check_bwd`: the bounds of tests/rowops_check.py (check_rows, check_sums), plus dpre
  exactly 0 wherever pre <= 0.

Pure torch, on any device: the GPU tests run it on the kernels' output, the CPU tests on a float32
stand-in and on mutations of it.
"""
import torch
import torch.nn.functional as F

from tests import rowops_check as rc


def relu_ln_fwd_reference(pre, gamma, beta):
    return rc.ln_fwd_reference(pre.double().clamp(min=0), gamma, beta)


def relu_ln_bwd_reference(dy, pre, gamma, relu=True):
    """relu=False: the plain LayerNorm backward in the same form (dpre = dx, dbias = its column sums)."""
    x = pre.double().clamp(min=0) if relu else pre.double()
    ref = rc.ln_bwd_reference(dy, x, gamma)
    live = (pre.double() > 0).double() if relu else torch.ones_like(x)
    dpre = ref["dx"] * live
    lin = dpre.to(dy.dtype).double()
    # the kernels take mean / rstd in fp32: each dgamma term dy * xhat carries an error of a few units of
    # 2^-24 in (|x| + |mean|) rstd, which is not an error of the summation that SUM_TOL bounds
    mean = x.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((x - mean) ** 2).mean(-1, keepdim=True) + rc.EPS)
    stat_slack = (dy.double().abs() * (x.abs() + mean.abs()) * rstd).sum(0) * 2.0 ** -20
    return dict(dx=ref["dx"], dpre=dpre, dgamma=ref["dgamma"], dbeta=ref["dbeta"], dbias=lin.sum(0),
                absg=ref["absg"], absb=ref["absb"], absd=lin.abs().sum(0), stat_slack=stat_slack)


def relu_ln_baseline(dy, pre, gamma, beta, relu=True):
    """y, dx, dpre of eager torch in the kernel dtype (relu=False: dpre = dx)."""
    p = pre.detach().clone().requires_grad_(True)
    r = F.relu(p) if relu else p * 1
    r.retain_grad()
    y = F.layer_norm(r, (pre.size(-1),), gamma, beta, rc.EPS)
    y.backward(dy)
    return dict(y=y.detach(), dx=r.grad, dpre=p.grad)


def _finite(base, ref):
    """The baseline where it is finite, else the reference: eager fp16 torch overflows to inf / NaN on a row
    whose relu is constant (rstd = 1e6), and a non-finite yardstick bounds nothing."""
    b = base.to(ref.device).double()
    return torch.where(torch.isfinite(b), b, ref.double())


def check_fwd(y, ref, base, dtype):
    return rc.check_rows("y", y, ref, _finite(base, ref), dtype)[0]


def check_bwd(out, ref, base, pre, dtype, relu=True):
    """Failures of out (dict: dx, dpre, dgamma, dbeta, dbias) against relu_ln_bwd_reference `ref` and
    relu_ln_baseline `base` (relu=False: out's dpre is None and dbias sums dx).  dbias may differ from
    the reference's by the columns' sums of |out's dpre - round(ref's dpre)| (the kernel sums its own
    rounded gradient); dgamma by the error of fp32 statistics (ref["stat_slack"])."""
    fails = []
    fails += rc.check_rows("dx", out["dx"], ref["dx"], _finite(base["dx"], ref["dx"]), dtype)[0]
    if relu:
        fails += rc.check_rows("dpre", out["dpre"], ref["dpre"], _finite(base["dpre"], ref["dpre"]), dtype)[0]
        dead = (pre <= 0).to(out["dpre"].device)
        if (out["dpre"][dead] != 0).any():
            fails.append("dpre: %d elements with pre <= 0 are not 0" % int((out["dpre"][dead] != 0).sum()))
    else:
        out = dict(out, dpre=out["dx"])
    fails += rc.check_sums("dgamma", out["dgamma"], ref["dgamma"], ref["absg"], slack=ref["stat_slack"])
    fails += rc.check_sums("dbeta", out["dbeta"], ref["dbeta"], ref["absb"])
    dev = ref["dpre"].device
    slack = (out["dpre"].to(dev).double() - ref["dpre"].to(out["dpre"].dtype).to(dev).double()).abs().sum(0)
    fails += rc.check_sums("dbias", out["dbias"], ref["dbias"], ref["absd"], slack=slack)
    return fails


def relu_ln_case(rows, W, dtype, seed, device="cpu"):
    """pre [rows, W] with negatives, exact zeros (every 7th column) and, for rows > 1, an all-negative
    row (row 1, whose relu is all zeros: variance 0); gamma / beta around 1 / 0; dy."""
    g = torch.Generator().manual_seed(seed)
    pre = torch.randn(rows, W, generator=g) * 1.5 + 0.2
    pre[:, ::7] = 0.0
    if rows > 1:
        pre[1] = -pre[1].abs() - 0.01
    gamma = 1.0 + 0.1 * torch.randn(W, generator=g)
    beta = 0.1 * torch.randn(W, generator=g)
    dy = torch.randn(rows, W, generator=g)
    if rows > 1:        # relu(row 1) is constant: rstd = 1e6, a dy of 2^-14 keeps its dx finite in fp16
        dy[1] *= 2.0 ** -14
    return tuple(t.to(device=device, dtype=dtype) for t in (pre, gamma, beta, dy))
