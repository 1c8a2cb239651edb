"""Reference, bounds and checker for the wgmma GEMM and its epilogues (ops.gemm / ub200_gemm,
csrc/gemm_impl.cuh).

* `gemm_reference`: float64 acc = A.B^T for any operand majors, and S = |A|.|B|^T, the sum of |terms|
  of every element.  Both are plain float64 matmuls (on the GPU in the GPU tests).
* `check_gemm`: applies the epilogue chain in the order include/ub200.h documents (bias -> dropout ->
  residual -> GELU / tanh -> dGELU(aux) -> accumulate -> store, column sum) to the reference in float64,
  carrying an elementwise bound on the kernel's error through it:
    accumulation      |acc32 - acc64| <= 2 (K + 16 + slices) u32 S   (any summation order, truncating
                      tensor-core adds, split-K slices meeting through atomics)
    each later fp32 op   + u32 |value|
    the 16-bit store     + u16 |value| (+ half the subnormal spacing)
  GELU is checked in two stages: out2 (the pre-activation, rounded to 16 bits before GELU) against the
  float64 pre-activation, then out against float64 gelu(out2) of the kernel's own out2, so that a
  rounding tie of the pre-activation cannot turn into a GELU failure.  GELU, dGELU and tanh are bounded
  by the rule of rowops_check: max(u16 |ref| + |x| DELTA_PHI + u32 terms, 1.25 x the error of the eager
  16-bit baseline), the baseline being the reference model's composed GELU (and its autograd
  derivative, and torch.tanh) in the kernel dtype.
  Column sums: the default mode sums the fp32 values in the epilogue (4 rows per thread, 3 shuffle
  levels, then atomics in any order); the deterministic mode sums the kernel's own 16-bit output in
  launch_colsum_det's order (as nn.Linear's bias gradient sums the 16-bit gradient).
* `exact_expect`: for operands that are small integers every product and partial sum is an exact
  fp32 integer, so the kernel's result is known bit for bit wherever the epilogue stays in integers
  (and where GELU / dGELU / tanh saturate to exactly 0 / 1 / +-1).
* `check_untouched`: bit-for-bit check that a pitched buffer holds its sentinel outside [:rows, :cols].

Pure torch, on any device: the GPU tests run it on the kernel's output, the CPU tests on a float32
stand-in and on mutations of it.
"""
import math

import torch

from oracle import encoder_oracle as orc
from tests.rowops_check import UNIT

EPI_BIAS, EPI_DROPOUT, EPI_RESIDUAL, EPI_GELU = 1, 2, 4, 8
EPI_DGELU, EPI_ACCUM, EPI_OUT_F32, EPI_COLSUM = 16, 32, 64, 128
EPI_ATOMIC, EPI_TANH = 256, 512

U32 = 2.0 ** -24
# Absolute error of the kernel's normal_cdf (csrc/ptx.cuh) in Phi: the A&S 7.1.26 formula's 1.5e-7 in erf
# (0.75e-7 in Phi), its fp32 Horner evaluation (up to 2.7e-7 in Phi around |x| < 2, from an exact-exp2
# emulation over every 16-bit x) and the MUFU rcp / ex2 approximations.  Absolute: for x < -4 it is a
# large relative error (Phi(-5) = 2.9e-7), which is why the GELU / dGELU bounds carry |x| DELTA_PHI.
DELTA_PHI = 4e-7
EX2_REL = 2.0 ** -20       # relative error of exp(-x^2/2) through ex2.approx (with the rounded argument)
TANH_ULPS = 2              # CUDA tanhf: 2 ulp
TINY = {torch.bfloat16: 2.0 ** -134, torch.float16: 2.0 ** -25}   # half the smallest subnormal spacing
SATURATED = 16.0           # |x| from which the kernel's GELU / dGELU / tanh are exactly x or 0 / 1 or 0 / +-1
BASE_MULT = 1.25


def _logical(x, major):
    """The [rows, K] float64 view of an operand stored K-major (major 0) or as [K, rows] (major 1)."""
    x = x.double()
    return x if major == 0 else x.t()


def gemm_reference(a, b, a_major=0, b_major=0, N=None):
    """(acc, S) [M, N] in float64.  `N` > the number of features b holds: the rest get acc = 0 (n_valid)."""
    A, B = _logical(a, a_major), _logical(b, b_major)
    acc, S = A @ B.t(), A.abs() @ B.abs().t()
    if N is not None and N > acc.shape[1]:
        pad = torch.zeros(acc.shape[0], N - acc.shape[1], dtype=acc.dtype, device=acc.device)
        acc, S = torch.cat([acc, pad], 1), torch.cat([S, pad], 1)
    return acc, S


# ----------------------------------------------------------------------------- elementwise functions
def gelu64(x):
    x = x.double()
    return x * 0.5 * torch.special.erfc(-x / math.sqrt(2.0))


def phi64(x):
    return torch.exp(-0.5 * x.double() ** 2) / math.sqrt(2.0 * math.pi)


def dgelu64(x):
    x = x.double()
    return 0.5 * torch.special.erfc(-x / math.sqrt(2.0)) + x * phi64(x)


def gelu_baseline(x16):
    """The reference model's GELU (model/layer.py:31-37) in the 16-bit dtype, as it runs under apex O2."""
    return orc.gelu_erf(x16)


def dgelu_baseline(x16):
    """d gelu / dx of the same composed 16-bit ops, through autograd."""
    x = x16.detach().clone().requires_grad_(True)
    orc.gelu_erf(x).backward(torch.ones_like(x))
    return x.grad


def _base_err(base, ref):
    """|baseline - ref|, with the baseline's own overflow / NaN (huge inputs) counted as no slack."""
    return torch.nan_to_num((base.double() - ref).abs(), nan=0.0, posinf=0.0)


def dgelu_bound(x, ref, dtype):
    """Bound of the kernel's dgelu(x) (before any rounding) against ref = dgelu64(x): (rigorous, baseline)."""
    xd = x.double()
    rig = DELTA_PHI + torch.nan_to_num((xd * phi64(xd)).abs()) * EX2_REL + 2 * U32 * ref.abs()
    return rig, _base_err(dgelu_baseline(x.to(dtype)), ref)


# ----------------------------------------------------------------------------- the checker
def _worst(name, err, bound, got=None, ref=None):
    """(failure strings, max err / bound) of an elementwise comparison; NaN fails."""
    ratio = err / bound.clamp(min=1e-300)
    bad = ~(err <= bound)
    r = ratio.max().item() if ratio.numel() else 0.0
    if not bad.any():
        return [], r
    ratio = torch.where(bad & torch.isnan(ratio), torch.full_like(ratio, math.inf), ratio)
    idx = int(torch.argmax(torch.where(bad, ratio, torch.full_like(ratio, -1.0)).reshape(-1)))
    pos = [idx] if err.dim() == 1 else [idx // err.shape[1], idx % err.shape[1]]
    where = ("col %d" % pos[0]) if err.dim() == 1 else ("row %d, col %d" % (pos[0], pos[1]))
    tail = ""
    if got is not None:
        tail = ": got %r, ref %r" % (got.reshape(-1)[idx].item(), ref.reshape(-1)[idx].item())
    return ["%s: %d elements out of bounds, worst at %s, err / bound = %.3g (err %.3e, bound %.3e)%s"
            % (name, int(bad.sum()), where, ratio.reshape(-1)[idx].item(), err.reshape(-1)[idx].item(),
               bound.reshape(-1)[idx].item(), tail)], r


def check_gemm(got, ref, K, epi, dtype, *, bias=None, residual=None, aux=None, out0=None, colsum0=None,
               keep=None, inv_keep=1.0, slices=1, deterministic=False):
    """Failures (list of strings) and {output: max err / bound} of a GEMM result against `ref` = (acc, S)
    of gemm_reference.

    got: dict with `out` [M, N] (16-bit, or fp32 with EPI_OUT_F32), `out2` (EPI_GELU), `colsum` (EPI_COLSUM).
    epi: the epilogue mask (EPI_ATOMIC is the split-K form of a plain fp32 product).  bias [N], residual /
    aux / out0 (the output's contents before an EPI_ACCUM launch) [M, N]; keep: the bool dropout keep
    mask and inv_keep its scale (rowops_check.keep_mask); slices: the number of split-K slices;
    deterministic: the column sum is that of the deterministic mode."""
    acc, S = ref
    dev = acc.device
    M, N = acc.shape
    u16 = UNIT[dtype]
    d = lambda t: t.to(dev).double()                         # noqa: E731
    fails, stats = [], {}
    v = acc.clone()
    e = 2.0 * (K + 16 + slices) * U32 * S
    base_err = None                                          # 1.25 x baseline, once a transcendental ran
    if epi & EPI_BIAS:
        v = v + d(bias)[None]
        e = e + U32 * (v.abs() + e)
    if epi & EPI_DROPOUT:
        kp = keep.to(dev)
        v = torch.where(kp, v * inv_keep, torch.zeros_like(v))
        e = torch.where(kp, e * inv_keep + U32 * (v.abs() + e * inv_keep), torch.zeros_like(e))
    if epi & EPI_RESIDUAL:
        v = v + d(residual)
        e = e + U32 * (v.abs() + e)
    if epi & EPI_GELU:
        pre = got["out2"]
        f, stats["out2"] = _worst("out2", (d(pre) - v).abs(), e + u16 * (v.abs() + e) + TINY[dtype], pre, v)
        fails += f
        x = d(pre)
        v = gelu64(x)
        e = x.abs() * DELTA_PHI + 2 * U32 * v.abs()
        base_err = BASE_MULT * _base_err(gelu_baseline(pre.to(dev)), v)
    if epi & EPI_TANH:
        t = torch.tanh(v)
        e = e + 2 * TANH_ULPS * U32 * t.abs()
        base_err = BASE_MULT * _base_err(torch.tanh(v.to(dtype)), t)
        v = t
    if epi & EPI_DGELU:
        xa = d(aux)
        g = dgelu64(xa)
        eg, bg = dgelu_bound(xa, g, dtype)
        vg = v * g
        e = e * g.abs() + v.abs() * eg + U32 * (vg.abs() + e * g.abs())
        be = v.abs() * bg
        base_err = BASE_MULT * be if base_err is None else base_err * g.abs() + BASE_MULT * be
        v = vg
    if epi & EPI_ACCUM:
        v = v + d(out0)
        e = e + U32 * (v.abs() + e)
    out = got["out"]
    if epi & (EPI_OUT_F32 | EPI_ATOMIC):
        bound = e
    else:
        bound = e + u16 * (v.abs() + e) + TINY[dtype]
    if base_err is not None:
        bound = torch.maximum(bound, base_err)
    f, stats["out"] = _worst("out", (d(out) - v).abs(), bound, out, v)
    fails += f
    if epi & EPI_COLSUM:
        c0 = d(colsum0) if colsum0 is not None else torch.zeros(N, dtype=torch.float64, device=dev)
        if deterministic:
            o = d(out)
            want = c0 + o.sum(0)
            depth = -(-M // 256) + 8 + 1
            cb = 2 * depth * U32 * (o.abs().sum(0) + c0.abs())
        else:
            want = c0 + v.sum(0)
            depth = 3 + 3 + -(-M // 32) + 1
            cb = e.sum(0) + 2 * depth * U32 * (v.abs().sum(0) + e.sum(0) + c0.abs())
        f, stats["colsum"] = _worst("colsum", (d(got["colsum"]) - want).abs(), cb, got["colsum"], want)
        fails += f
    return fails, stats


# ----------------------------------------------------------------------------- integer operands
def exact_expect(acc, epi, dtype, *, bias=None, residual=None, aux=None, out0=None, keep=None):
    """(want, exact, want_pre) for integer operands: `want` [M, N] float64 holds the kernel's output value
    wherever `exact` (bool [M, N]) is set — everywhere except kept dropout positions (scaled by 1/keep)
    and GELU / dGELU / tanh inputs below SATURATED in magnitude; want_pre is the GELU pre-activation
    (exact everywhere).  Stores round the exact fp32 integer once, as `want.to(dtype)` does."""
    dev = acc.device
    d = lambda t: t.to(dev).double()                         # noqa: E731
    v = acc.clone()
    exact = torch.ones_like(v, dtype=torch.bool)
    pre = None
    if epi & EPI_BIAS:
        v = v + d(bias)[None]
    if epi & EPI_DROPOUT:
        kp = keep.to(dev)
        v = torch.where(kp, v, torch.zeros_like(v))
        exact &= ~kp
    if epi & EPI_RESIDUAL:
        v = v + d(residual)
    if epi & EPI_GELU:
        pre = v.to(dtype).double()
        v = torch.where(pre > 0, pre, torch.zeros_like(pre))
        exact &= pre.abs() >= SATURATED
    if epi & EPI_TANH:
        exact &= v.abs() >= SATURATED
        v = torch.sign(v)
    if epi & EPI_DGELU:
        xa = d(aux)
        exact &= xa.abs() >= SATURATED
        v = torch.where(xa > 0, v, torch.zeros_like(v))
    if epi & EPI_ACCUM:
        v = v + d(out0)
    return v, exact, pre


def check_exact_at(name, got, want, exact):
    """Bit-for-bit equality (as values) of `got` with `want` (float64, converted to got's dtype) where
    `exact` is set."""
    w = want.to(got.dtype).to(got.device)
    sel = exact.to(got.device)
    if torch.equal(got[sel], w[sel]):
        return []
    diff = (got != w) & sel
    i, j = [int(t) for t in diff.nonzero()[0]]
    return ["%s: %d elements differ, first (row %d, col %d): got %r, want %r"
            % (name, int(diff.sum()), i, j, got[i, j].item(), w[i, j].item())]


def check_untouched(buf, sentinel, rows, cols):
    """Failures if any element of the pitched buffer `buf` outside [:rows, :cols] differs, bit for bit,
    from `sentinel` (a scalar of buf's dtype)."""
    want = torch.full((), sentinel, dtype=buf.dtype, device=buf.device)
    ib = buf.view(torch.int16) if buf.element_size() == 2 else buf.view(torch.int32)
    iw = want.reshape(1).view(ib.dtype)[0]
    bad = ib != iw
    bad[:rows, :cols] = False
    if not bad.any():
        return []
    i, j = [int(t) for t in bad.nonzero()[0]]
    return ["untouched: %d elements outside [:%d, :%d] overwritten, first (row %d, col %d)"
            % (int(bad.sum()), rows, cols, i, j)]
