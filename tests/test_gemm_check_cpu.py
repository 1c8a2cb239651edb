"""CPU: the checker of tests/gemm_check.py.  It must accept a float32 stand-in for a GEMM kernel (the
same epilogue chain in torch ops, another summation order) and reject each single mutation of it that
a tiling, rounding, epilogue-order, pitch or reduction bug would produce."""
import pytest
import torch

from tests import gemm_check as gc
from tests import rowops_check as rc

M, N, K = 150, 136, 72                   # ragged against 128-row tiles, 64-column chunks and 64-deep k-blocks
LDR, LDO = 152, 144                      # row pitches of the residual and of the output
SEED, STREAM, P = 11, (3 << 20) | 2, 0.1
SENTINEL = -777.0


def _round(x, dtype, rtz=False):
    """float32 -> dtype, round to nearest even (or toward zero)."""
    r = x.to(dtype)
    if not rtz:
        return r
    over = r.float().abs() > x.abs()
    bits = r.view(torch.int16)
    return torch.where(over, bits - 1, bits).view(dtype)


def _gelu_tanh(x):
    return 0.5 * x * (1 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))


def _standin(a, b, epi, dtype, bias, residual_buf, aux, out0, keep, inv_keep, mutation=None):
    """What the kernel computes, in float32 torch ops: acc summed k-block by k-block in reverse order.
    Returns (out, out2, colsum, out_buf) with out living in a sentinel-filled [M + 2, LDO] buffer."""
    nkb = (K + 63) // 64
    acc = torch.zeros(M, N)
    for kb in reversed(range(nkb)):
        if mutation == "K-tail k-block dropped" and kb == nkb - 1:
            continue
        acc += a[:, 64 * kb:64 * kb + 64].float() @ b[:, 64 * kb:64 * kb + 64].float().t()
    v = acc
    if mutation == "bias added after the 16-bit rounding":
        v = v.to(dtype).float()
    if epi & gc.EPI_BIAS:
        v = v + bias.float()
    if epi & gc.EPI_DROPOUT:
        v = torch.where(keep, v * inv_keep, torch.zeros_like(v))
    if epi & gc.EPI_RESIDUAL:
        ld = LDO if mutation == "residual read with pitch ldo" else LDR
        res = residual_buf.reshape(-1)[:(M - 1) * ld + N].as_strided((M, N), (ld, 1))
        v = v + res.float()
    out2 = None
    if epi & gc.EPI_GELU:
        out2 = v.to(dtype)
        x = v if mutation == "GELU of the unrounded pre-activation" else out2.float()
        if mutation == "tanh-approximation GELU":
            v = _gelu_tanh(x)
        else:
            v = gc.gelu64(x).float()
    if epi & gc.EPI_DGELU:
        v = v * gc.dgelu64(aux).float()
    if epi & gc.EPI_ACCUM:
        v = v + out0.float()
    colsum = v.sum(0) if epi & gc.EPI_COLSUM else None
    if mutation == "one row tile missing from the column sum":
        colsum = colsum - v[128:256].sum(0)
    out = _round(v, dtype, rtz=mutation == "round toward zero")
    if mutation == "two columns swapped inside a 64-column chunk":
        out = out.clone()
        out[:, [67, 70]] = out[:, [70, 67]]
    buf = torch.full((M + 2, LDO), SENTINEL, dtype=dtype)
    buf[:M, :N] = out
    if mutation == "one row written past M":
        buf[M, :N] = out[M - 1]
    return buf[:M, :N], out2, colsum, buf


def _case(dtype, epi, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(dtype)
    b = (torch.randn(N, K, generator=g) * 0.3).to(dtype)
    a[::9] = (a[::9].float() + 8).to(dtype)                       # rows with |mean| >> std
    bias = torch.randn(N, generator=g).to(dtype)
    residual_buf = torch.randn(M + 1, LDR, generator=g).to(dtype)
    aux = (torch.randn(M, N, generator=g) * 2).to(dtype)
    out0 = torch.randn(M, N, generator=g).to(dtype)
    keep, inv = rc.keep_mask(SEED, STREAM, P, M, N, counter=5)
    if epi & gc.EPI_GELU:                 # pre-activations over GELU's curved part and its left tail
        bias = (torch.rand(N, generator=g) * 6 - 4).to(dtype)
        b = (b.float() * 0.1).to(dtype)
    return a, b, bias, residual_buf, aux, out0, keep, inv


def _run(dtype, epi, mutation=None):
    a, b, bias, residual_buf, aux, out0, keep, inv = _case(dtype, epi)
    out, out2, colsum, buf = _standin(a, b, epi, dtype, bias, residual_buf, aux, out0, keep, inv, mutation)
    ref = gc.gemm_reference(a, b)
    fails, stats = gc.check_gemm(dict(out=out, out2=out2, colsum=colsum), ref, K, epi, dtype, bias=bias,
                                 residual=residual_buf[:M, :N], aux=aux, out0=out0, keep=keep, inv_keep=inv)
    fails += gc.check_untouched(buf, SENTINEL, M, N)
    return fails, stats


EPIS = [gc.EPI_BIAS | gc.EPI_DROPOUT | gc.EPI_RESIDUAL | gc.EPI_COLSUM,
        gc.EPI_BIAS | gc.EPI_GELU,
        gc.EPI_DGELU | gc.EPI_ACCUM | gc.EPI_COLSUM]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("epi", EPIS)
def test_standin_passes(dtype, epi):
    fails, stats = _run(dtype, epi)
    assert not fails, fails
    # the rounding-dominated output sits near its bound: a 1-ulp fault cannot hide under it
    if not epi & gc.EPI_GELU:
        assert stats["out"] > 0.5, stats


MUTATIONS = [
    ("K-tail k-block dropped", gc.EPI_BIAS, "out"),
    ("two columns swapped inside a 64-column chunk", gc.EPI_BIAS, "out"),
    ("bias added after the 16-bit rounding", gc.EPI_BIAS, "out"),
    ("round toward zero", gc.EPI_BIAS | gc.EPI_RESIDUAL, "out"),
    ("residual read with pitch ldo", gc.EPI_BIAS | gc.EPI_RESIDUAL, "out"),
    ("one row written past M", gc.EPI_BIAS | gc.EPI_RESIDUAL, "untouched"),
    ("one row tile missing from the column sum", gc.EPI_BIAS | gc.EPI_DROPOUT | gc.EPI_RESIDUAL | gc.EPI_COLSUM,
     "colsum"),
]
GELU_MUTATIONS = ["tanh-approximation GELU", "GELU of the unrounded pre-activation"]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mutation,epi,name", MUTATIONS, ids=[m[0] for m in MUTATIONS])
def test_mutation_fails(dtype, mutation, epi, name):
    fails, _ = _run(dtype, epi, mutation)
    assert any(f.startswith(name) for f in fails), "%s not caught in %s: %s" % (mutation, name, fails)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mutation", GELU_MUTATIONS)
def test_gelu_mutation_fails(dtype, mutation):
    fails, _ = _run(dtype, gc.EPI_BIAS | gc.EPI_GELU, mutation)
    assert any(f.startswith("out:") for f in fails), "%s not caught: %s" % (mutation, fails)


def test_check_untouched_and_exact_expect():
    buf = torch.full((4, 16), SENTINEL, dtype=torch.bfloat16)
    buf[:3, :8] = 1
    assert not gc.check_untouched(buf, SENTINEL, 3, 8)
    buf[1, 8] = 0
    assert gc.check_untouched(buf, SENTINEL, 3, 8)
    acc = torch.tensor([[20.0, -20.0, 3.0]], dtype=torch.float64)
    want, exact, pre = gc.exact_expect(acc, gc.EPI_GELU, torch.bfloat16)
    assert exact.tolist() == [[True, True, False]] and want[0, :2].tolist() == [20.0, 0.0]
    assert torch.equal(pre, acc)
