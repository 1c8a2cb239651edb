"""GPU: every GEMM instantiation and epilogue against float64 (tests/gemm_check.py).

(a) Small-integer operands make every product and partial sum an exact fp32 integer, whatever the
    summation order, so the kernel's output is known bit for bit: all operand majors, tile widths,
    clusters, the masks the dispatcher specialises and generic ones, ragged M / N / K, distinct row
    pitches with poisoned pitch padding, sentinel-filled output buffers, many tiles per CTA, split-K,
    n_valid, the grouped wgrad and the deterministic-mode forms.
(b) Random operands at the encoder's shapes, checked against float64 with rigorous elementwise bounds.
(c) Every finite 16-bit input of the GELU, dGELU and tanh epilogues.
Each float64 reference is computed once per shape, on the GPU, and reused across tile configurations.
"""
import contextlib
import ctypes as C
import math

import pytest
import torch

from tests import gemm_check as gc
from tests import rowops_check as rc

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
TILES = [(0, 0), (64, 1), (128, 1), (192, 1), (256, 1), (128, 2), (256, 2)]
INT_MAX = {torch.bfloat16: 4, torch.float16: 2}       # K max^2 < 2^24 and fp16 outputs < 65504
POISON = 1024.0                                       # pitch padding of A and B: changes any result that reads it
SENTINEL = -777.0
P_DROP, SEED, STREAM = 0.25, 99, (6 << 20) | 5

B, D, R, G, T, DG = gc.EPI_BIAS, gc.EPI_DROPOUT, gc.EPI_RESIDUAL, gc.EPI_GELU, gc.EPI_TANH, gc.EPI_DGELU
ACC, F32, CS, ATOM = gc.EPI_ACCUM, gc.EPI_OUT_F32, gc.EPI_COLSUM, gc.EPI_ATOMIC
# (a_major, b_major) -> the masks dispatch_major specialises, then generic (runtime-mask) ones
MASKS = {
    (0, 0): [B, B | G, B | R, B | D | R] + [0, R | ACC, B | F32, B | T, D, B | R | CS, ACC | F32, B | R | G],
    (0, 1): [0, R, DG | CS] + [DG | R, R | ACC, DG, B | F32, DG | ACC, DG | R | ACC | CS],
    (1, 1): [0, ACC] + [ACC | F32, F32, B | R, CS, D | R, B | ACC | CS],
}
DEV = "cuda"                                          # "cpu" runs the case logic against a host stand-in


def _sync():
    if DEV == "cuda":
        torch.cuda.synchronize()


SHAPES = [(1, 72, 40), (127, 200, 776), (129, 8, 8), (257, 776, 72), (257, 136, 40)]


@contextlib.contextmanager
def deterministic(on=True):
    from uniter_b200 import _lib
    lib = _lib.load()
    prev = lib.ub200_set_deterministic(1 if on else 0)
    try:
        yield
    finally:
        lib.ub200_set_deterministic(prev)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ints(shape, lim, g, dtype):
    return torch.randint(-lim, lim + 1, shape, generator=g, device=DEV).to(dtype)


def _pitched(rows, cols, ld, dtype, fill, extra_rows=2):
    """(buffer [rows + extra_rows, ld] filled with `fill`, its [rows, cols] view)."""
    buf = torch.full((rows + extra_rows, ld), fill, device=DEV, dtype=dtype)
    return buf, buf[:rows, :cols]


def _operand(x, major, pad):
    """x: the logical [rows, K] operand; stored K-major (major 0) or as [K, rows] (major 1) in a buffer
    whose row pitch is `pad` elements (a multiple of 8) past the logical width, padding poisoned."""
    s = x if major == 0 else x.t()
    w = (s.shape[1] + 7) // 8 * 8 + pad
    buf, view = _pitched(s.shape[0], s.shape[1], w, x.dtype, POISON, extra_rows=1)
    view.copy_(s)
    return view


def _launch(a, b, a_major, b_major, M, N, K, epi, dtype, out, out2=None, bias=None, residual=None, aux=None,
            colsum=None, tile_n=0, cluster=0, max_ctas=0, k_splits=0, n_valid=0, counter=None):
    from uniter_b200 import _lib
    lib = _lib.load()
    args = _lib.GemmArgs(
        a=a.data_ptr(), b=b.data_ptr(), lda=a.stride(0), ldb=b.stride(0), a_major=a_major, b_major=b_major,
        M=M, N=N, K=K, dtype=_lib.dtype_code(dtype), epilogue=epi, bias=_lib.ptr(bias),
        residual=_lib.ptr(residual), aux=_lib.ptr(aux), out=out.data_ptr(), out2=_lib.ptr(out2),
        colsum=_lib.ptr(colsum), ldr=residual.stride(0) if residual is not None else 0,
        ldaux=aux.stride(0) if aux is not None else 0, ldo=out.stride(0),
        dropout_p=P_DROP if epi & D else 0.0, rng_seed=SEED, rng_stream=STREAM, tile_n=tile_n,
        max_ctas=max_ctas, cluster=cluster, k_splits=k_splits, n_valid=n_valid,
        rng_offset_dev=_lib.ptr(counter))
    _lib.check(lib.ub200_gemm(C.byref(args), _lib.current_stream()))


class Case(object):
    """Operands, side inputs and pitched output buffers of one (shape, majors, mask); `run` launches one
    tile configuration into freshly re-filled buffers and returns the outputs."""

    def __init__(self, M, N, K, a_major, b_major, epi, dtype, seed, make, n_valid=0, counter=None):
        g = _gen(seed)
        self.M, self.N, self.K, self.am, self.bm, self.epi, self.dtype = M, N, K, a_major, b_major, epi, dtype
        nb = n_valid or N
        self.a = _operand(make((M, K), g), a_major, 8)
        self.b = _operand(make((nb, K), g), b_major, 16)
        self.n_valid = n_valid
        self.bias = make((N,), g) if epi & B else None
        self.residual = _pitched(M, N, N + 40, dtype, SENTINEL)[1] if epi & R else None
        if self.residual is not None:
            self.residual.copy_(make((M, N), g))
        self.aux = None
        if epi & DG:
            self.aux = _pitched(M, N, N + 56, dtype, SENTINEL)[1]
            self.aux.copy_(make((M, N), g, aux=True))
        odt = torch.float32 if epi & (F32 | ATOM) else dtype
        self.out0 = make((M, N), g).to(odt) if epi & ACC else None
        self.colsum0 = make((N,), g).float() if epi & CS else None
        self.counter = counter
        self.keep, self.inv = (rc.keep_mask(SEED, STREAM, P_DROP, M, N, device=DEV,
                                            counter=int(counter.item()) if counter is not None else None)
                               if epi & D else (None, 1.0))
        self.odt = odt
        self.ref = gc.gemm_reference(self.a, self.b, a_major, b_major, N)

    def run(self, **kw):
        M, N = self.M, self.N
        ob, out = _pitched(M, N, N + 24, self.odt, SENTINEL)
        if self.epi & ATOM:
            out.zero_()
        if self.out0 is not None:
            out.copy_(self.out0)
        o2b, out2 = _pitched(M, N, N + 24, self.dtype, SENTINEL) if self.epi & G else (None, None)
        csb = torch.full((1, N + 8), SENTINEL, device=DEV) if self.epi & CS else None
        if csb is not None:
            csb[0, :N] = self.colsum0
        _launch(self.a, self.b, self.am, self.bm, M, N, self.K, self.epi, self.dtype, out, out2, self.bias,
                self.residual, self.aux, csb[0, :N] if csb is not None else None, n_valid=self.n_valid,
                counter=self.counter, **kw)
        _sync()
        fails = gc.check_untouched(ob, SENTINEL, M, N)
        if o2b is not None:
            fails += ["out2 " + f for f in gc.check_untouched(o2b, SENTINEL, M, N)]
        if csb is not None:
            fails += ["colsum " + f for f in gc.check_untouched(csb, SENTINEL, 1, N)]
        return dict(out=out, out2=out2, colsum=csb[0, :N] if csb is not None else None), fails

    def side(self):
        return dict(bias=self.bias, residual=self.residual, aux=self.aux, out0=self.out0, keep=self.keep)


def _int_maker(dtype):
    lim = INT_MAX[dtype]

    def make(shape, g, aux=False):
        if aux:       # dGELU inputs saturated: gelu'(x) is exactly 0 or 1 in the kernel
            return (torch.where(torch.rand(shape, generator=g, device=DEV) < 0.5, -1.0, 1.0)
                    * gc.SATURATED * 2).to(dtype)
        return _ints(shape, lim, g, dtype)
    return make


def _exact_fails(case, got, det=False, slices=False):
    want, exact, pre = gc.exact_expect(case.ref[0], case.epi & ~ATOM, case.dtype, **case.side())
    fails = gc.check_exact_at("out", got["out"], want, exact)
    if pre is not None:
        fails += gc.check_exact_at("out2", got["out2"], pre, torch.ones_like(exact))
    if case.epi & CS:
        assert bool(exact.all())
        terms = want.to(case.dtype).double() if det else want
        assert bool((terms.abs().sum(0) < 2 ** 24).all())        # every partial sum is an exact fp32 integer
        cs = (case.colsum0.double() + terms.sum(0))[None]
        fails += gc.check_exact_at("colsum", got["colsum"][None], cs, torch.ones_like(cs, dtype=torch.bool))
    return fails


# ------------------------------------------------------------------------------------ (a) exact
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("majors,epi", [(m, e) for m, es in MASKS.items() for e in es])
def test_exact_every_instantiation(dtype, majors, epi):
    fails = []
    for si, (M, N, K) in enumerate(SHAPES):
        case = Case(M, N, K, majors[0], majors[1], epi, dtype, seed=si, make=_int_maker(dtype))
        for tn, cl in TILES:
            got, f = case.run(tile_n=tn, cluster=cl)
            fails += ["%s tile (%d, %d): %s" % ((M, N, K), tn, cl, x) for x in f + _exact_fails(case, got)]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("majors,epi", [((0, 0), B | G), ((0, 1), DG | CS), ((1, 1), ACC)])
def test_exact_encoder_shape(dtype, majors, epi):
    """One multi-wave encoder shape: 27 row tiles, 3072 columns, K = 768."""
    M, N, K = 3456, 3072, 768
    case = Case(M, N, K, majors[0], majors[1], epi, dtype, seed=7, make=_int_maker(dtype))
    fails = []
    for tn, cl in [(0, 0), (128, 1), (256, 2)]:
        got, f = case.run(tile_n=tn, cluster=cl)
        fails += ["tile (%d, %d): %s" % (tn, cl, x) for x in f + _exact_fails(case, got)]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("majors,epi", [((0, 0), B | G), ((0, 0), B | D | R), ((0, 1), DG | CS), ((1, 1), ACC)])
def test_exact_many_tiles_per_cta(dtype, majors, epi):
    """max_ctas 1 / 3 / 7: every CTA runs many tiles, so the TMA stage ring and the hand-off chunk ring
    wrap at every phase; ragged N makes a CTA's last tile send fewer chunks than a full one."""
    M, N, K = 257, 776, 136
    counter = torch.tensor([3], device=DEV, dtype=torch.int64) if epi & D else None
    case = Case(M, N, K, majors[0], majors[1], epi, dtype, seed=11, make=_int_maker(dtype), counter=counter)
    fails = []
    for tn, cl in [(128, 2), (256, 2), (192, 1), (64, 1)]:
        for mc in (1, 3, 7):
            got, f = case.run(tile_n=tn, cluster=cl, max_ctas=mc)
            fails += ["tile (%d, %d) max_ctas %d: %s" % (tn, cl, mc, x) for x in f + _exact_fails(case, got)]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b_major", [0, 1])
def test_exact_split_k(dtype, b_major):
    """k_splits 2 / 3 / 7 / -1 over 13 k-blocks (the last slice is short, the last k-block 8 deep)."""
    M, N, K = 190, 200, 776
    case = Case(M, N, K, 0, b_major, F32 | ATOM, dtype, seed=13, make=_int_maker(dtype))
    fails = []
    for ks in (2, 3, 7, -1):
        for tn in (0, 64, 128):
            got, f = case.run(tile_n=tn, k_splits=ks)
            fails += ["k_splits %d tile %d: %s" % (ks, tn, x) for x in f + _exact_fails(case, got)]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("b_major", [0, 1])
def test_exact_n_valid(dtype, b_major):
    """B holds only n_valid of the N features (the tied decoder and its dgrad form): padding columns
    are bias only, bit for bit, and B's rows / columns past n_valid (poisoned) are never read."""
    M, K = 129, 72
    fails = []
    for nv in (131, 773):
        N = (nv + 7) // 8 * 8
        case = Case(M, N, K, 0, b_major, B, dtype, seed=nv, make=_int_maker(dtype), n_valid=nv)
        for tn, cl in TILES:
            got, f = case.run(tile_n=tn, cluster=cl)
            f = f + _exact_fails(case, got)
            if not torch.equal(got["out"][:, nv:], case.bias[nv:].expand(M, N - nv)):
                f.append("padding columns are not bias only")
            fails += ["n_valid %d tile (%d, %d): %s" % (nv, tn, cl, x) for x in f]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("accumulate", [False, True])
def test_exact_grouped_wgrad(dtype, accumulate):
    """ub200_gemm_grouped: four wgrad problems with ragged M / N and distinct output pitches."""
    from uniter_b200 import _lib
    lib = _lib.load()
    K = 200
    probs = [(200, 136), (776, 72), (129, 776), (8, 8)]
    make = _int_maker(dtype)
    g = _gen(21)
    ops_ = []
    for i, (M, N) in enumerate(probs):
        a = _operand(make((M, K), g), 1, 8 * (i + 1))
        b = _operand(make((N, K), g), 1, 8 * (i + 2))
        out0 = make((M, N), g) if accumulate else None
        ops_.append((M, N, a, b, out0, gc.gemm_reference(a, b, 1, 1)[0]))
    fails = []
    for tn in (0, 128, 192, 256):
        args = (_lib.GemmArgs * 4)()
        bufs = []
        for i, (M, N, a, b, out0, acc) in enumerate(ops_):
            ob, out = _pitched(M, N, N + 8 * (2 * i + 3), dtype, SENTINEL)
            if accumulate:
                out.copy_(out0)
            bufs.append((ob, out))
            args[i] = _lib.GemmArgs(a=a.data_ptr(), b=b.data_ptr(), lda=a.stride(0), ldb=b.stride(0), a_major=1,
                                    b_major=1, M=M, N=N, K=K, dtype=_lib.dtype_code(dtype),
                                    epilogue=ACC if accumulate else 0, out=out.data_ptr(), ldo=out.stride(0),
                                    tile_n=tn)
        _lib.check(lib.ub200_gemm_grouped(args, 4, _lib.current_stream()))
        _sync()
        for i, ((M, N, a, b, out0, acc), (ob, out)) in enumerate(zip(ops_, bufs)):
            want = acc + (out0.double() if accumulate else 0)
            f = gc.check_untouched(ob, SENTINEL, M, N) + gc.check_exact_at("out", out, want, torch.ones_like(
                want, dtype=torch.bool))
            fails += ["tile %d problem %d: %s" % (tn, i, x) for x in f]
    assert not fails, fails[:8]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("majors,epi", [((0, 1), DG | CS), ((0, 0), B | CS), ((0, 1), R | ACC), ((1, 1), B | R),
                                        ((0, 0), F32 | ATOM), ((0, 1), F32 | ATOM)])
def test_exact_deterministic_forms(dtype, majors, epi):
    """ub200_set_deterministic(1): the EPI = -2 generic kernel, DGELU | COLSUM as DGELU followed by the
    fixed-order column sum of the 16-bit output, ATOMIC as ACCUM over one slice of all of K."""
    fails = []
    with deterministic():
        for si, (M, N, K) in enumerate(SHAPES[1:]):
            case = Case(M, N, K, majors[0], majors[1], epi, dtype, seed=30 + si, make=_int_maker(dtype))
            for tn, cl in [(0, 0), (128, 2), (192, 1)]:
                got, f = case.run(tile_n=tn, cluster=cl, k_splits=3 if epi & ATOM else 0)
                fails += ["%s tile (%d, %d): %s" % ((M, N, K), tn, cl, x)
                          for x in f + _exact_fails(case, got, det=True)]
    assert not fails, fails[:8]


def test_ops_gemm_gelu_with_pitched_out():
    """ops.gemm allocates out2 with out's row pitch, which is where the kernel stores it."""
    from uniter_b200 import ops
    dtype = torch.bfloat16
    g = _gen(5)
    M, N, K = 130, 200, 64
    x, w, bias = _ints((M, K), 4, g, dtype), _ints((N, K), 4, g, dtype), _ints((N,), 4, g, dtype)
    ob, out = _pitched(M, N, N + 40, dtype, SENTINEL)
    o, pre = ops.gemm(x, w, bias=bias, out=out, gelu=True)
    _sync()
    assert o.data_ptr() == out.data_ptr() and pre.stride(0) == out.stride(0)
    acc = gc.gemm_reference(x, w)[0] + bias.double()
    assert torch.equal(pre, acc.to(dtype))
    assert not gc.check_untouched(ob, SENTINEL, M, N)
    with pytest.raises(AssertionError):
        ops.gemm(x, w, bias=bias[:N - 8])
    with pytest.raises(AssertionError):
        ops.gemm(x, w, residual=out[:, :N - 8])


# ------------------------------------------------------------------------------------ (b) random
def _rand_maker(dtype, scale_b=0.05, aux_scale=2.0):
    def make(shape, g, aux=False):
        if aux:
            return (torch.randn(shape, generator=g, device=DEV) * aux_scale).to(dtype)
        x = torch.randn(shape, generator=g, device=DEV)
        if len(shape) == 2 and shape[0] > 8:
            x[::7] += 6.0                     # rows with |mean| >> std: the S-based bound is not trivially loose
        return x.to(dtype)
    return make


def _random_check(name, M, N, K, majors, epi, dtype, seed, kw=None, n_valid=0, counter=None, det=False):
    case = Case(M, N, K, majors[0], majors[1], epi, dtype, seed, _rand_maker(dtype), n_valid=n_valid,
                counter=counter)
    # B at the scale of a weight, so that GELU / tanh see pre-activations of order 1
    case.b.mul_(0.05)
    case.ref = gc.gemm_reference(case.a, case.b, majors[0], majors[1], N)
    got, fails = case.run(**(kw or {}))
    slices = 0
    if kw and kw.get("k_splits"):
        slices = (K + 63) // 64
    f, stats = gc.check_gemm(got, case.ref, K, epi, dtype,
                             colsum0=case.colsum0, inv_keep=case.inv, slices=max(slices, 1), deterministic=det,
                             **case.side())
    print("RATIO %s %s %s" % (name, str(dtype).split(".")[-1],
                               " ".join("%s=%.3f" % kv for kv in sorted(stats.items()))))
    return fails + f


T_C2 = 3456
ROLES = [
    ("qkv fwd", (T_C2, 2304, 768), (0, 0), B, {}),
    ("attn-out fwd", (T_C2, 768, 768), (0, 0), B | D | R, {}),
    ("ffn1 fwd", (T_C2, 3072, 768), (0, 0), B | G, {}),
    ("ffn2 fwd", (T_C2, 768, 3072), (0, 0), B | D | R, {}),
    ("ffn2 dgrad", (T_C2, 3072, 768), (0, 1), DG | CS, {}),
    ("ffn1 dgrad", (T_C2, 768, 3072), (0, 1), R, {}),
    ("qkv dgrad", (T_C2, 768, 2304), (0, 1), R, {}),
    ("ffn1 wgrad", (3072, 768, T_C2), (1, 1), ACC, {}),
    ("pooler fwd", (64, 768, 768), (0, 0), B | T, {}),
    ("decoder dgrad split-K", (190, 768, 28996), (0, 1), F32 | ATOM, {"k_splits": -1}),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("role", ROLES, ids=[r[0] for r in ROLES])
def test_random_roles(dtype, role):
    name, (M, N, K), majors, epi, kw = role
    counter = torch.tensor([9], device=DEV, dtype=torch.int64) if epi & D else None
    fails = _random_check(name, M, N, K, majors, epi, dtype, seed=M + N + K, kw=kw, counter=counter)
    assert not fails, fails


@pytest.mark.parametrize("dtype", DTYPES)
def test_random_decoder_n_valid(dtype):
    fails = _random_check("decoder n_valid", 190, 29000, 768, (0, 0), B, dtype, seed=3, n_valid=28996)
    assert not fails, fails


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("majors", list(MASKS))
def test_random_every_mask_ragged(dtype, majors):
    fails = []
    for epi in MASKS[majors]:
        fails += _random_check("mask %d majors %s" % (epi, majors), 257, 200, 776, majors, epi, dtype, seed=epi)
    with deterministic():
        fails += _random_check("det colsum majors %s" % (majors,), 257, 200, 776, majors,
                               (DG | CS) if majors == (0, 1) else CS, dtype, seed=1, det=True)
    assert not fails, fails


# ------------------------------------------------------------------------------------ (c) exhaustive
def _all_finite(dtype):
    """Every finite 16-bit value, as a [256, 256] matrix (non-finite patterns replaced by 0)."""
    x = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16).view(dtype)
    return torch.where(torch.isfinite(x), x, torch.zeros_like(x)).reshape(256, 256)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("epi", [B | G, T], ids=["gelu", "tanh"])
def test_exhaustive_gelu_tanh(dtype, epi):
    """acc = I . X^T = X^T exactly, so out[m, n] = f(X[n, m]) for every finite X: BIAS | GELU with a zero
    bias (the specialised kernel), TANH alone (the generic one).  GELU also states normal_cdf's budget:
    |Phi_kernel(x) - Phi(x)| <= DELTA_PHI, Phi_kernel recovered as out / x."""
    X = _all_finite(dtype)
    eye = torch.eye(256, device=DEV, dtype=dtype)
    out = torch.empty(256, 256, device=DEV, dtype=dtype)
    out2 = torch.empty_like(out) if epi & G else None
    bias = torch.zeros(256, device=DEV, dtype=dtype)
    _launch(eye, X, 0, 0, 256, 256, 256, epi, dtype, out, out2, bias=bias if epi & B else None)
    _sync()
    x = X.t()
    ref = (gc.gemm_reference(eye, X)[0], torch.abs(x.double()))
    assert torch.equal(ref[0], x.double())
    fails, stats = gc.check_gemm(dict(out=out, out2=out2), ref, 256, epi, dtype, bias=bias)
    if epi & G:
        xd = x.double()
        nz = xd != 0
        phi_k = out.double()[nz] / xd[nz]
        phi = 0.5 * torch.special.erfc(-xd[nz] / math.sqrt(2.0))
        lim = gc.DELTA_PHI + (rc.UNIT[dtype] * out.double()[nz].abs() + gc.TINY[dtype]) / xd[nz].abs() \
            + 2 * gc.U32 * phi_k.abs()
        err = (phi_k - phi).abs()
        f, r = gc._worst("Phi", err, lim)
        fails += f
        stats["Phi"] = r
        tail = (xd[nz] < -3)
        print("RATIO Phi tail max |err| %.3e (x < -3), overall %.3e" % (err[tail].max().item(), err.max().item()))
    print("RATIO exhaustive %s %s %s" % ("gelu" if epi & G else "tanh", str(dtype).split(".")[-1],
                                          " ".join("%s=%.3f" % kv for kv in sorted(stats.items()))))
    assert not fails, fails


@pytest.mark.parametrize("dtype", DTYPES)
def test_exhaustive_dgelu(dtype):
    """acc = 1 exactly (one unit product per element) and aux = every finite value: the specialised
    DGELU | COLSUM dgrad kernel evaluates gelu'(x) on every 16-bit x."""
    M = N = 256
    K = 8
    a = torch.zeros(M, K, device=DEV, dtype=dtype)
    a[:, 0] = 1
    b = torch.zeros(K, N, device=DEV, dtype=dtype)
    b[0] = 1
    aux = _all_finite(dtype)
    out = torch.empty(M, N, device=DEV, dtype=dtype)
    colsum = torch.zeros(N, device=DEV)
    _launch(a, b, 0, 1, M, N, K, DG | CS, dtype, out, aux=aux, colsum=colsum)
    _sync()
    ref = gc.gemm_reference(a, b, 0, 1)
    assert bool((ref[0] == 1).all())
    fails, stats = gc.check_gemm(dict(out=out, colsum=colsum), ref, K, DG | CS, dtype, aux=aux)
    print("RATIO exhaustive dgelu %s %s" % (str(dtype).split(".")[-1],
                                            " ".join("%s=%.3f" % kv for kv in sorted(stats.items()))))
    assert not fails, fails
