"""GPU: wgmma GEMM core vs a plain torch fp32 reference of the same op (floating-point kernel:
tolerance = a few ulps of the 16-bit output type, stated per dtype)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 2e-2, torch.float16: 4e-3}   # relative to max|ref| (>= 1)


def _close(got, ref, tol, what):
    err = (got.float() - ref).abs().max().item()
    lim = tol * max(1.0, ref.abs().max().item())
    assert err <= lim, "%s: max err %.4e > %.4e" % (what, err, lim)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(128, 128, 64), (333, 768, 768), (3451, 2304, 768), (777, 768, 3072),
                                   (1, 64, 64), (130, 8, 72)])
@pytest.mark.parametrize("tn,cluster", [(0, 0), (64, 1), (128, 1), (192, 1), (256, 1), (128, 2), (256, 2)])
def test_gemm_operand_majors(dtype, shape, tn, cluster):
    from uniter_b200 import ops
    M, N, K = shape
    torch.manual_seed(M * 7 + N)
    x = torch.randn(M, K, device="cuda").to(dtype)
    w = (torch.randn(N, K, device="cuda") * 0.05).to(dtype)
    ref = x.float() @ w.float().t()
    _close(ops.gemm(x, w, tile_n=tn, cluster=cluster), ref, TOL[dtype], "K-major x K-major")
    wt = w.t().contiguous()
    _close(ops.gemm(x, wt, b_major=1, tile_n=tn, cluster=cluster), ref, TOL[dtype],
           "K-major x MN-major (dgrad form)")
    Mp = (M + 7) // 8 * 8
    xt = torch.zeros(K, Mp, device="cuda", dtype=dtype)[:, :M]
    xt.copy_(x.t())
    _close(ops.gemm(xt, wt, a_major=1, b_major=1, tile_n=tn, cluster=cluster), ref, TOL[dtype],
           "MN-major x MN-major (wgrad form)")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_gemm_epilogues(dtype):
    from uniter_b200 import ops
    tol = TOL[dtype]
    torch.manual_seed(1)
    M, N, K = 515, 768, 768
    x = torch.randn(M, K, device="cuda").to(dtype)
    w = (torch.randn(N, K, device="cuda") * 0.05).to(dtype)
    bias = torch.randn(N, device="cuda").to(dtype)
    res = torch.randn(M, N, device="cuda").to(dtype)
    base = x.float() @ w.float().t()
    _close(ops.gemm(x, w, bias=bias), base + bias.float(), tol, "bias")
    _close(ops.gemm(x, w, bias=bias, residual=res), base + bias.float() + res.float(), tol, "bias+res")
    out, pre = ops.gemm(x, w, bias=bias, gelu=True)
    _close(pre, base + bias.float(), tol, "pre-activation")
    _close(out, torch.nn.functional.gelu(base + bias.float()), tol, "erf gelu")
    aux = torch.randn(M, N, device="cuda").to(dtype)
    a32 = aux.float().requires_grad_(True)
    torch.nn.functional.gelu(a32).sum().backward()
    _close(ops.gemm(x, w, aux=aux, dgelu=True), base * a32.grad, tol, "dgelu")
    cs = torch.zeros(N, device="cuda")
    ops.gemm(x, w, bias=bias, colsum=cs)
    _close(cs[None], (base + bias.float()).sum(0)[None], 1e-4, "colsum")
    acc = torch.randn(M, N, device="cuda")
    acc0 = acc.clone()
    ops.gemm(x, w, out=acc, accumulate=True)
    _close(acc, base + acc0, 1e-5, "fp32 accumulate")
    acc = torch.randn(M, N, device="cuda").to(dtype)
    acc0 = acc.clone()
    ops.gemm(x, w, out=acc, accumulate=True)
    _close(acc, base + acc0.float(), tol, "16-bit accumulate")


def test_gemm_dropout_is_deterministic_and_unbiased():
    from uniter_b200 import ops
    torch.manual_seed(2)
    M, N, K = 1024, 768, 256
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    a = ops.gemm(x, w, dropout_p=0.1, rng_seed=5, rng_stream=1)
    b = ops.gemm(x, w, dropout_p=0.1, rng_seed=5, rng_stream=1)
    c = ops.gemm(x, w, dropout_p=0.1, rng_seed=5, rng_stream=2)
    assert torch.equal(a, b)
    assert (a != c).float().mean().item() > 0.1
    frac = (a == 0).float().mean().item()
    assert abs(frac - 0.1) < 5e-3, frac
    ref = (x.float() @ w.float().t()) / 0.9
    kept = a != 0
    assert ((a.float() - ref).abs() * kept).max().item() < 0.05


def test_gemm_rejects_bad_arguments():
    from uniter_b200 import ops
    x = torch.randn(16, 60, device="cuda").bfloat16()   # pitch 60 is not a multiple of 8
    w = torch.randn(16, 60, device="cuda").bfloat16()
    with pytest.raises(RuntimeError):
        ops.gemm(x, w)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("tn", [0, 128, 192, 256])
def test_grouped_wgrad_matches_separate_gemms(dtype, accumulate, tn):
    """ub200_gemm_grouped: the four weight-gradient shapes of a base layer in one launch."""
    import ctypes as C
    from uniter_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(3)
    T, H, I = 1237, 768, 3072
    probs = [(H, I), (I, H), (3 * H, H), (H, H)]           # (M, N) of dW2, dW1, dWqkv, dWo
    args = (_lib.GemmArgs * 4)()
    keep, refs, outs = [], [], []
    for i, (M, N) in enumerate(probs):
        a = (torch.randn(T, M, device="cuda") * 0.1).to(dtype)
        b = torch.randn(T, N, device="cuda").to(dtype)
        out = (torch.randn(M, N, device="cuda") * 0.5).to(dtype) if accumulate else \
            torch.empty(M, N, device="cuda", dtype=dtype)
        ref = a.float().t() @ b.float() + (out.float() if accumulate else 0)
        keep += [a, b]; outs.append(out); refs.append(ref)
        args[i] = _lib.GemmArgs(a=a.data_ptr(), b=b.data_ptr(), lda=M, ldb=N, a_major=1, b_major=1,
                                M=M, N=N, K=T, dtype=_lib.dtype_code(dtype),
                                epilogue=_lib.EPI_ACCUM if accumulate else 0, out=out.data_ptr(), ldo=N,
                                tile_n=tn)
    _lib.check(lib.ub200_gemm_grouped(args, 4, _lib.current_stream()))
    torch.cuda.synchronize()
    for out, ref in zip(outs, refs):
        _close(out, ref, TOL[dtype], "grouped wgrad")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape,splits", [((190, 768, 28996), -1), ((190, 768, 28996), 7), ((64, 128, 1000), 3),
                                          ((300, 256, 200), 16), ((130, 64, 64), -1)])
def test_gemm_split_k_atomic(dtype, shape, splits):
    """Few output tiles, long K (the MLM decoder's dgrad, K = vocabulary): K slices run as
    independent work units and meet through fp32 atomics; K tails are zero-filled by TMA."""
    from uniter_b200 import ops
    M, N, K = shape
    torch.manual_seed(M + K)
    Kp = (K + 7) // 8 * 8
    x = torch.zeros(M, Kp, device="cuda", dtype=dtype)[:, :K]
    x.copy_((torch.randn(M, K, device="cuda") * 0.05).to(dtype))
    wt = (torch.randn(K, N, device="cuda") * 0.05).to(dtype)          # [K, N]: dgrad form
    ref = x.float() @ wt.float()
    out = ops.gemm(x, wt, b_major=1, k_splits=splits)
    assert out.dtype == torch.float32
    _close(out, ref, 2e-3, "split-K dgrad form")
    w = wt.t().contiguous()
    wp = torch.zeros(N, Kp, device="cuda", dtype=dtype)[:, :K]
    wp.copy_(w)
    _close(ops.gemm(x, wp, k_splits=splits), ref, 2e-3, "split-K K-major")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("M,V,K", [(190, 28996, 768), (5, 1001, 128), (300, 2004, 128)])
def test_gemm_n_valid_over_unpadded_weight(dtype, M, V, K):
    """N padded to a multiple of 8 over a weight that only has V rows (tied decoder [28996, H]):
    the padding columns see acc = 0 (+ bias), nothing past the weight is read into valid columns."""
    from uniter_b200 import ops
    torch.manual_seed(V)
    Vp = (V + 7) // 8 * 8
    x = torch.randn(M, K, device="cuda").to(dtype)
    w = (torch.randn(V, K, device="cuda") * 0.05).to(dtype)
    bias = torch.full((Vp,), -30000.0, device="cuda", dtype=dtype)
    bias[:V] = torch.randn(V, device="cuda").to(dtype)
    out = torch.empty(M, Vp, device="cuda", dtype=dtype)
    ops.gemm(x, w, bias=bias, out=out, n_valid=V)
    ref = x.float() @ w.float().t() + bias[:V].float()
    _close(out[:, :V], ref, TOL[dtype], "n_valid forward")
    if Vp != V:
        assert (out[:, V:] == bias[V:]).all()          # acc = 0 exactly, bias only
    # wgrad over the same padded buffer: A = out[:, :V] read MN-major with row pitch Vp
    z = torch.randn(M, K, device="cuda").to(dtype)
    d = (torch.randn(M, Vp, device="cuda") * 0.1).to(dtype)
    dv = d[:, :V]
    _close(ops.gemm(dv, z, a_major=1, b_major=1), dv.float().t() @ z.float(), TOL[dtype], "wgrad M = V")
