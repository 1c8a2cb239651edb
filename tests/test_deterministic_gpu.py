"""GPU: the fixed-order reductions of the deterministic mode (ub200_set_deterministic), site by site.

Each site runs at C2-like shapes with inputs spanning about 1e-4 .. 1e4, under several SM reserves
(which resize the SM-sized grids) and with all-zero rows appended (the dummy sequence of GraphedStep):
the outputs must be bit-identical, and match a float64 reference (or, where the order is fully
specified, a host replay of it bit for bit).  Where the default mode's bits depend on the grid (column
sums, LayerNorm backward, split-K, the attention bias flush), the test also shows that they do, so the
check would catch a nondeterministic form.  The default forms of the table scatter, the weighted column
sums and the sum of squares use a grid fixed by the shape; their atomics differ only with scheduling,
which no single run shows reliably, so those sites have no such check.
"""
import contextlib

import numpy as np
import pytest
import torch


pytestmark = pytest.mark.gpu

RESERVES = (0, 6, 38)


@contextlib.contextmanager
def deterministic(on=True):
    from uniter_b200 import _lib
    lib = _lib.load()
    prev = lib.ub200_set_deterministic(1 if on else 0)
    try:
        yield
    finally:
        lib.ub200_set_deterministic(prev)


@contextlib.contextmanager
def sm_reserve(n):
    from uniter_b200 import _lib
    lib = _lib.load()
    prev = lib.ub200_set_sm_reserve(n)
    try:
        yield
    finally:
        lib.ub200_set_sm_reserve(prev)


def _spread(shape, seed, dtype=torch.bfloat16):
    """Values of both signs whose magnitudes span about 1e-4 .. 1e4 (order-sensitive sums)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    mag = torch.pow(10.0, torch.rand(shape, generator=g, device="cuda") * 8 - 4)
    sign = torch.where(torch.rand(shape, generator=g, device="cuda") < 0.5, -1.0, 1.0)
    return (mag * sign).to(dtype)


def _across_geometries(fn, pad_fn=None):
    """fn() under every SM reserve (and pad_fn() under reserve 0): list of output tuples (cloned)."""
    outs = []
    for r in RESERVES:
        with sm_reserve(r):
            outs.append(tuple(t.clone() for t in fn()))
    if pad_fn is not None:
        outs.append(tuple(t.clone() for t in pad_fn()))
    torch.cuda.synchronize()
    return outs


def _all_equal(outs):
    return all(torch.equal(a, b) for o in outs[1:] for a, b in zip(outs[0], o))


def _distinct(outs, i=0):
    return len({o[i].float().cpu().numpy().tobytes() for o in outs})


def _c2_lens():
    from uniter_b200.synth import synth_batch
    b = synth_batch(64, 12, 28, 26, 46, 1234, mlm_prob=0.15)
    return [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]


# ------------------------------------------------------------------------------ per reduction site
def test_colsum_is_fixed_order():
    from uniter_b200 import ops
    T, N = 3451, 2304
    x = _spread((T, N), 1)
    xp = torch.cat([x, torch.zeros(127, N, device="cuda", dtype=x.dtype)])
    ref = x.double().sum(0)
    with deterministic():
        outs = _across_geometries(lambda: (ops.colsum(x),), lambda: (ops.colsum(xp),))
    assert _all_equal(outs)
    tol = 1e-6 * x.double().abs().sum(0) + 1e-6
    assert ((outs[0][0].double() - ref).abs() <= tol).all()
    with deterministic(False):
        default = _across_geometries(lambda: (ops.colsum(x),), lambda: (ops.colsum(xp),))
    assert _distinct(default) >= 2


@pytest.mark.parametrize("case", ["encoder", "front_end"])
def test_layernorm_backward_is_fixed_order(case):
    from uniter_b200 import ops
    T, H = 3451, 768
    x, dy = _spread((T, H), 2), _spread((T, H), 3)
    gamma = (torch.rand(H, device="cuda") + 0.5).to(torch.bfloat16)
    pad = torch.zeros(127, H, device="cuda", dtype=x.dtype)
    from oracle.philox import dropout_params, rand16
    x64, dy64 = x.double(), dy.double()
    mean = x64.mean(1, keepdim=True)
    xhat = (x64 - mean) / torch.sqrt(((x64 - mean) ** 2).mean(1, keepdim=True) + 1e-12)
    if case == "encoder":
        def run(xx, dd):
            _, dxd, dg, db, dbias = ops.layernorm_bwd(dd, xx, gamma, dropout_p=0.1, rng_seed=5, rng_stream=77)
            return dg, db, dbias, dxd[:T]
        g_eff, active = dy64, torch.ones(T, 1, device="cuda", dtype=torch.float64)
    else:
        kind = (torch.arange(T + 127, device="cuda", dtype=torch.int32) % 3 == 0).int()

        def run(xx, dd):
            _, _, dg, db, _ = ops.layernorm_bwd(dd, xx, gamma, row_kind=kind[:xx.shape[0]], kind=0,
                                                want_dbias=False, dropout_p=0.1, rng_seed=5, rng_stream=78,
                                                dropout_on_dy=True)
            return dg, db
        thr, inv_keep = dropout_params(0.1)       # y = dropout(LN(x)): the mask applies to dy
        keep = rand16(5, 78, np.arange(T * H, dtype=np.uint64)) >= thr
        keep = torch.from_numpy(keep.reshape(T, H)).cuda()
        g_eff = torch.where(keep, dy64 * inv_keep, torch.zeros_like(dy64))
        active = (kind[:T] == 0).double()[:, None]
    with deterministic():
        outs = _across_geometries(lambda: run(x, dy), lambda: run(torch.cat([x, pad]), torch.cat([dy, pad])))
    assert _all_equal(outs)
    terms = [g_eff * xhat * active, g_eff * active]
    if case == "encoder":
        terms.append(outs[0][3].double())          # the Linear bias gradient sums the 16-bit dx_drop
    for got, t in zip(outs[0], terms):
        ref = t.sum(0)
        assert ((got.double() - ref).abs() <= 1e-5 * t.abs().sum(0) + 1e-6).all()
    with deterministic(False):
        default = _across_geometries(lambda: run(x, dy))
    assert _distinct(default) >= 2


def test_attention_bias_gradient_is_fixed_order_and_long_sequences_are_refused():
    from uniter_b200 import ops
    lens = _c2_lens()
    T, heads, H = sum(lens), 12, 768

    def run(ls):
        Tn = sum(ls)
        cu = torch.tensor([0] + list(torch.tensor(ls).cumsum(0)), device="cuda", dtype=torch.int32)
        g = torch.Generator(device="cuda").manual_seed(6)
        qkv = torch.cat([(torch.randn(T, 3 * H, device="cuda", generator=g)).to(torch.bfloat16),
                         torch.zeros(Tn - T, 3 * H, device="cuda", dtype=torch.bfloat16)])
        dctx = torch.cat([_spread((T, H), 7), torch.zeros(Tn - T, H, device="cuda", dtype=torch.bfloat16)])
        ctx, lse = ops.attn_fwd(qkv, cu, 128, heads, dropout_p=0.1, rng_seed=3, rng_stream=9)
        dbias = torch.zeros(3 * H, device="cuda")
        dqkv = ops.attn_bwd(qkv, ctx, lse, dctx, cu, 128, heads, dropout_p=0.1, rng_seed=3, rng_stream=9,
                            dbias=dbias)
        return dqkv[:T], dbias
    with deterministic():
        outs = _across_geometries(lambda: run(lens), lambda: run(lens + [127]))
    assert _all_equal(outs)
    ref = outs[0][0].double().sum(0)
    assert ((outs[0][1].double() - ref).abs() <= 1e-6 * outs[0][0].double().abs().sum(0) + 1e-6).all()
    with deterministic(False):
        default = _across_geometries(lambda: run(lens))
    assert all(torch.equal(o[0], outs[0][0]) for o in default)   # dqkv: same kernels, same bits
    assert ((default[0][1].double() - ref).norm() <= 1e-2 * ref.norm()).item()
    assert _distinct(default, 1) >= 2                            # the default flush follows the grid
    # dQ of sequences longer than one key block has no fixed-order form: an error, not a silent fallback
    cu = torch.tensor([0, 200], device="cuda", dtype=torch.int32)
    qkv = torch.randn(200, 3 * H, device="cuda").to(torch.bfloat16)
    ctx, lse = ops.attn_fwd(qkv, cu, 200, heads)
    with deterministic(), pytest.raises(RuntimeError, match="deterministic"):
        ops.attn_bwd(qkv, ctx, lse, torch.randn_like(ctx), cu, 200, heads)


def test_gemm_bias_gradient_and_decoder_dgrad_are_fixed_order():
    from uniter_b200 import ops
    T, H, I = 3451, 768, 3072
    g = torch.Generator(device="cuda").manual_seed(4)
    dy = _spread((T, H), 4) * 1e-2
    w2 = (torch.randn(H, I, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    pre = torch.randn(T, I, device="cuda", generator=g).to(torch.bfloat16)

    def ffn(pad):
        z = lambda n: torch.zeros(pad, n, device="cuda", dtype=torch.bfloat16)   # noqa: E731
        db1 = torch.zeros(I, device="cuda")
        d = ops.gemm(torch.cat([dy, z(H)]), w2, b_major=1, dgelu=True, aux=torch.cat([pre, z(I)]), colsum=db1)
        return d[:T], db1
    # MLM decoder dgrad: K = vocab, M = masked tokens (k_splits=-1: split-K over the SMs by default)
    V, M = 28996, 448
    dl = _spread((M, V + 4), 5) * 1e-3
    word = (torch.randn(V, H, device="cuda", generator=g) * 0.02).to(torch.bfloat16)

    def decoder():
        return (ops.gemm(dl[:, :V], word, b_major=1, k_splits=-1),)
    with deterministic():
        outs = _across_geometries(lambda: ffn(0), lambda: ffn(127))
        dec = _across_geometries(decoder)
    assert _all_equal(outs) and _all_equal(dec)
    d16 = outs[0][0].double()
    assert ((outs[0][1].double() - d16.sum(0)).abs() <= 1e-5 * d16.abs().sum(0) + 1e-6).all()
    ref = dl[:, :V].double() @ word.double()
    assert ((dec[0][0].double() - ref).abs() <= 1e-5 * (dl[:, :V].double().abs() @ word.double().abs()) + 1e-6).all()
    with deterministic(False):
        default_dec = _across_geometries(decoder)
        default_ffn = ffn(0)
    assert _distinct(default_dec) >= 2                 # the default split count follows the SM count
    assert torch.equal(default_ffn[0], outs[0][0])     # the dGELU dgrad itself has no cross-CTA sum
    assert ((default_ffn[1].double() - outs[0][1].double()).norm() <= 1e-2 * outs[0][1].double().norm()).item()


def _embed_rows(T, seed):
    """Packed rows of a C2-like batch: kind (0 text / 1 image), word ids drawn with heavy repetition
    (some ids occur hundreds of times, far apart), position ids, type ids, image source rows."""
    g = torch.Generator().manual_seed(seed)
    kind = (torch.rand(T, generator=g) < 0.55).int()
    word = torch.where(torch.rand(T, generator=g) < 0.5, torch.randint(0, 40, (T,), generator=g),
                       torch.randint(0, 28996, (T,), generator=g)).int()
    pos = torch.randint(0, 40, (T,), generator=g).int()
    typ = torch.randint(0, 2, (T,), generator=g).int()
    img_src = torch.where(kind == 1, torch.arange(T), torch.full((T,), -1)).int()
    return kind, word, pos, typ, img_src


def test_embedding_table_scatter_is_fixed_order():
    """Each id's text rows are summed in ascending row order in fp32 and added once to the table row,
    which already holds the tied decoder's weight gradient: replayed on the host bit for bit."""
    import ctypes as C
    from uniter_b200 import _lib
    lib = _lib.load()
    T, H, V, P = 3451, 768, 28996, 512
    kind, word, pos, _, _ = _embed_rows(T, 8)
    du = _spread((T, H), 9)
    init = (torch.randn(V, H, device="cuda") * 0.01).to(torch.bfloat16)     # tied decoder wgrad

    def run(n_pad):
        k = torch.cat([kind, torch.zeros(n_pad, dtype=torch.int32)]).cuda()
        w = torch.cat([word, torch.full((n_pad,), 7, dtype=torch.int32)]).cuda()
        ps = torch.cat([pos, torch.zeros(n_pad, dtype=torch.int32)]).cuda()
        d = torch.cat([du, torch.zeros(n_pad, H, device="cuda", dtype=du.dtype)])
        dw, dp = init.clone(), torch.zeros(P, H, device="cuda")
        _lib.check(lib.ub200_embed_bwd_scatter(d.data_ptr(), k.data_ptr(), w.data_ptr(), ps.data_ptr(),
                                               dw.data_ptr(), dp.data_ptr(), T + n_pad, H, _lib.BF16,
                                               C.c_void_p(_lib.current_stream())))
        return dw, dp
    with deterministic():
        outs = _across_geometries(lambda: run(0), lambda: run(127))
    assert _all_equal(outs)

    def ordered_sums(ids, nrows):
        """fp32 sums of the text rows of every id, row by row in ascending order (the kernel's order)."""
        text = (kind == 0).nonzero().flatten()
        dut = du.float().cpu()[text]
        idt = ids[text].long()
        acc = torch.zeros(nrows, H)
        order = torch.argsort(idt * T + text, stable=True)      # by id, then row
        idt, dut = idt[order], dut[order]
        first = torch.ones_like(idt, dtype=torch.bool)
        first[1:] = idt[1:] != idt[:-1]
        rank = torch.arange(len(idt)) - torch.cummax(torch.where(first, torch.arange(len(idt)), 0), 0)[0]
        for r in range(int(rank.max()) + 1):                     # r-th row of every id, in order
            sel = rank == r
            acc[idt[sel]] += dut[sel]
        return acc, torch.unique(idt)
    acc_w, ids_w = ordered_sums(word, V)
    want_w = init.float().cpu().clone()
    want_w[ids_w] = (want_w[ids_w] + acc_w[ids_w]).to(torch.bfloat16).float()
    assert torch.equal(outs[0][0].float().cpu(), want_w)
    acc_p, _ = ordered_sums(pos, P)
    assert torch.equal(outs[0][1].cpu(), acc_p)
    # and against float64
    ref = torch.zeros(V, H, dtype=torch.float64).index_add_(0, word[kind == 0].long(), du.double().cpu()[kind == 0])
    err = (outs[0][0].double().cpu() - init.double().cpu() - ref).abs()
    assert (err <= 2 ** -7 * (init.double().cpu() + ref).abs() + 1e-6).all()


def test_weighted_column_sums_are_fixed_order():
    import ctypes as C
    from uniter_b200 import _lib
    lib = _lib.load()
    T, H = 3451, 768
    kind, _, _, typ, img_src = _embed_rows(T, 10)
    x = _spread((T, H), 11)
    feat = torch.rand(T, 7, device="cuda") * 2 - 0.5

    def run(mode, n_pad):
        xx = torch.cat([x, torch.zeros(n_pad, H, device="cuda", dtype=x.dtype)])
        ty = torch.cat([typ, torch.zeros(n_pad, dtype=torch.int32)]).cuda()
        kd = torch.cat([kind, torch.ones(n_pad, dtype=torch.int32)]).cuda()
        src = torch.cat([img_src, torch.zeros(n_pad, dtype=torch.int32)]).cuda()
        out = torch.zeros(2, H, device="cuda") if mode == 0 else torch.zeros(H, 7, device="cuda")
        a = _lib.EmbedColsumArgs(x=xx.data_ptr(), type_id=ty.data_ptr(), kind=kd.data_ptr(), img_src=src.data_ptr(),
                                 pos_feat=feat.data_ptr(), out=out.data_ptr(), T=T + n_pad, hidden=H, mode=mode,
                                 type_vocab=2, dtype=_lib.BF16)
        _lib.check(lib.ub200_embed_bwd_colsums(C.byref(a), C.c_void_p(_lib.current_stream())))
        return (out,)
    x64 = x.double()
    w = feat.to(torch.bfloat16).double()
    img = (kind == 1).cuda()
    for mode in (0, 1):
        with deterministic():
            outs = _across_geometries(lambda: run(mode, 0), lambda: run(mode, 127))
        assert _all_equal(outs)
        if mode == 0:
            oh = torch.nn.functional.one_hot(typ.long().cuda(), 2).double()
            ref, mag = oh.t() @ x64, oh.t() @ x64.abs()
        else:
            ref, mag = x64[img].t() @ w[img], x64[img].abs().t() @ w[img].abs()
        assert ((outs[0][0].double() - ref).abs() <= 1e-5 * mag + 1e-6).all()


def test_gradient_sum_of_squares_is_fixed_order():
    from uniter_b200.optim import FusedAdamW
    shapes = [(28996, 768), (3072, 768), (768,), (2304,)]
    params = []
    for i, sh in enumerate(shapes):
        p = torch.nn.Parameter(torch.zeros(sh, device="cuda", dtype=torch.bfloat16))
        p.grad = _spread(sh, 20 + i) * 1e-2
        params.append(p)
    opt = FusedAdamW(params, lr=1e-3)
    ref = sum((p.grad.double() ** 2).sum() for p in params)
    with deterministic():
        outs = []
        for r in RESERVES:
            with sm_reserve(r):
                opt.step(max_grad_norm=1.0)
                outs.append((opt.last_sumsq.clone(),))
    torch.cuda.synchronize()
    assert _all_equal(outs)
    assert abs(outs[0][0].item() - ref.item()) <= 1e-5 * ref.item()
