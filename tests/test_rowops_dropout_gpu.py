"""GPU: the LayerNorm kernels (csrc/rowops.cu) and the embedding front-end kernels (csrc/embed.cu)
against float64 references, with every dropout mask replayed on the host (tests/rowops_check.py),
and the dropout masks of the GEMM epilogue, the LayerNorm backward and the embedding rows against
the host mirror bit for bit, down to p = 1e-6 where the threshold clamps to 1."""
import contextlib
import ctypes as C
import functools

import pytest
import torch

from oracle import encoder_oracle as orc
from tests import rowops_check as rc
from tests.test_gemm_epilogue_overlap_gpu import TILES

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
SEED = (0x5EED << 32) | 0x1234567
STREAM = (7 << 20) | (0xFFFF << 4) | 2
MASK_PS = [1e-6, 0.1, 0.5, 0.9999]


@functools.lru_cache(maxsize=None)
def _keep(p, rows, ncols, counter=None, seed=SEED, stream=STREAM):
    return rc.keep_mask(seed, stream, p, rows, ncols, "cuda", counter)


@contextlib.contextmanager
def _form(form):
    """LayerNorm backward forms: the fused one-pass kernel, the split row + column kernels
    (stats workspace), and the fixed-order kernels of the deterministic mode."""
    if form != "deterministic":
        yield form == "split"
        return
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield False
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ----------------------------------------------------------------------------- LayerNorm forward
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [1, 7, 3451])
@pytest.mark.parametrize("H", [128, 264, 768, 1024])
def test_layernorm_fwd_against_float64(H, rows, dtype):
    from uniter_b200 import ops
    g = _gen(H * 10 + rows)
    x = torch.randn(rows, H, device="cuda", generator=g) * 2 + 0.3
    x[::3] += 100.0                                           # rows with |mean| >> std
    x = x.to(dtype)
    gamma = (1 + 0.1 * torch.randn(H, device="cuda", generator=g)).to(dtype)
    beta = (0.1 * torch.randn(H, device="cuda", generator=g)).to(dtype)
    y = ops.layernorm_fwd(x, gamma, beta)
    fails, stats = rc.check_rows("y", y, rc.ln_fwd_reference(x, gamma, beta), rc.ln_fwd_baseline(x, gamma, beta),
                                 dtype)
    assert not fails, (fails, stats)


# ----------------------------------------------------------------------------- LayerNorm backward
LN_CASES = {
    # name: (dropout p, dropout on dy, kind (None: no row kind), zero_inactive, dbias, device offset)
    "plain": (0.0, False, None, False, True, None),
    "dropout_dx": (0.1, False, None, False, True, None),
    "dropout_dy_kind0": (0.1, True, 0, False, False, None),
    "dropout_dy_kind1_zero_inactive": (0.1, True, 1, True, True, None),
    "kind1_zero_inactive": (0.0, False, 1, True, True, None),
    "dropout_dx_device_offset": (0.1, False, None, False, True, 5),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H", [128, 264, 768, 1024])
@pytest.mark.parametrize("case", list(LN_CASES))
@pytest.mark.parametrize("form", ["fused", "split", "deterministic"])
def test_layernorm_bwd_against_float64(form, case, H, dtype):
    from uniter_b200 import ops
    p, on_dy, kind, zero_inactive, want_dbias, counter = LN_CASES[case]
    rows = 3451
    g = _gen(H + rows + len(case))
    x = (torch.randn(rows, H, device="cuda", generator=g) * 2 + 0.3).to(dtype)
    gamma = (1 + 0.1 * torch.randn(H, device="cuda", generator=g)).to(dtype)
    dy = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    init = [torch.randn(H, device="cuda", generator=g) for _ in range(3)]   # accumulated onto
    row_kind = (torch.randint(0, 2, (rows,), device="cuda", generator=g, dtype=torch.int32)
                if kind is not None else None)
    sentinel = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    keep, inv = _keep(p, rows, H, counter) if p else (None, 1.0)
    off = torch.tensor([counter], device="cuda", dtype=torch.int64) if counter is not None else None

    dx, dgamma, dbeta, dbias = sentinel.clone(), init[0].clone(), init[1].clone(), init[2].clone()
    with _form(form) as split:
        _, dx_drop, _, _, _ = ops.layernorm_bwd(
            dy, x, gamma, dropout_p=p, rng_seed=SEED, rng_stream=STREAM, row_kind=row_kind, kind=kind or 0,
            dropout_on_dy=on_dy, dx=dx, dgamma=dgamma, dbeta=dbeta, dbias=dbias if want_dbias else None,
            want_dbias=want_dbias, zero_inactive=zero_inactive,
            rng_offset_dev=off.data_ptr() if off is not None else None, split=split)
    torch.cuda.synchronize()
    dx0 = None if (kind is None or zero_inactive) else sentinel
    ref = rc.ln_bwd_reference(dy, x, gamma, keep, inv, on_dy, row_kind, kind or 0, dx0, init[0], init[1],
                              init[2] if want_dbias else None)
    act = ref["active"]
    base = rc.ln_bwd_baseline(dy[act], x[act], gamma, keep[act] if keep is not None else None, inv, on_dy)
    out = dict(dx=dx, dx_drop=dx_drop, dgamma=dgamma, dbeta=dbeta, dbias=dbias if want_dbias else None)
    fails = rc.check_ln_bwd(out, ref, base, dtype, dx0=dx0, dgamma0=init[0], dbeta0=init[1],
                            dbias0=init[2] if want_dbias else None)
    assert not fails, fails


# ----------------------------------------------------------------------------- mask identity
def _gemm_operands(M, N, K, dtype, seed):
    g = _gen(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.1).to(dtype)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).to(dtype)
    return a, w, bias


@pytest.mark.parametrize("p", MASK_PS)
@pytest.mark.parametrize("N", [768, 200])
def test_gemm_dropout_mask_is_the_host_mirror(N, p):
    """For every (tile_n, cluster): the fp32 output at p is the kernel's own p = 0 output times
    inv_keep where the host mirror keeps, and 0 where it drops; the 16-bit output with a zero
    residual is that value rounded."""
    from uniter_b200 import ops
    M, K, dtype = 3451, 64, torch.bfloat16
    a, w, bias = _gemm_operands(M, N, K, dtype, N)
    keep, inv = _keep(p, M, N)
    zero = torch.zeros(M, N, device="cuda", dtype=dtype)
    for bn, c in TILES:
        kw = dict(bias=bias, tile_n=bn, cluster=c, k_splits=1)
        v = ops.gemm(a, w, out_fp32=True, **kw)
        want = torch.where(keep, v * inv, torch.zeros_like(v))
        d32 = ops.gemm(a, w, out_fp32=True, dropout_p=p, rng_seed=SEED, rng_stream=STREAM, **kw)
        d16 = ops.gemm(a, w, residual=zero, dropout_p=p, rng_seed=SEED, rng_stream=STREAM, **kw)
        what = "tile_n %d cluster %d p %g: " % (bn, c, p)
        assert torch.equal(d32 != 0, keep), what + "%d mask elements differ from the host mirror" % int(
            ((d32 != 0) != keep).sum())
        assert torch.equal(d32, want), what + "kept values are not v * inv_keep"
        assert torch.equal(d16, want.to(dtype)), what + "16-bit output"


@pytest.mark.parametrize("p", MASK_PS)
@pytest.mark.parametrize("form", ["fused", "split", "deterministic"])
def test_layernorm_bwd_dropout_mask_is_the_host_mirror(form, p):
    from uniter_b200 import ops
    rows, H, dtype = 3451, 768, torch.bfloat16
    g = _gen(11)
    x = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    dy = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    gamma = (1 + 0.1 * torch.randn(H, device="cuda", generator=g)).to(dtype)
    keep, inv = _keep(p, rows, H)
    with _form(form) as split:
        dx, dxd, _, _, _ = ops.layernorm_bwd(dy, x, gamma, dropout_p=p, rng_seed=SEED, rng_stream=STREAM,
                                             split=split)
    nz = dx != 0
    assert torch.equal((dxd != 0) & nz, keep & nz), "%d mask elements differ from the host mirror" % int(
        (((dxd != 0) != keep) & nz).sum())
    want = dx.float() * inv * keep
    assert ((dxd.float() - want).abs() <= 2 ** -6 * want.abs()).all()


# ----------------------------------------------------------------------------- embedding kernels
def _embed_inputs(T, H, dtype, seed, V=300, P=64, n_box=500):
    """Front-end parameters (16-bit, keyed like UniterModel.state_dict()) and per-row inputs of
    ub200_embed_rows_fwd: about half text rows, half image rows."""
    from uniter_b200.synth import seeded_state, uniter_state_shapes
    st = seeded_state(uniter_state_shapes(H, 0, 4, V, P, 2, 8), seed=seed)
    st = {k: v.to("cuda", dtype) for k, v in st.items()
          if k.startswith("embeddings.") or k.startswith("img_embeddings.")}
    g = _gen(seed)
    kind = torch.randint(0, 2, (T,), device="cuda", generator=g, dtype=torch.int32)
    rows = dict(kind=kind,
                word_id=torch.randint(0, V, (T,), device="cuda", generator=g, dtype=torch.int32) * (kind == 0),
                pos_id=torch.randint(0, P, (T,), device="cuda", generator=g, dtype=torch.int32) * (kind == 0),
                type_id=torch.randint(0, 2, (T,), device="cuda", generator=g, dtype=torch.int32),
                img_src=torch.where(kind == 1, torch.randint(0, n_box, (T,), device="cuda", generator=g,
                                                             dtype=torch.int32), -1).to(torch.int32))
    G = torch.randn(T, H, device="cuda", generator=g).to(dtype)
    box = torch.rand(n_box, 7, device="cuda", generator=g)
    return st, rows, G, box


def _embed_rows(st, rows, G, box, p, counter=None):
    from uniter_b200 import _lib
    lib = _lib.load()
    T, H = G.shape
    x, u, ppre = (torch.empty_like(G) for _ in range(3))
    off = torch.tensor([counter], device="cuda", dtype=torch.int64) if counter is not None else None

    def ptr(k):
        return st[k].contiguous().data_ptr()
    r = _lib.EmbedRowsArgs(
        kind=rows["kind"].data_ptr(), word_id=rows["word_id"].data_ptr(), pos_id=rows["pos_id"].data_ptr(),
        type_id=rows["type_id"].data_ptr(), img_src=rows["img_src"].data_ptr(),
        word_emb=ptr("embeddings.word_embeddings.weight"), pos_emb=ptr("embeddings.position_embeddings.weight"),
        type_emb=ptr("embeddings.token_type_embeddings.weight"),
        ln_txt_g=ptr("embeddings.LayerNorm.weight"), ln_txt_b=ptr("embeddings.LayerNorm.bias"),
        img_linear_out=G.data_ptr(), pos_feat=box.data_ptr(),
        w_pos=ptr("img_embeddings.pos_linear.weight"), b_pos=ptr("img_embeddings.pos_linear.bias"),
        ln_img_g=ptr("img_embeddings.img_layer_norm.weight"), ln_img_b=ptr("img_embeddings.img_layer_norm.bias"),
        ln_pos_g=ptr("img_embeddings.pos_layer_norm.weight"), ln_pos_b=ptr("img_embeddings.pos_layer_norm.bias"),
        ln_out_g=ptr("img_embeddings.LayerNorm.weight"), ln_out_b=ptr("img_embeddings.LayerNorm.bias"),
        x=x.data_ptr(), u=u.data_ptr(), ppre=ppre.data_ptr(), T=T, hidden=H, dtype=_lib.dtype_code(G.dtype),
        dropout_p=float(p), rng_seed=SEED, rng_stream=STREAM,
        rng_offset_dev=off.data_ptr() if off is not None else None)
    _lib.check(lib.ub200_embed_rows_fwd(C.byref(r), _lib.current_stream()))
    torch.cuda.synchronize()
    return dict(x=x, u=u, ppre=ppre)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H", [128, 768, 1024])
@pytest.mark.parametrize("p,counter", [(0.0, None), (0.1, None), (0.1, 9)])
def test_embed_rows_fwd_against_float64(p, counter, H, dtype):
    T = 3451
    st, rows, G, box = _embed_inputs(T, H, dtype, seed=H)
    out = _embed_rows(st, rows, G, box, p, counter)
    keep, inv = _keep(p, T, H, counter) if p else (None, 1.0)
    box16 = box.to(dtype)                                     # the kernel rounds the boxes to the model dtype
    ref = rc.embed_rows_reference(st, rows, G, box16, keep, inv)
    base = rc.embed_rows_reference(st, rows, G, box16, keep, inv, dtype=dtype)
    fails = []
    for n in ("x", "u", "ppre"):
        fails += rc.check_rows(n, out[n], ref[n], base[n], dtype)[0]
    fails += rc.check_exact("ppre (text rows)", out["ppre"][rows["kind"] == 0],
                            torch.zeros_like(out["ppre"][rows["kind"] == 0]))
    assert not fails, fails


@pytest.mark.parametrize("p", MASK_PS)
def test_embed_rows_dropout_mask_is_the_host_mirror(p):
    """x at p = the kernel's own p = 0 output times inv_keep (in fp32, rounded) where the host
    mirror keeps, 0 where it drops."""
    T, H, dtype = 3451, 768, torch.bfloat16
    st, rows, G, box = _embed_inputs(T, H, dtype, seed=5)
    x0 = _embed_rows(st, rows, G, box, 0.0)["x"]
    x = _embed_rows(st, rows, G, box, p)["x"]
    keep, inv = _keep(p, T, H)
    nz = x0 != 0
    assert torch.equal((x != 0) & nz, keep & nz), "%d mask elements differ from the host mirror" % int(
        (((x != 0) != keep) & nz).sum())
    assert torch.equal(x, torch.where(keep, x0.float() * inv, torch.zeros_like(x0.float())).to(dtype))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("feat_dtype", ["fp32", "16bit"])
@pytest.mark.parametrize("D", [64, 2048])
def test_embed_gather_cast_bit_exact(D, feat_dtype, dtype):
    """out[t] = 16-bit(feat[img_src[t]]), + the mask row after rounding where mask_flag[t], and zeros
    for text rows (img_src = -1)."""
    from uniter_b200 import _lib
    lib = _lib.load()
    T, n = 1001, 300
    g = _gen(D)
    feat = torch.randn(n, D, device="cuda", generator=g) * 3
    if feat_dtype == "16bit":
        feat = feat.to(dtype)
    img_src = torch.randint(-1, n, (T,), device="cuda", generator=g, dtype=torch.int32)
    mask_flag = torch.randint(0, 2, (T,), device="cuda", generator=g, dtype=torch.int32)
    mask_row = torch.randn(D, device="cuda", generator=g).to(dtype)
    out = torch.full((T, D), float("nan"), device="cuda", dtype=dtype)
    _lib.check(lib.ub200_embed_gather_cast(feat.data_ptr(), 1 if feat.dtype == torch.float32 else 0,
                                           img_src.data_ptr(), mask_flag.data_ptr(), mask_row.data_ptr(),
                                           out.data_ptr(), T, D, _lib.dtype_code(dtype), _lib.current_stream()))
    f16 = feat[img_src.clamp(min=0).long()].to(dtype)
    masked = (f16.float() + mask_row.float()).to(dtype)
    want = torch.where((mask_flag != 0)[:, None], masked, f16)
    want = torch.where((img_src >= 0)[:, None], want, torch.zeros_like(want))
    assert not rc.check_exact("gather_cast", out, want)


# ----------------------------------------------------------------------------- front-end, train mode
FRONT_GRADS = ["embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
               "embeddings.token_type_embeddings.weight", "embeddings.LayerNorm.weight", "embeddings.LayerNorm.bias",
               "img_embeddings.img_linear.weight", "img_embeddings.img_linear.bias",
               "img_embeddings.img_layer_norm.weight", "img_embeddings.img_layer_norm.bias",
               "img_embeddings.pos_layer_norm.weight", "img_embeddings.pos_layer_norm.bias",
               "img_embeddings.pos_linear.weight", "img_embeddings.pos_linear.bias",
               "img_embeddings.mask_embedding.weight",
               "img_embeddings.LayerNorm.weight", "img_embeddings.LayerNorm.bias"]


def _front_reference(state, b, img_masks, txt_type, img_type, pack_idx, keep, inv, dtype):
    """Packed, dropped-out front-end rows [T, H] in `dtype` from leaf parameters `state`, and the
    taps of the sums before the text and image LayerNorms (model inputs as the kernels read them:
    features and boxes rounded to the model dtype)."""
    tt, it = {}, {}
    txt = orc.text_embeddings(state, b["input_ids"], b["position_ids"], txt_type, taps=tt)
    img = orc.image_embeddings(state, b["img_feat16"].to(dtype), b["img_pos_feat16"].to(dtype), img_type,
                               img_masks, taps=it)
    emb = orc.gather_embeddings(txt, img, b["gather_index"])
    x = emb.reshape(-1, emb.size(-1))[pack_idx.long()]
    return orc.dropout(x, keep, inv), tt["u"], it["u"], it["ppre"]


def test_front_end_train_mode_gradients_against_float64():
    """_EmbedFront at C2 shapes (64 samples, 3451 tokens, H = 768, img_dim 2048) with dropout 0.1,
    img_masks and custom type ids: the output and every front-end parameter gradient of a random
    projection, against float64 autograd of the oracle under the replayed mask.  Stated magnitudes:
    the table gradients are sums over rows (the word table's with 16-bit atomics), so theirs is the
    sum of |terms| per table row; pos_linear.weight's is a column sum over the image rows, bounded
    like attn_check's bias gradient."""
    from tests import util
    from uniter_b200 import model as um
    from uniter_b200.synth import synth_batch
    dtype, p = torch.bfloat16, 0.1
    cfg = dict(util.BASE_L1)
    state = util.make_state(cfg, seed=4)
    model = util.make_model(cfg, state, dtype).train()
    batch = synth_batch(64, 12, 28, 26, 46, 1234, img_dim=cfg["img_dim"], vocab_size=cfg["vocab_size"])
    b = util.batch_to(batch, "cuda")
    g = torch.Generator().manual_seed(8)
    B, Lt = b["input_ids"].shape
    Li = b["img_feat"].size(1)
    nbb = torch.tensor(batch["num_bbs"])
    img_masks = ((torch.rand(B, Li, generator=g) < 0.15) & (torch.arange(Li)[None] < nbb[:, None])).cuda()
    txt_type = torch.randint(0, 2, (B, Lt), generator=g).cuda()
    img_type = torch.randint(0, 2, (B, Li), generator=g).cuda()
    meta = model._pack_meta(b["attn_masks"])
    T, H = meta["total"], cfg["hidden_size"]
    assert T == 3451
    model.embeddings.dropout.p = model.img_embeddings.dropout.p = p
    model._weight_table()
    anchor = torch.zeros(1, device="cuda", requires_grad=True)
    x = um._EmbedFront.apply(anchor, model, meta, 0, b["input_ids"], b["position_ids"], b["img_feat"],
                             b["img_pos_feat"], b["gather_index"], img_masks, txt_type, img_type, p)
    offset = um._rng_offset[0]
    seed = torch.cuda.initial_seed() & 0xFFFFFFFFFFFFFFFF
    keep, inv = rc.keep_mask(seed, (offset << 20) | (0xFFFF << 4) | 4, p, T, H, "cuda")
    R = torch.randn(T, H, generator=torch.Generator().manual_seed(9)).to(dtype).float().cuda()   # exact in dtype
    (x.float() * R).sum().backward()
    torch.cuda.synchronize()
    grads = {n: prm.grad for n, prm in model.named_parameters() if n in FRONT_GRADS}

    b["img_feat16"], b["img_pos_feat16"] = b["img_feat"].to(dtype), b["img_pos_feat"].to(dtype)
    sd = {k: v for k, v in model.state_dict().items() if k in FRONT_GRADS}
    res = {}
    for d in (torch.float64, dtype):
        st = {k: v.to(d).requires_grad_(True) for k, v in sd.items()}
        y, ut, ui, pp = _front_reference(st, b, img_masks, txt_type, img_type, meta["pack_idx"], keep, inv, d)
        for t in (ut, ui, pp):
            t.retain_grad()
        (y.double() * R.double()).sum().backward()
        res[d] = (y.detach(), {k: v.grad for k, v in st.items()}, ut.grad, ui.grad, pp.grad)
    (y64, g64, dut, dui, dpp), (y16, g16, _, _, _) = res[torch.float64], res[dtype]

    fails = rc.check_rows("x", x, y64, y16, dtype)[0]
    # stated magnitudes of the table gradients: per table row, the sum of |terms| that meet there
    ids = b["input_ids"].reshape(-1)
    pos = b["position_ids"].expand(B, Lt).reshape(-1)
    at = dut.abs().reshape(-1, H)
    ai = dui.abs().reshape(-1, H)
    mags = {"embeddings.word_embeddings.weight": torch.zeros_like(g64["embeddings.word_embeddings.weight"])
            .index_add_(0, ids, at),
            "embeddings.position_embeddings.weight": torch.zeros_like(g64["embeddings.position_embeddings.weight"])
            .index_add_(0, pos, at),
            "embeddings.token_type_embeddings.weight":
            torch.zeros_like(g64["embeddings.token_type_embeddings.weight"]).index_add_(0, txt_type.reshape(-1), at)
            .index_add_(0, img_type.reshape(-1), ai),
            # a column sum over the image rows (K = T): attn_check's bias-gradient rule,
            # 4 u sqrt(sum over rows of term^2)
            "img_embeddings.pos_linear.weight":
            2 * ((dpp ** 2).reshape(-1, H).t() @ (b["img_pos_feat16"].double() ** 2).reshape(-1, 7)).sqrt()}
    for n in FRONT_GRADS:
        ref, base, got = g64[n], g16[n], grads[n]
        assert got is not None, n
        v = (lambda t: t.reshape(-1, t.size(-1)) if t.dim() > 1 else t.reshape(1, -1))
        fails += rc.check_rows(n, v(got), v(ref), v(base), dtype, mag=v(mags[n]) if n in mags else None)[0]
    assert not fails, fails
