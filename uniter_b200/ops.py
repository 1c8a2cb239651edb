"""Thin Python wrappers over the C ABI (one function per ub200_* entry point).

These allocate outputs with torch (the ABI never allocates), pass raw pointers and launch on
torch's current CUDA stream.  No torch math happens here.
"""
import ctypes as C
import functools

import torch

from . import _lib
from ._lib import (EPI_ACCUM, EPI_ATOMIC, EPI_BIAS, EPI_COLSUM, EPI_DGELU, EPI_DROPOUT, EPI_GELU,
                   EPI_OUT_F32, EPI_RESIDUAL)


def _follows_torch(fn):
    """Launch in the mode _lib.select_mode() gives at the call: torch.use_deterministic_algorithms, or
    inside an autograd backward the mode of its forward."""
    @functools.wraps(fn)
    def call(*args, **kwargs):
        with _lib.library_mode(_lib.select_mode()):
            return fn(*args, **kwargs)
    return call


@_follows_torch
def gemm(a, b, *, a_major=0, b_major=0, bias=None, residual=None, aux=None, out=None,
         gelu=False, dgelu=False, accumulate=False, out_fp32=False, colsum=None,
         dropout_p=0.0, rng_seed=0, rng_stream=0, tile_n=0, max_ctas=0, cluster=0, k_splits=0,
         n_valid=0, rng_offset_dev=None, tanh=False):
    """D = epilogue(A . B^T) on the wgmma GEMM core.  Returns `out` (and pre-activation if gelu).

    a: [M,K] (a_major=0) or [K,M] (a_major=1);  b: [N,K] (b_major=0) or [K,N] (b_major=1).
    k_splits > 1 (or -1 = fill the SMs): split-K into a zero-initialised fp32 `out` through atomics.
    n_valid: b holds only n_valid of the N (= out.size(1)) output features; the rest get acc = 0.
    """
    lib = _lib.load()
    assert a.is_cuda and b.is_cuda and a.dtype == b.dtype
    assert a.stride(-1) == 1 and b.stride(-1) == 1
    if a_major == 0:
        M, K = a.shape
    else:
        K, M = a.shape
    if b_major == 0:
        N, Kb = b.shape
    else:
        Kb, N = b.shape
    assert K == Kb, "contraction mismatch %d vs %d" % (K, Kb)
    if n_valid:
        assert n_valid == N, "n_valid is the number of output features b really holds"
        N = out.size(1) if out is not None else (N + 7) // 8 * 8
    splitk = k_splits > 1 or k_splits == -1
    if out is None:
        if splitk:
            out = torch.zeros(M, N, device=a.device, dtype=torch.float32)
        else:
            out = torch.empty(M, N, device=a.device, dtype=torch.float32 if out_fp32 else a.dtype)
    # the kernel reads and writes [M, N] at the row pitches it is given: check every side tensor here,
    # before the launch, rather than let it touch memory outside them
    for name, t, dt in (("out", out, None), ("residual", residual, a.dtype), ("aux", aux, a.dtype)):
        if t is not None:
            assert tuple(t.shape) == (M, N) and t.stride(1) == 1 and t.device == a.device, \
                "%s must be [%d, %d] with unit column stride, got %s / %s" % (name, M, N, tuple(t.shape), t.stride())
            assert dt is None or t.dtype == dt, "%s must be %s, got %s" % (name, dt, t.dtype)
    assert out.dtype in (a.dtype, torch.float32), "out must be %s or float32, got %s" % (a.dtype, out.dtype)
    assert bias is None or (bias.numel() == N and bias.dtype == a.dtype and bias.is_contiguous()), \
        "bias must hold %d contiguous %s elements" % (N, a.dtype)
    # out2 has out's row pitch (include/ub200.h): the kernel stores it at row * ldo + col
    out2 = torch.empty(M, out.stride(0), device=a.device, dtype=a.dtype)[:, :N] if gelu else None
    epi = 0
    if bias is not None:
        epi |= EPI_BIAS
    if dropout_p > 0:
        epi |= EPI_DROPOUT
    if residual is not None:
        epi |= EPI_RESIDUAL
    if gelu:
        epi |= EPI_GELU
    if tanh:
        epi |= _lib.EPI_TANH
    if dgelu:
        epi |= EPI_DGELU
    if accumulate:
        epi |= EPI_ACCUM
    if out.dtype == torch.float32:
        epi |= EPI_OUT_F32
    if colsum is not None:
        epi |= EPI_COLSUM
    if splitk:
        assert out.dtype == torch.float32 and epi == EPI_OUT_F32, "split-K: fp32 out, no other epilogue"
        epi |= EPI_ATOMIC
    args = _lib.GemmArgs(
        a=a.data_ptr(), b=b.data_ptr(), lda=a.stride(0), ldb=b.stride(0),
        a_major=a_major, b_major=b_major, M=M, N=N, K=K,
        dtype=_lib.dtype_code(a.dtype), epilogue=epi,
        bias=_lib.ptr(bias), residual=_lib.ptr(residual), aux=_lib.ptr(aux),
        out=out.data_ptr(), out2=_lib.ptr(out2), colsum=_lib.ptr(colsum),
        ldr=residual.stride(0) if residual is not None else 0,
        ldaux=aux.stride(0) if aux is not None else 0,
        ldo=out.stride(0),
        dropout_p=float(dropout_p), rng_seed=int(rng_seed), rng_stream=int(rng_stream),
        tile_n=int(tile_n), max_ctas=int(max_ctas), cluster=int(cluster), k_splits=int(k_splits),
        n_valid=int(n_valid), rng_offset_dev=rng_offset_dev)
    _lib.check(lib.ub200_gemm(C.byref(args), _lib.current_stream()))
    return (out, out2) if gelu else out


def _out_buffer(buf, shape, like, dtype):
    """`buf` checked as a contiguous output of `shape` / `dtype` on like's device, or a new one."""
    if buf is None:
        return torch.empty(shape, device=like.device, dtype=dtype)
    assert tuple(buf.shape) == tuple(shape) and buf.dtype == dtype and buf.is_contiguous() \
        and buf.device == like.device, "output buffer must be a contiguous %s %s" % (dtype, tuple(shape))
    return buf


@_follows_torch
def attn_fwd(qkv, cu_seqlens, max_seqlen, num_heads, dropout_p=0.0, rng_seed=0, rng_stream=0,
             rng_offset_dev=None, ctx=None, lse=None):
    """ctx [T, H], lse [heads, T] = fused varlen attention over packed qkv [T, 3H].
    ctx / lse: optional preallocated outputs (written, not accumulated into)."""
    lib = _lib.load()
    T, H3 = qkv.shape
    H = H3 // 3
    ctx = _out_buffer(ctx, (T, H), qkv, qkv.dtype)
    lse = _out_buffer(lse, (num_heads, T), qkv, torch.float32)
    a = _lib.AttnArgs(qkv=qkv.data_ptr(), ctx=ctx.data_ptr(), lse=lse.data_ptr(),
                      cu_seqlens=cu_seqlens.data_ptr(), batch=cu_seqlens.numel() - 1,
                      total_tokens=T, max_seqlen=max_seqlen, hidden=H, num_heads=num_heads,
                      dtype=_lib.dtype_code(qkv.dtype), dropout_p=float(dropout_p),
                      rng_seed=int(rng_seed), rng_stream=int(rng_stream), rng_offset_dev=rng_offset_dev)
    _lib.check(lib.ub200_attn_fwd(C.byref(a), _lib.current_stream()))
    return ctx, lse


def attn_bwd(qkv, ctx, lse, dctx, cu_seqlens, max_seqlen, num_heads, dropout_p=0.0, rng_seed=0,
             rng_stream=0, dbias=None, rng_offset_dev=None, dqkv=None):
    """dqkv [T, 3H] of attn_fwd; dbias [3H] fp32, if given, is accumulated into (column sums of dqkv).
    dqkv: optional preallocated output (written, not accumulated into).  Under
    torch.use_deterministic_algorithms, max_seqlen > 128 raises (warn_only: runs in the default mode)."""
    with _lib.library_mode(_lib.select_mode(max_seqlen)):
        return _attn_bwd(qkv, ctx, lse, dctx, cu_seqlens, max_seqlen, num_heads, dropout_p, rng_seed,
                         rng_stream, dbias, rng_offset_dev, dqkv)


def _attn_bwd(qkv, ctx, lse, dctx, cu_seqlens, max_seqlen, num_heads, dropout_p, rng_seed, rng_stream,
              dbias, rng_offset_dev, dqkv):
    lib = _lib.load()
    T, H3 = qkv.shape
    H = H3 // 3
    dqkv = _out_buffer(dqkv, (T, H3), qkv, qkv.dtype)
    ws_bytes = lib.ub200_attn_bwd_workspace_bytes(T, H, max_seqlen)
    ws = torch.empty(max(ws_bytes, 1), device=qkv.device, dtype=torch.uint8)
    a = _lib.AttnArgs(qkv=qkv.data_ptr(), ctx=ctx.data_ptr(), lse=lse.data_ptr(),
                      cu_seqlens=cu_seqlens.data_ptr(), batch=cu_seqlens.numel() - 1,
                      total_tokens=T, max_seqlen=max_seqlen, hidden=H, num_heads=num_heads,
                      dtype=_lib.dtype_code(qkv.dtype), dropout_p=float(dropout_p),
                      rng_seed=int(rng_seed), rng_stream=int(rng_stream),
                      dctx=dctx.data_ptr(), dqkv=dqkv.data_ptr(),
                      workspace=ws.data_ptr() if ws_bytes else None, dbias=_lib.ptr(dbias),
                      rng_offset_dev=rng_offset_dev)
    _lib.check(lib.ub200_attn_bwd(C.byref(a), _lib.current_stream()))
    return dqkv


@_follows_torch
def layernorm_fwd(x, gamma, beta, relu=False):
    """y = LayerNorm(x) (or LayerNorm(relu(x)) with relu) over rows of up to 2048 columns."""
    lib = _lib.load()
    rows, H = x.shape
    y = torch.empty_like(x)
    if relu:
        _lib.check(lib.ub200_layernorm_fwd_act(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
                                               rows, H, _lib.dtype_code(x.dtype), _lib.LN_ACT_RELU,
                                               _lib.current_stream()))
        return y
    _lib.check(lib.ub200_layernorm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
                                       rows, H, _lib.dtype_code(x.dtype), _lib.current_stream()))
    return y


@_follows_torch
def layernorm_bwd(dy, x, gamma, dropout_p=0.0, rng_seed=0, rng_stream=0, want_dbias=True,
                  row_kind=None, kind=0, dropout_on_dy=False, dx=None, dgamma=None, dbeta=None, dbias=None,
                  zero_inactive=False, rng_offset_dev=None, split=False, relu=False):
    """Returns dx, dx_drop (or None), dgamma, dbeta, dbias (fp32).  split=True: row kernel + column
    kernel (plain case only; in the deterministic mode every case is split).
    relu=True: x is `pre` of y = LayerNorm(relu(pre)); the second result is then dpre = dx o (pre > 0)
    and dbias its column sums (no dropout, no row kind).  Rows wider than 1024 and ReLU rows always
    take the split form."""
    lib = _lib.load()
    rows, H = x.shape
    if dx is None:
        dx = torch.empty_like(x) if row_kind is None else torch.zeros_like(x)
    dx_drop = torch.empty_like(x) if (relu or (dropout_p > 0 and not dropout_on_dy)) else None
    if dgamma is None:
        dgamma = torch.zeros(H, device=x.device, dtype=torch.float32)
    if dbeta is None:
        dbeta = torch.zeros(H, device=x.device, dtype=torch.float32)
    if dbias is None and want_dbias:
        dbias = torch.zeros(H, device=x.device, dtype=torch.float32)
    a = _lib.LnBwdArgs(dy=dy.data_ptr(), x=x.data_ptr(), gamma=gamma.data_ptr(), dx=dx.data_ptr(),
                       dx_drop=_lib.ptr(dx_drop), dgamma=dgamma.data_ptr(), dbeta=dbeta.data_ptr(),
                       dbias=_lib.ptr(dbias), rows=rows, hidden=H, dtype=_lib.dtype_code(x.dtype),
                       dropout_p=float(dropout_p), rng_seed=int(rng_seed), rng_stream=int(rng_stream),
                       row_kind=_lib.ptr(row_kind), kind=int(kind),
                       dropout_on_dy=(1 if dropout_on_dy else 0) | (2 if zero_inactive else 0),
                       rng_offset_dev=rng_offset_dev, act=_lib.LN_ACT_RELU if relu else _lib.LN_ACT_NONE)
    if split or relu or H > 1024 or _lib.deterministic():   # the deterministic mode always takes the split form
        ws = torch.empty(rows, 2, device=x.device, dtype=torch.float32)
        a.stats_ws = ws.data_ptr()
    _lib.check(lib.ub200_layernorm_bwd(C.byref(a), _lib.current_stream()))
    return dx, dx_drop, dgamma, dbeta, dbias


@_follows_torch
def colsum(x, out=None):
    lib = _lib.load()
    rows, N = x.shape
    if out is None:
        out = torch.zeros(N, device=x.device, dtype=torch.float32)
    _lib.check(lib.ub200_colsum(x.data_ptr(), out.data_ptr(), rows, N, x.stride(0),
                                _lib.dtype_code(x.dtype), _lib.current_stream()))
    return out


@_follows_torch
def cvt_from_f32(src, dtype, out=None, accumulate=False):
    """16-bit copy of an fp32 tensor (one launch)."""
    lib = _lib.load()
    src = src.contiguous()
    if out is None:
        out = torch.empty(src.shape, device=src.device, dtype=dtype)
    if src.numel():
        _lib.check(lib.ub200_cvt_from_f32(src.data_ptr(), out.data_ptr(), src.numel(),
                                          1 if accumulate else 0, _lib.dtype_code(dtype),
                                          _lib.current_stream()))
    return out


@_follows_torch
def ce_fwd(logits, targets, vocab):
    """loss [n] fp32, lse [n] fp32 of softmax cross-entropy over logits[:, :vocab] (16-bit, row
    pitch a multiple of 8)."""
    lib = _lib.load()
    n = logits.size(0)
    loss = torch.empty(n, device=logits.device, dtype=torch.float32)
    lse = torch.empty(n, device=logits.device, dtype=torch.float32)
    assert targets.dtype == torch.int64 and targets.is_contiguous() and logits.stride(1) == 1
    _lib.check(lib.ub200_ce_fwd(logits.data_ptr(), logits.stride(0), targets.data_ptr(), loss.data_ptr(),
                                lse.data_ptr(), n, vocab, _lib.dtype_code(logits.dtype),
                                _lib.current_stream()))
    return loss, lse


@_follows_torch
def ce_bwd_(logits, targets, lse, dloss, vocab):
    """In place: logits[:, c] <- (softmax - onehot) * dloss for c < vocab, 0 for the padding columns."""
    lib = _lib.load()
    n, ncols = logits.shape
    assert dloss.dtype == torch.float32 and dloss.is_contiguous()
    _lib.check(lib.ub200_ce_bwd(logits.data_ptr(), logits.data_ptr(), logits.stride(0), targets.data_ptr(),
                                lse.data_ptr(), dloss.data_ptr(), n, vocab, ncols,
                                _lib.dtype_code(logits.dtype), _lib.current_stream()))
    return logits


@_follows_torch
def dgelu_mul(dy, pre):
    lib = _lib.load()
    out = torch.empty_like(dy)
    assert dy.is_contiguous() and pre.is_contiguous() and dy.numel() % 8 == 0
    _lib.check(lib.ub200_dgelu_mul(dy.data_ptr(), pre.data_ptr(), out.data_ptr(), dy.numel(),
                                   _lib.dtype_code(dy.dtype), _lib.current_stream()))
    return out


@_follows_torch
def dtanh_mul(dy, y):
    """dy * (1 - y^2): backward of y = tanh(.) (BertPooler)."""
    lib = _lib.load()
    out = torch.empty_like(dy)
    assert dy.is_contiguous() and y.is_contiguous() and dy.numel() % 8 == 0
    _lib.check(lib.ub200_dtanh_mul(dy.data_ptr(), y.data_ptr(), out.data_ptr(), dy.numel(),
                                   _lib.dtype_code(dy.dtype), _lib.current_stream()))
    return out


def _region_args(rows, weight, seg, obj_masks, mode, margin):
    """Shared fields of ub200_region_score_args.  seg: int32 [2, B] (starts, lengths); obj_masks:
    [B, S] uint8 or bool, non-zero = masked."""
    assert rows.dim() == 2 and rows.is_contiguous() and weight.is_contiguous()
    assert seg.dtype == torch.int32 and seg.is_contiguous() and seg.dim() == 2 and seg.size(0) == 2
    assert obj_masks.dtype in (torch.uint8, torch.bool) and obj_masks.is_contiguous()
    B, S = obj_masks.shape
    assert seg.size(1) == B
    return _lib.RegionScoreArgs(
        rows=rows.data_ptr(), weight=weight.data_ptr(), seg_start=seg[0].data_ptr(), seg_len=seg[1].data_ptr(),
        obj_masks=obj_masks.data_ptr(), R=rows.size(0), hidden=rows.size(1), batch=B, max_regions=S,
        mode=int(mode), dtype=_lib.dtype_code(rows.dtype), margin=float(margin))


@_follows_torch
def region_score_fwd(rows, weight, bias, seg, obj_masks, targets=None, neg_plan=None, mode=_lib.RE_SCORES,
                     margin=0.0):
    """Referring-expression scores [B, S] (16-bit, masked positions = -1e4) and, for mode RE_CLS /
    RE_RANK, the per-sample loss [B] fp32 with what the backward needs: lse [B] fp32 (cls) or the chosen
    negative neg_ix [B] int32 (rank).  targets / neg_plan: int64 [B] (neg_plan -1 = hard negative)."""
    lib = _lib.load()
    a = _region_args(rows, weight, seg, obj_masks, mode, margin)
    B, S = obj_masks.shape
    dev = rows.device
    scores = torch.empty(B, S, device=dev, dtype=rows.dtype)
    loss = lse = neg = None
    a.bias, a.scores = _lib.ptr(bias), scores.data_ptr()
    if mode != _lib.RE_SCORES:
        assert targets.dtype == torch.int64 and targets.is_contiguous() and targets.numel() == B
        loss = torch.empty(B, device=dev, dtype=torch.float32)
        a.targets, a.loss = targets.data_ptr(), loss.data_ptr()
    if mode == _lib.RE_CLS:
        lse = torch.empty(B, device=dev, dtype=torch.float32)
        a.lse = lse.data_ptr()
    elif mode == _lib.RE_RANK:
        assert neg_plan.dtype == torch.int64 and neg_plan.is_contiguous() and neg_plan.numel() == B
        neg = torch.empty(B, device=dev, dtype=torch.int32)
        a.neg_plan, a.neg_ix = neg_plan.data_ptr(), neg.data_ptr()
    _lib.check(lib.ub200_region_score_fwd(C.byref(a), _lib.current_stream()))
    return scores, loss, lse, neg


@_follows_torch
def region_score_bwd(rows, weight, seg, obj_masks, targets, scores, lse, neg, dloss, mode, margin=0.0):
    """Backward of region_score_fwd: d_rows [R, H] (16-bit, zero on padding rows), dweight [H] and
    dbias [1] in fp32 (written, summed in sample order)."""
    lib = _lib.load()
    a = _region_args(rows, weight, seg, obj_masks, mode, margin)
    B, H = obj_masks.size(0), rows.size(1)
    assert dloss.dtype == torch.float32 and dloss.is_contiguous() and dloss.numel() == B
    d_rows = torch.empty_like(rows)
    dw = torch.empty(H, device=rows.device, dtype=torch.float32)
    db = torch.empty(1, device=rows.device, dtype=torch.float32)
    ws_bytes = lib.ub200_region_score_workspace_bytes(B, H)
    ws = torch.empty(ws_bytes // 4, device=rows.device, dtype=torch.float32)
    a.targets, a.scores, a.lse, a.neg_ix = targets.data_ptr(), scores.data_ptr(), _lib.ptr(lse), _lib.ptr(neg)
    a.dloss, a.d_rows, a.dweight, a.dbias = dloss.data_ptr(), d_rows.data_ptr(), dw.data_ptr(), db.data_ptr()
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws_bytes
    _lib.check(lib.ub200_region_score_bwd(C.byref(a), _lib.current_stream()))
    return d_rows, dw, db


def _wra_args(packed, cu_seqlens, txt_len, batch, max_m, max_n, workspace):
    assert packed.dim() == 2 and packed.is_contiguous()
    assert cu_seqlens.dtype == torch.int32 and cu_seqlens.numel() >= batch + 1
    assert txt_len.dtype == torch.int32 and txt_len.is_contiguous() and txt_len.numel() == batch
    assert workspace.dtype == torch.float32 and workspace.is_contiguous()
    return _lib.WraArgs(
        packed=packed.data_ptr(), cu_seqlens=cu_seqlens.data_ptr(), txt_len=txt_len.data_ptr(),
        workspace=workspace.data_ptr(), workspace_bytes=workspace.numel() * 4, total_rows=packed.size(0),
        hidden=packed.size(1), batch=batch, max_m=int(max_m), max_n=int(max_n), dtype=_lib.dtype_code(packed.dtype))


def wra_workspace(batch, max_m, max_n, device):
    """fp32 workspace of ub200_wra_fwd / _bwd: the transport plans and row norms of every pair."""
    return torch.empty(_lib.load().ub200_wra_workspace_bytes(batch, max_m, max_n) // 4, device=device,
                       dtype=torch.float32)


@_follows_torch
def wra_fwd(packed, cu_seqlens, txt_len, batch, max_m, max_n, workspace):
    """Word-region alignment distance [batch] (fp32 holding 16-bit-rounded values) of the pairs of the
    packed encoder output [T_pad, H]: pair b owns rows cu_seqlens[b] .. cu_seqlens[b+1] - 1, its txt_len[b]
    text rows first.  max_m / max_n bound every pair's text / region count.  Writes the plans and norms
    the backward reads into `workspace` (wra_workspace)."""
    lib = _lib.load()
    a = _wra_args(packed, cu_seqlens, txt_len, batch, max_m, max_n, workspace)
    dist = torch.empty(batch, device=packed.device, dtype=torch.float32)
    a.dist = dist.data_ptr()
    _lib.check(lib.ub200_wra_fwd(C.byref(a), _lib.current_stream()))
    return dist


@_follows_torch
def wra_bwd(packed, cu_seqlens, txt_len, batch, max_m, max_n, workspace, d_dist):
    """Backward of wra_fwd with its plans held constant: d_packed [T_pad, H] 16-bit, zero on rows from
    cu_seqlens[batch] on."""
    lib = _lib.load()
    a = _wra_args(packed, cu_seqlens, txt_len, batch, max_m, max_n, workspace)
    assert d_dist.dtype == torch.float32 and d_dist.is_contiguous() and d_dist.numel() == batch
    d_packed = torch.empty_like(packed)
    a.d_dist, a.d_packed = d_dist.data_ptr(), d_packed.data_ptr()
    _lib.check(lib.ub200_wra_bwd(C.byref(a), _lib.current_stream()))
    return d_packed


@_follows_torch
def gather_rows(src, index, rows=None):
    """dst[r] = src[index[r]] if index[r] >= 0 else 0 (int32 index; bit-exact row mover)."""
    lib = _lib.load()
    src = src.contiguous()
    rows = index.numel() if rows is None else rows
    H = src.size(-1)
    dst = torch.empty(rows, H, device=src.device, dtype=src.dtype)
    if rows:
        _lib.check(lib.ub200_gather_rows(src.data_ptr(), dst.data_ptr(), index.data_ptr(), rows,
                                         H * src.element_size(), _lib.current_stream()))
    return dst
