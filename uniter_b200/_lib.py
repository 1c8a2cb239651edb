"""ctypes binding of libub200.so — the only way Python reaches the CUDA kernels.

There is deliberately no fallback: if the library is missing or the device is not sm_90 the
import of the compute path raises.
"""
import contextlib
import ctypes as C
import functools
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libub200.so")

F16, BF16 = 0, 1
EPI_BIAS, EPI_DROPOUT, EPI_RESIDUAL, EPI_GELU = 1, 2, 4, 8
EPI_DGELU, EPI_ACCUM, EPI_OUT_F32, EPI_COLSUM = 16, 32, 64, 128
EPI_ATOMIC = 256
EPI_TANH = 512


class GemmArgs(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("b", C.c_void_p),
        ("lda", C.c_int64), ("ldb", C.c_int64),
        ("a_major", C.c_int32), ("b_major", C.c_int32),
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("dtype", C.c_int32), ("epilogue", C.c_int32),
        ("bias", C.c_void_p), ("residual", C.c_void_p), ("aux", C.c_void_p),
        ("out", C.c_void_p), ("out2", C.c_void_p), ("colsum", C.c_void_p),
        ("ldr", C.c_int64), ("ldaux", C.c_int64), ("ldo", C.c_int64),
        ("dropout_p", C.c_float),
        ("rng_seed", C.c_uint64), ("rng_stream", C.c_uint64),
        ("tile_n", C.c_int32), ("max_ctas", C.c_int32), ("cluster", C.c_int32),
        ("k_splits", C.c_int32), ("n_valid", C.c_int32),
        ("rng_offset_dev", C.c_void_p),
    ]


class AttnArgs(C.Structure):
    _fields_ = [
        ("qkv", C.c_void_p), ("ctx", C.c_void_p), ("lse", C.c_void_p), ("cu_seqlens", C.c_void_p),
        ("batch", C.c_int32), ("total_tokens", C.c_int32), ("max_seqlen", C.c_int32),
        ("hidden", C.c_int32), ("num_heads", C.c_int32), ("dtype", C.c_int32),
        ("dropout_p", C.c_float), ("rng_seed", C.c_uint64), ("rng_stream", C.c_uint64),
        ("dctx", C.c_void_p), ("dqkv", C.c_void_p), ("workspace", C.c_void_p), ("dbias", C.c_void_p),
        ("rng_offset_dev", C.c_void_p),
    ]


class LnBwdArgs(C.Structure):
    _fields_ = [
        ("dy", C.c_void_p), ("x", C.c_void_p), ("gamma", C.c_void_p), ("dx", C.c_void_p),
        ("dx_drop", C.c_void_p), ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("dbias", C.c_void_p),
        ("rows", C.c_int32), ("hidden", C.c_int32), ("dtype", C.c_int32),
        ("dropout_p", C.c_float), ("rng_seed", C.c_uint64), ("rng_stream", C.c_uint64),
        ("row_kind", C.c_void_p), ("kind", C.c_int32), ("dropout_on_dy", C.c_int32),
        ("rng_offset_dev", C.c_void_p), ("stats_ws", C.c_void_p), ("act", C.c_int32),
    ]


LN_ACT_NONE, LN_ACT_RELU = 0, 1


class EmbedPrepArgs(C.Structure):
    _fields_ = [
        ("pack_idx", C.c_void_p), ("gather_index", C.c_void_p), ("input_ids", C.c_void_p),
        ("position_ids", C.c_void_p), ("txt_type_ids", C.c_void_p), ("img_type_ids", C.c_void_p),
        ("img_masks", C.c_void_p),
        ("T", C.c_int32), ("L", C.c_int32), ("Lt", C.c_int32), ("Li", C.c_int32),
        ("pos_rows", C.c_int32), ("mode", C.c_int32),
        ("kind", C.c_void_p), ("word_id", C.c_void_p), ("pos_id", C.c_void_p),
        ("type_id", C.c_void_p), ("img_src", C.c_void_p), ("mask_flag", C.c_void_p),
    ]


class EmbedRowsArgs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "kind", "word_id", "pos_id", "type_id", "img_src", "word_emb", "pos_emb", "type_emb",
        "ln_txt_g", "ln_txt_b", "img_linear_out", "pos_feat", "w_pos", "b_pos",
        "ln_img_g", "ln_img_b", "ln_pos_g", "ln_pos_b", "ln_out_g", "ln_out_b", "x", "u", "ppre")] + [
        ("T", C.c_int32), ("hidden", C.c_int32), ("dtype", C.c_int32),
        ("dropout_p", C.c_float), ("rng_seed", C.c_uint64), ("rng_stream", C.c_uint64),
        ("rng_offset_dev", C.c_void_p)]


class EmbedColsumArgs(C.Structure):
    _fields_ = [("x", C.c_void_p), ("type_id", C.c_void_p), ("kind", C.c_void_p),
                ("img_src", C.c_void_p), ("pos_feat", C.c_void_p), ("out", C.c_void_p),
                ("T", C.c_int32), ("hidden", C.c_int32), ("mode", C.c_int32),
                ("type_vocab", C.c_int32), ("dtype", C.c_int32)]


class AdamSegment(C.Structure):
    _fields_ = [("grad", C.c_void_p), ("master", C.c_void_p), ("exp_avg", C.c_void_p),
                ("exp_avg_sq", C.c_void_p), ("model", C.c_void_p), ("n", C.c_int64),
                ("step_size", C.c_float), ("lr_wd", C.c_float),
                ("grad_dtype", C.c_int32), ("model_dtype", C.c_int32),
                ("weight_decay", C.c_float), ("group", C.c_int32), ("step_offset", C.c_int32),
                ("flags", C.c_int32)]


class LossScalerEntry(C.Structure):
    _fields_ = [("scale", C.c_float), ("unskipped", C.c_int32), ("inv_scale", C.c_float),
                ("window", C.c_int32), ("max_scale", C.c_float), ("min_scale", C.c_float),
                ("_pad", C.c_int32 * 2)]


MAX_PEERS = 8


class PeerAllreduceArgs(C.Structure):
    _fields_ = [("buf", C.c_void_p * MAX_PEERS), ("stage", C.c_void_p * MAX_PEERS),
                ("flags", C.POINTER(C.c_uint32) * MAX_PEERS),
                ("rank", C.c_int32), ("world", C.c_int32),
                ("offset", C.c_int64), ("count", C.c_int64), ("stage_bytes", C.c_int64),
                ("dtype", C.c_int32), ("max_ctas", C.c_int32), ("scale", C.c_float),
                ("timeout_ms", C.c_int32)]


RE_SCORES, RE_CLS, RE_RANK = 0, 1, 2


class RegionScoreArgs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "rows", "weight", "bias", "seg_start", "seg_len", "obj_masks", "targets", "neg_plan", "scores",
        "loss", "lse", "neg_ix", "dloss", "d_rows", "dweight", "dbias", "workspace")] + [
        ("workspace_bytes", C.c_int64),
        ("R", C.c_int32), ("hidden", C.c_int32), ("batch", C.c_int32), ("max_regions", C.c_int32),
        ("mode", C.c_int32), ("dtype", C.c_int32), ("margin", C.c_float)]


class WraArgs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("packed", "cu_seqlens", "txt_len", "dist", "d_dist", "d_packed",
                                          "workspace")] + [
        ("workspace_bytes", C.c_int64),
        ("total_rows", C.c_int32), ("hidden", C.c_int32), ("batch", C.c_int32), ("max_m", C.c_int32),
        ("max_n", C.c_int32), ("dtype", C.c_int32)]


WRA_MAX_MN = 11264      # UB200_WRA_MAX_MN

F32 = 2
_lib = None


def load():
    """Load libub200.so (building is the job of ``uniter_b200.build`` / ``__graft_entry__``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libub200.so not found at %s — run `python -m uniter_b200.build` "
            "(there is no non-CUDA fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.ub200_version.restype = C.c_int
    lib.ub200_last_error_string.restype = C.c_char_p
    lib.ub200_device_check.restype = C.c_int
    lib.ub200_set_sm_reserve.restype = C.c_int
    lib.ub200_set_sm_reserve.argtypes = [C.c_int]
    lib.ub200_set_deterministic.restype = C.c_int
    lib.ub200_set_deterministic.argtypes = [C.c_int]
    lib.ub200_deterministic.restype = C.c_int
    lib.ub200_deterministic.argtypes = []
    lib.ub200_gemm.restype = C.c_int
    lib.ub200_gemm.argtypes = [C.POINTER(GemmArgs), C.c_void_p]
    lib.ub200_gemm_grouped.restype = C.c_int
    lib.ub200_gemm_grouped.argtypes = [C.POINTER(GemmArgs), C.c_int32, C.c_void_p]
    for name in ("ub200_attn_fwd", "ub200_attn_bwd"):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = [C.POINTER(AttnArgs), C.c_void_p]
    lib.ub200_attn_bwd_workspace_bytes.restype = C.c_int64
    lib.ub200_attn_bwd_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    lib.ub200_layernorm_fwd.restype = C.c_int
    lib.ub200_layernorm_fwd.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_layernorm_fwd_act.restype = C.c_int
    lib.ub200_layernorm_fwd_act.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_layernorm_bwd.restype = C.c_int
    lib.ub200_layernorm_bwd.argtypes = [C.POINTER(LnBwdArgs), C.c_void_p]
    lib.ub200_colsum.restype = C.c_int
    lib.ub200_colsum.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_int32,
                                 C.c_void_p]
    lib.ub200_embed_prep.restype = C.c_int
    lib.ub200_embed_prep.argtypes = [C.POINTER(EmbedPrepArgs), C.c_void_p]
    lib.ub200_embed_gather_cast.restype = C.c_int
    lib.ub200_embed_gather_cast.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_embed_rows_fwd.restype = C.c_int
    lib.ub200_embed_rows_fwd.argtypes = [C.POINTER(EmbedRowsArgs), C.c_void_p]
    lib.ub200_embed_bwd_scatter.restype = C.c_int
    lib.ub200_embed_bwd_scatter.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_embed_bwd_colsums.restype = C.c_int
    lib.ub200_embed_bwd_colsums.argtypes = [C.POINTER(EmbedColsumArgs), C.c_void_p]
    lib.ub200_cvt_from_f32_strided.restype = C.c_int
    lib.ub200_cvt_from_f32_strided.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64,
                                               C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_ce_fwd.restype = C.c_int
    lib.ub200_ce_fwd.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_ce_bwd.restype = C.c_int
    lib.ub200_ce_bwd.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_dgelu_mul.restype = C.c_int
    lib.ub200_dgelu_mul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
    lib.ub200_dtanh_mul.restype = C.c_int
    lib.ub200_dtanh_mul.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p]
    lib.ub200_cvt_from_f32.restype = C.c_int
    lib.ub200_cvt_from_f32.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_adam_chunk.restype = C.c_int32
    lib.ub200_grad_sumsq.restype = C.c_int
    lib.ub200_grad_sumsq.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
    lib.ub200_grad_sumsq_workspace_bytes.restype = C.c_int64
    lib.ub200_grad_sumsq_workspace_bytes.argtypes = [C.c_int32]
    lib.ub200_grad_sumsq_ws.restype = C.c_int
    lib.ub200_grad_sumsq_ws.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_int64, C.c_void_p]
    lib.ub200_adamw_step.restype = C.c_int
    lib.ub200_adamw_step.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                     C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]
    lib.ub200_adam_prep.restype = C.c_int
    lib.ub200_adam_prep.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    lib.ub200_adam_prep_scaled.restype = C.c_int
    lib.ub200_adam_prep_scaled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
    lib.ub200_adamw_step_scaled.restype = C.c_int
    lib.ub200_adamw_step_scaled.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_float,
                                            C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_int32, C.c_void_p]
    lib.ub200_region_score_workspace_bytes.restype = C.c_int64
    lib.ub200_region_score_workspace_bytes.argtypes = [C.c_int32, C.c_int32]
    for name in ("ub200_region_score_fwd", "ub200_region_score_bwd"):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = [C.POINTER(RegionScoreArgs), C.c_void_p]
    lib.ub200_wra_workspace_bytes.restype = C.c_int64
    lib.ub200_wra_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32]
    for name in ("ub200_wra_fwd", "ub200_wra_bwd"):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = [C.POINTER(WraArgs), C.c_void_p]
    lib.ub200_gather_rows.restype = C.c_int
    lib.ub200_gather_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
    lib.ub200_peer_flags_bytes.restype = C.c_int64
    lib.ub200_peer_stage_bytes.restype = C.c_int64
    lib.ub200_peer_stage_bytes.argtypes = [C.c_int64, C.c_int32]
    lib.ub200_peer_allreduce.restype = C.c_int
    lib.ub200_peer_allreduce.argtypes = [C.POINTER(PeerAllreduceArgs), C.c_void_p]
    lib.ub200_peer_ipc_export.restype = C.c_int
    lib.ub200_peer_ipc_export.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
    lib.ub200_peer_ipc_open.restype = C.c_int
    lib.ub200_peer_ipc_open.argtypes = [C.c_char_p, C.POINTER(C.c_void_p)]
    lib.ub200_peer_ipc_close.restype = C.c_int
    lib.ub200_peer_ipc_close.argtypes = [C.c_void_p]
    _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError("libub200 error %d: %s" % (rc, load().ub200_last_error_string().decode()))


def dtype_code(t, allow_f32=False):
    import torch
    if t == torch.bfloat16:
        return BF16
    if t == torch.float16:
        return F16
    if t == torch.float32 and allow_f32:
        return F32
    raise TypeError("libub200 computes in fp16 or bf16, got %s" % t)


def ptr(t):
    return None if t is None else t.data_ptr()


def deterministic():
    """Whether the library's deterministic mode (ub200_set_deterministic) is on: read from the library."""
    return bool(load().ub200_deterministic())


# Longest sequence whose attention backward has a fixed-order form (attn.cu: SH_MAXSEQ).  Longer
# sequences sum dQ over key blocks with float atomics; the deterministic mode refuses them.
DET_ATTN_BWD_MAX_SEQLEN = 128

_pinned_modes = []      # modes of the enclosing library_mode() scopes, innermost last


def select_mode(max_seqlen=None):
    """The library mode for launches made here: the one place where torch's determinism flags are read.

    Returns None when torch.use_deterministic_algorithms is off (the library's switch is left as it is,
    so C callers and tests that set it keep their mode), 1 when it is on, and 0 for work the fixed-order
    mode cannot cover under warn_only.  Inside a library_mode() scope (an autograd backward, a captured
    step) the scope's mode is returned instead of reading torch's flags again.

    max_seqlen: the host-known longest sequence of work that includes an attention backward.  Above
    DET_ATTN_BWD_MAX_SEQLEN the mode has no fixed-order form: this raises a RuntimeError, or with
    warn_only=True warns and returns 0 (that work runs in the default mode)."""
    import torch
    if _pinned_modes:
        mode = _pinned_modes[-1]
    else:
        mode = 1 if torch.are_deterministic_algorithms_enabled() else None
    if mode == 1 and max_seqlen is not None and max_seqlen > DET_ATTN_BWD_MAX_SEQLEN:
        msg = ("libub200 attention backward with max_seqlen %d > %d has no deterministic implementation "
               "(dQ is summed over key blocks with float atomics); it is refused under "
               "torch.use_deterministic_algorithms(True)" % (max_seqlen, DET_ATTN_BWD_MAX_SEQLEN))
        if not torch.is_deterministic_algorithms_warn_only_enabled():
            raise RuntimeError(msg + ".  Pass warn_only=True to run it in the default mode with a warning.")
        import warnings
        warnings.warn(msg + "; with warn_only=True it runs in the default mode.", UserWarning, stacklevel=3)
        return 0
    return mode


@contextlib.contextmanager
def library_mode(mode):
    """Run the enclosed launches in `mode` (a select_mode() result) and restore the previous value of
    the library's switch afterwards.  None leaves the switch untouched."""
    lib = load() if mode is not None else None
    prev = lib.ub200_set_deterministic(mode) if mode is not None else None
    _pinned_modes.append(mode)
    try:
        yield
    finally:
        _pinned_modes.pop()
        if mode is not None:
            lib.ub200_set_deterministic(prev)


def forward_in_mode(max_seqlen=None):
    """Decorator for the forward of a torch.autograd.Function that launches library work: runs it in
    select_mode() and stores that mode in ctx for backward_in_mode.  max_seqlen(ctx, *args): the
    longest sequence whose attention backward this node will run, or None."""
    def wrap(fn):
        @functools.wraps(fn)
        def forward(ctx, *args):
            mode = select_mode(max_seqlen(ctx, *args) if max_seqlen is not None else None)
            ctx.ub200_mode = mode
            with library_mode(mode):
                return fn(ctx, *args)
        return forward
    return wrap


def backward_in_mode(fn):
    """Decorator for the backward of a Function whose forward has forward_in_mode: the backward runs in
    the mode of its forward, whatever torch's flags are when it runs."""
    @functools.wraps(fn)
    def backward(ctx, *grads):
        with library_mode(ctx.ub200_mode):
            return fn(ctx, *grads)
    return backward


def current_stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


class PinnedRing(object):
    """Rotating pinned host staging buffers for small per-step H2D copies (packing metadata,
    optimizer segment tables).  A copy from PAGEABLE memory makes the host wait until the stream
    has drained, i.e. it costs a full synchronisation per step; from pinned memory it is just
    another asynchronous stream operation.  A slot is reused only after the copy that last read it
    has completed (event), which in steady state is always already true."""

    def __init__(self, slots=8):
        self.slots = [None] * slots
        self.events = [None] * slots
        self.i = 0

    def upload(self, host_tensor, device):
        """Async copy of a contiguous CPU tensor to `device` through a pinned slot."""
        import torch
        nbytes = host_tensor.numel() * host_tensor.element_size()
        k = self.i
        self.i = (self.i + 1) % len(self.slots)
        if self.events[k] is not None:
            self.events[k].synchronize()
        buf = self.slots[k]
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(nbytes, 1 << 16), dtype=torch.uint8).pin_memory()
            self.slots[k] = buf
        stage = buf[:nbytes].view(host_tensor.dtype)
        stage.copy_(host_tensor.reshape(-1))
        dev = torch.empty(host_tensor.numel(), dtype=host_tensor.dtype, device=device)
        dev.copy_(stage, non_blocking=True)
        ev = self.events[k]
        if ev is None:
            ev = torch.cuda.Event()
            self.events[k] = ev
        ev.record(torch.cuda.current_stream(device))
        return dev
