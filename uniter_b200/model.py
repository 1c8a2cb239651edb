"""Drop-in `UniterModel` for ChenRocks/UNITER running the encoder on libub200 (sm_90a).

Mirrors the reference's Python contract for the hot path (SURVEY.md §8b-B1):

* ``UniterConfig`` — model/model.py:24-114 (same constructor, ``from_dict`` / ``from_json_file``)
* ``UniterPreTrainedModel`` — model/model.py:117-214 (``init_weights``, ``from_pretrained`` incl.
  the gamma/beta rename and the optional ``bert.`` prefix)
* ``UniterModel(config, img_dim)`` — model/model.py:295-367: same submodule tree, parameter names
  and shapes (so ``uniter-base.pt`` / ``uniter-large.pt`` load unchanged and name-based weight-decay
  grouping, optim/misc.py:14-22, keeps working), same ``forward`` signature and return types.

What differs underneath: the encoder stack runs over PACKED valid tokens ([T, H], no padding
compute) through hand-written CUDA kernels behind a C ABI; rows where ``attention_mask == 0`` are
returned as zeros (the reference returns garbage there that no head reads).  There is no
CPU / eager fallback: parameters must be fp16 or bf16 and live on an H100.
"""
import copy
import ctypes as C
import json
import logging
import math
import weakref

import numpy as np
import torch
from torch import nn

from . import _lib

logger = logging.getLogger(__name__)


# ============================================================================ config
class UniterConfig(object):
    """Same fields and construction rules as the reference (model/model.py:24-114)."""

    def __init__(self, vocab_size_or_config_json_file, hidden_size=768, num_hidden_layers=12,
                 num_attention_heads=12, intermediate_size=3072, hidden_act="gelu",
                 hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                 max_position_embeddings=512, type_vocab_size=2, initializer_range=0.02):
        if isinstance(vocab_size_or_config_json_file, str):
            with open(vocab_size_or_config_json_file, "r", encoding="utf-8") as reader:
                for key, value in json.loads(reader.read()).items():
                    self.__dict__[key] = value
        elif isinstance(vocab_size_or_config_json_file, int):
            self.vocab_size = vocab_size_or_config_json_file
            self.hidden_size = hidden_size
            self.num_hidden_layers = num_hidden_layers
            self.num_attention_heads = num_attention_heads
            self.hidden_act = hidden_act
            self.intermediate_size = intermediate_size
            self.hidden_dropout_prob = hidden_dropout_prob
            self.attention_probs_dropout_prob = attention_probs_dropout_prob
            self.max_position_embeddings = max_position_embeddings
            self.type_vocab_size = type_vocab_size
            self.initializer_range = initializer_range
        else:
            raise ValueError("First argument must be either a vocabulary size (int) or the path "
                             "to a pretrained model config file (str)")

    @classmethod
    def from_dict(cls, json_object):
        config = UniterConfig(vocab_size_or_config_json_file=-1)
        for key, value in json_object.items():
            config.__dict__[key] = value
        return config

    @classmethod
    def from_json_file(cls, json_file):
        with open(json_file, "r", encoding="utf-8") as reader:
            return cls.from_dict(json.loads(reader.read()))

    def __repr__(self):
        return str(self.to_json_string())

    def to_dict(self):
        return copy.deepcopy(self.__dict__)

    def to_json_string(self):
        return json.dumps(self.to_dict(), indent=2, sort_keys=True) + "\n"


_CONFIG_FIELDS = ("vocab_size", "hidden_size", "num_hidden_layers", "num_attention_heads",
                  "intermediate_size", "hidden_act", "hidden_dropout_prob",
                  "attention_probs_dropout_prob", "max_position_embeddings", "type_vocab_size",
                  "initializer_range")


class UniterPreTrainedModel(nn.Module):
    """Weight init + checkpoint loading with the reference's semantics (model/model.py:117-214)."""

    def __init__(self, config, *inputs, **kwargs):
        super().__init__()
        missing = [f for f in _CONFIG_FIELDS if not hasattr(config, f)]
        if missing:  # accepts the reference's own UniterConfig instances (duck-typed)
            raise ValueError("Parameter config in `{}(config)` should be a UniterConfig; missing "
                             "fields {}".format(self.__class__.__name__, missing))
        self.config = config

    def init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=self.config.initializer_range)
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)
        if isinstance(module, nn.Linear) and module.bias is not None:
            module.bias.data.zero_()

    @classmethod
    def from_pretrained(cls, config_file, state_dict, *inputs, **kwargs):
        config = UniterConfig.from_json_file(config_file)
        logger.info("Model config {}".format(config))
        model = cls(config, *inputs, **kwargs)
        # TF-style names: gamma -> weight, beta -> bias (model/model.py:166-176)
        state_dict = state_dict.copy()
        metadata = getattr(state_dict, "_metadata", None)
        for key in list(state_dict.keys()):
            new_key = None
            if "gamma" in key:
                new_key = key.replace("gamma", "weight")
            if "beta" in key:
                new_key = key.replace("beta", "bias")
            if new_key:
                state_dict[new_key] = state_dict.pop(key)
        if metadata is not None:
            state_dict._metadata = metadata
        missing_keys, unexpected_keys, error_msgs = [], [], []

        def load(module, prefix=""):
            local_metadata = {} if metadata is None else metadata.get(prefix[:-1], {})
            module._load_from_state_dict(state_dict, prefix, local_metadata, True, missing_keys,
                                         unexpected_keys, error_msgs)
            for name, child in module._modules.items():
                if child is not None:
                    load(child, prefix + name + ".")

        start_prefix = ""
        if not hasattr(model, "bert") and any(s.startswith("bert.") for s in state_dict.keys()):
            start_prefix = "bert."
        load(model, prefix=start_prefix)
        if missing_keys:
            logger.info("Weights of {} not initialized from pretrained model: {}".format(
                model.__class__.__name__, missing_keys))
        if unexpected_keys:
            logger.info("Weights from pretrained model not used in {}: {}".format(
                model.__class__.__name__, unexpected_keys))
        if error_msgs:
            raise RuntimeError("Error(s) in loading state_dict for {}:\n\t{}".format(
                model.__class__.__name__, "\n\t".join(error_msgs)))
        return model


# ============================================================================ parameter containers
# These modules own the nn.Parameters at the reference's attribute paths.  The encoder-layer
# containers never run a torch forward: the kernels read the parameters by pointer.
class BertSelfAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        if config.hidden_size % config.num_attention_heads != 0:
            raise ValueError("The hidden size (%d) is not a multiple of the number of attention "
                             "heads (%d)" % (config.hidden_size, config.num_attention_heads))
        self.num_attention_heads = config.num_attention_heads
        self.attention_head_size = config.hidden_size // config.num_attention_heads
        self.all_head_size = config.hidden_size
        self.query = nn.Linear(config.hidden_size, config.hidden_size)
        self.key = nn.Linear(config.hidden_size, config.hidden_size)
        self.value = nn.Linear(config.hidden_size, config.hidden_size)
        self.dropout = nn.Dropout(config.attention_probs_dropout_prob)


class BertSelfOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class BertAttention(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.self = BertSelfAttention(config)
        self.output = BertSelfOutput(config)


class BertIntermediate(nn.Module):
    def __init__(self, config):
        super().__init__()
        if config.hidden_act != "gelu":
            raise ValueError("libub200 implements hidden_act='gelu' (erf form) only, got %r"
                             % (config.hidden_act,))
        self.dense = nn.Linear(config.hidden_size, config.intermediate_size)


class BertOutput(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.intermediate_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)


class BertLayer(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.attention = BertAttention(config)
        self.intermediate = BertIntermediate(config)
        self.output = BertOutput(config)


class BertPooler(nn.Module):
    """tanh(dense(x[:, 0])) — model/layer.py:173-185 — on libub200: the [CLS] rows are read in place
    from the [B, L, H] tensor (row pitch L*H), one wgmma GEMM with the bias + tanh epilogue."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.activation = nn.Tanh()

    def forward(self, hidden_states):
        first = hidden_states[:, 0] if hidden_states.dim() == 3 else hidden_states
        return LibLinear.apply(first, self.dense.weight, self.dense.bias, False, True)


class UniterTextEmbeddings(nn.Module):
    """model/model.py:217-245."""

    def __init__(self, config):
        super().__init__()
        self.word_embeddings = nn.Embedding(config.vocab_size, config.hidden_size, padding_idx=0)
        self.position_embeddings = nn.Embedding(config.max_position_embeddings, config.hidden_size)
        self.token_type_embeddings = nn.Embedding(config.type_vocab_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, input_ids, position_ids, token_type_ids=None):
        if token_type_ids is None:
            token_type_ids = torch.zeros_like(input_ids)
        embeddings = (self.word_embeddings(input_ids) + self.position_embeddings(position_ids)
                      + self.token_type_embeddings(token_type_ids))
        return self.dropout(self.LayerNorm(embeddings))


class UniterImageEmbeddings(nn.Module):
    """model/model.py:248-272."""

    def __init__(self, config, img_dim):
        super().__init__()
        self.img_linear = nn.Linear(img_dim, config.hidden_size)
        self.img_layer_norm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.pos_layer_norm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.pos_linear = nn.Linear(7, config.hidden_size)
        self.mask_embedding = nn.Embedding(2, img_dim, padding_idx=0)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)
        self.dropout = nn.Dropout(config.hidden_dropout_prob)

    def forward(self, img_feat, img_pos_feat, type_embeddings, img_masks=None):
        if img_masks is not None:
            self.mask_embedding.weight.data[0, :].fill_(0)
            img_feat = img_feat + self.mask_embedding(img_masks.long())
        transformed_im = self.img_layer_norm(self.img_linear(img_feat))
        transformed_pos = self.pos_layer_norm(self.pos_linear(img_pos_feat))
        embeddings = self.LayerNorm(transformed_im + transformed_pos + type_embeddings)
        return self.dropout(embeddings)


class UniterEncoder(nn.Module):
    def __init__(self, config):
        super().__init__()
        layer = BertLayer(config)
        self.layer = nn.ModuleList([copy.deepcopy(layer) for _ in range(config.num_hidden_layers)])


# ============================================================================ ctypes mirrors
class _LayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("wqkv", "bqkv", "wo", "bo", "ln1_g", "ln1_b", "w1", "b1",
                                          "w2", "b2", "ln2_g", "ln2_b")]


class _LayerGrads(C.Structure):
    _fields_ = [("dwqkv", C.c_void_p), ("dwo", C.c_void_p), ("dw1", C.c_void_p),
                ("dw2", C.c_void_p), ("small", C.c_void_p)]


class _EncoderDesc(C.Structure):
    _fields_ = [("hidden", C.c_int32), ("intermediate", C.c_int32), ("num_heads", C.c_int32),
                ("num_layers", C.c_int32), ("dtype", C.c_int32), ("batch", C.c_int32),
                ("total_tokens", C.c_int32), ("max_seqlen", C.c_int32),
                ("cu_seqlens", C.c_void_p), ("hidden_dropout_p", C.c_float),
                ("attn_dropout_p", C.c_float), ("rng_seed", C.c_uint64), ("rng_offset", C.c_uint64),
                ("layer_offset", C.c_int32), ("rng_offset_dev", C.c_void_p)]


_lib_ready = False


def _bind():
    global _lib_ready
    lib = _lib.load()
    if not _lib_ready:
        lib.ub200_encoder_act_bytes_per_layer.restype = C.c_int64
        lib.ub200_encoder_act_bytes_per_layer.argtypes = [C.POINTER(_EncoderDesc)]
        lib.ub200_encoder_bwd_scratch_bytes.restype = C.c_int64
        lib.ub200_encoder_bwd_scratch_bytes.argtypes = [C.POINTER(_EncoderDesc)]
        lib.ub200_encoder_small_grad_count.restype = C.c_int64
        lib.ub200_encoder_small_grad_count.argtypes = [C.c_int32, C.c_int32]
        lib.ub200_encoder_fwd.restype = C.c_int
        lib.ub200_encoder_fwd.argtypes = [C.POINTER(_EncoderDesc), C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
        lib.ub200_encoder_bwd.restype = C.c_int
        lib.ub200_encoder_bwd.argtypes = [C.POINTER(_EncoderDesc), C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]
        lib.ub200_gather_rows.restype = C.c_int
        lib.ub200_gather_rows.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                          C.c_void_p]
        _lib_ready = True
    return lib


_rng_offset = [0]
# Graph mode (uniter_b200.graphed.GraphedStep): the host-side offset of a launch is frozen inside a
# captured CUDA graph, so the per-step part of the dropout stream id comes from a DEVICE counter
# (bumped inside the graph at the start of every replay) and the host only numbers the calls
# within one step.
_RNG_GRAPH = {"dev": None, "call": 0}


def _next_rng(device):
    """(seed, host offset, device-counter pointer or None) for one forward call that draws dropout."""
    seed = torch.cuda.initial_seed() & 0xFFFFFFFFFFFFFFFF
    if _RNG_GRAPH["dev"] is not None:
        _RNG_GRAPH["call"] += 1
        return seed, _RNG_GRAPH["call"], _RNG_GRAPH["dev"].data_ptr()
    _rng_offset[0] += 1
    return seed, _rng_offset[0], None


_META_CACHE = {}
_META_RING = _lib.PinnedRing(8)


def _meta_key(t):
    return (t._version, t.size(0), t.size(1))


def _meta_lookup(t):
    """Cache entry for THIS tensor object (weak reference + version), never for whatever tensor
    happens to live at the same address: the caching allocator hands the block of a freed mask to
    the next mask of the same shape, so an address-keyed cache would serve stale lengths."""
    hit = _META_CACHE.get(id(t))
    if hit is not None and hit[0]() is t and hit[1] == _meta_key(t):
        return hit[2]
    return None


def _meta_store(t, meta):
    if len(_META_CACHE) > 64:
        for k in [k for k, v in _META_CACHE.items() if v[0]() is None]:
            del _META_CACHE[k]
        if len(_META_CACHE) > 64:
            _META_CACHE.clear()
    _META_CACHE[id(t)] = (weakref.ref(t), _meta_key(t), meta)


def _prefix_pack_host(lens, L, T_pad=None):
    """Packing bookkeeping of a batch of PREFIX masks ([1]*S_b + [0]*(L-S_b)) from the host-known
    lengths, as ONE int32 buffer (sections start on 16-byte boundaries):

        cu_seqlens [B+2]   row range of sequence b; entry B+1 closes a DUMMY sequence (see below)
        pack_idx   [T_pad] packed row -> flat position b*L+j it is computed from
        pack_inv   [T_pad] the same, but -1 on dummy rows (inverse map for gradients)
        unpack_idx [B*L+1] flat position -> packed row, -1 at masked positions; the extra last entry
                           is -1 so that index B*L means "no row" (padding of index lists)

    `T_pad` > T (graph mode) pads the token count to a bucket size with one DUMMY sequence of
    T_pad - T rows after the real ones, so that a captured CUDA graph (whose launch shapes are
    frozen) serves every batch of the bucket.  Dummy rows are computed from the first valid position
    (finite values), attend only to each other, are referenced by no output position and receive a
    zero gradient, so they change neither the loss nor any gradient — bit for bit.
    Returns (buffer, offsets dict, T)."""
    B = len(lens)
    lens_a = np.asarray(lens, dtype=np.int64).reshape(B)
    cu = np.zeros(B + 2, dtype=np.int64)
    np.cumsum(lens_a, out=cu[1:B + 1])
    T = int(cu[B])
    T_pad = T if T_pad is None else int(T_pad)
    assert T_pad >= T
    cu[B + 1] = T_pad
    row_b = np.repeat(np.arange(B, dtype=np.int64), lens_a)     # (torch.repeat_interleave on CPU
    pack = np.arange(T, dtype=np.int64) - cu[row_b] + row_b * L  #  costs ~20 ms here; numpy ~20 us)
    o_pack = (B + 2 + 3) // 4 * 4
    o_inv = o_pack + (T_pad + 3) // 4 * 4
    o_unpack = o_inv + (T_pad + 3) // 4 * 4
    buf = np.full(o_unpack + B * L + 1, -1, dtype=np.int32)
    buf[:B + 2] = cu
    buf[o_pack:o_pack + T] = pack
    buf[o_pack + T:o_pack + T_pad] = pack[0] if T else 0
    buf[o_inv:o_inv + T] = pack
    buf[o_unpack + pack] = np.arange(T, dtype=np.int32)
    host = torch.from_numpy(buf)
    return host, dict(cu=0, pack=o_pack, inv=o_inv, unpack=o_unpack, size=buf.size), T


def _meta_from_buffer(devbuf, offs, B, L, T_pad, max_seqlen, lens_host, dummy):
    """Meta dict over a device copy of the _prefix_pack_host buffer."""
    return dict(batch=B + 1 if dummy else B, L=L, total=T_pad, max_seqlen=max_seqlen,
                cu_seqlens=devbuf[offs["cu"]:offs["cu"] + B + 2],
                pack_idx=devbuf[offs["pack"]:offs["pack"] + T_pad],
                pack_inv=devbuf[offs["inv"]:offs["inv"] + T_pad],
                unpack_idx=devbuf[offs["unpack"]:offs["unpack"] + B * L],
                unpack_ext=devbuf[offs["unpack"]:offs["unpack"] + B * L + 1],
                lens_host=lens_host, n_batch=B)


def register_lengths(attention_mask_dev, lens_host, prefix=False):
    """Tell the model the per-sample valid lengths of a device attention mask that the host
    already knows (the loader computed them before the H2D copy), so forward() does not have to
    read them back.  Bound to this tensor OBJECT (and its version): pass the same object to
    forward().  `prefix=True` additionally asserts that the mask is a prefix mask
    ([1]*S_b + [0]*(L-S_b), what every reference collate emits, e.g. data/vqa.py:39,53): the pack
    indices are then computed arithmetically."""
    _meta_store(attention_mask_dev, {"lens_host": [int(v) for v in lens_host], "prefix": bool(prefix)})


# ============================================================================ autograd glue
class _GatherRows(torch.autograd.Function):
    """dst[r] = src[index[r]] (index >= 0) else 0 — bit-exact row mover (ub200_gather_rows).

    Backward: if `inverse` (an index with dst = inverse-gather of grad) is given, the gradient is
    itself a row gather (pack <-> unpack are mutually inverse); otherwise rows are scatter-ADDED
    back, so duplicates in an arbitrary gather_index accumulate like torch.gather's backward."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, src, index, n_src_rows, inverse):
        lib = _bind()
        src = src.contiguous()
        rows = index.numel()
        H = src.size(-1)
        dst = torch.empty(rows, H, device=src.device, dtype=src.dtype)
        _lib.check(lib.ub200_gather_rows(src.data_ptr(), dst.data_ptr(), index.data_ptr(), rows,
                                         H * src.element_size(), _lib.current_stream()))
        ctx.n_src_rows = n_src_rows
        ctx.src_shape = src.shape
        ctx.has_inverse = inverse is not None
        ctx.save_for_backward(inverse if inverse is not None else index)
        return dst

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, grad):
        (index,) = ctx.saved_tensors
        grad = grad.contiguous()
        H = grad.size(-1)
        if ctx.has_inverse:
            lib = _bind()
            out = torch.empty(ctx.n_src_rows, H, device=grad.device, dtype=grad.dtype)
            _lib.check(lib.ub200_gather_rows(grad.data_ptr(), out.data_ptr(), index.data_ptr(),
                                             ctx.n_src_rows, H * grad.element_size(),
                                             _lib.current_stream()))
        else:
            out = torch.zeros(ctx.n_src_rows, H, device=grad.device, dtype=grad.dtype)
            valid = (index >= 0).unsqueeze(1)
            out.index_add_(0, index.clamp(min=0).long(), grad * valid)
        return out.view(ctx.src_shape), None, None, None


class LibLinear(torch.autograd.Function):
    """y = act(x W^T + b) with W [N, K] (an nn.Linear weight, `w_kn` False), or y = act(x W + b) with
    W [K, N] (`w_kn` True: the reference's `F.linear(h, weight.t(), bias)` of RegionFeatureRegression,
    model/pretrain.py:29-32, whose weight is the tied img_linear.weight) — forward, dgrad and wgrad on
    the wgmma GEMM (operands read un-transposed in every direction), bias gradient by ub200_colsum.
    act = tanh when `tanh` (BertPooler).  N may be any size (padded to 8 internally: ITM's 2
    classes, the 1601 region labels).  Parameters that live in a gradient arena get their gradients
    written there directly (None is returned to autograd); others are returned normally."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, x, weight, bias, w_kn, tanh):
        from . import ops
        if not x.is_cuda or x.dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError("libub200 heads need fp16/bf16 CUDA tensors (no fp32 / CPU fallback)")
        K = x.size(-1)
        x2 = x if x.dim() == 2 and x.stride(1) == 1 and x.stride(0) % 8 == 0 else x.reshape(-1, K).contiguous()
        N = weight.size(1) if w_kn else weight.size(0)
        Np = (N + 7) // 8 * 8
        w = weight if weight.is_contiguous() else weight.contiguous()
        if w_kn and Np != N:
            raise RuntimeError("LibLinear: a [K, N] weight needs N % 8 == 0")
        if bias is not None and Np != N:
            bias_p = torch.zeros(Np, device=x.device, dtype=x.dtype)
            bias_p[:N] = bias
        else:
            bias_p = bias
        out = torch.empty(x2.size(0), Np, device=x.device, dtype=x.dtype)
        ops.gemm(x2, w, b_major=1 if w_kn else 0, bias=bias_p, out=out, tanh=bool(tanh),
                 n_valid=N if Np != N else 0)
        ctx.save_for_backward(x2, w, out if tanh else None)
        ctx.meta = (bool(w_kn), bool(tanh), N, Np, weight, bias, x.shape)
        return out[:, :N] if Np != N else out

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, dy):
        from . import ops
        x2, w, y = ctx.saved_tensors
        w_kn, tanh, N, Np, weight, bias, x_shape = ctx.meta
        dtype = x2.dtype
        if Np != N or not dy.is_contiguous():
            d = torch.zeros(dy.size(0), Np, device=dy.device, dtype=dtype)
            d[:, :N] = dy
            dy = d
        if tanh:
            dy = ops.dtanh_mul(dy, y)
        dyv = dy[:, :N]                       # [n, N] view with row pitch Np
        arena = getattr(weight, "_ub_arena", None)
        if arena is not None and (id(weight) not in arena._views or not arena._still_valid()):
            arena = None
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            # dx = dy W (w [N, K]: B read as [K=N, N=K] b_major 1)  |  dx = dy W^T (w [K, N]: b_major 0)
            dx = ops.gemm(dyv, w, b_major=0 if w_kn else 1).view(x_shape)
        if weight.requires_grad:
            if arena is not None:
                arena.mark_managed([weight])
                acc = arena.claim([weight])
                tgt = arena.view(weight)
            else:
                acc, tgt = False, torch.empty_like(w)
            if w_kn:      # dW [K, N] = x^T dy
                ops.gemm(x2, dyv, a_major=1, b_major=1, out=tgt, accumulate=acc)
            else:         # dW [N, K] = dy^T x
                ops.gemm(dyv, x2, a_major=1, b_major=1, out=tgt, accumulate=acc)
            dw = None if arena is not None else tgt
        if bias is not None and bias.requires_grad:
            cs = ops.colsum(dy)[:N]
            if arena is not None and id(bias) in arena._views:
                arena.mark_managed([bias])
                ops.cvt_from_f32(cs, dtype, out=arena.view(bias), accumulate=arena.claim([bias]))
            else:
                db = ops.cvt_from_f32(cs, dtype)
        return dx, dw, db, None, None


class _EmbedFront(torch.autograd.Function):
    """Embedding front-end straight into packed rows (model/model.py:217-334) on libub200:
    ub200_embed_prep -> ub200_embed_gather_cast -> ub200_gemm (img_linear) -> ub200_embed_rows_fwd.
    Backward: row-kind masked ub200_layernorm_bwd x4, wgrad GEMM for img_linear, table scatter.

    The parameters are NOT autograd inputs: the kernels read them by pointer and the backward writes
    their gradients straight into the model's gradient arena (uniter_b200.arena) — `anchor` is the
    requires-grad handle that makes autograd call backward."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, anchor, model, meta, mode, input_ids, position_ids, img_feat, img_pos_feat,
                gather_index, img_masks, txt_type_ids, img_type_ids, dropout_p):
        from . import ops
        lib = _bind()
        te, ie = model.embeddings, model.img_embeddings
        word_w, pos_w, type_w = (te.word_embeddings.weight, te.position_embeddings.weight,
                                 te.token_type_embeddings.weight)
        T, L = meta["total"], meta["L"]
        dev, dtype = word_w.device, word_w.dtype
        H = word_w.size(1)
        dt = _lib.dtype_code(dtype)
        stream = _lib.current_stream()
        idx = torch.empty(6, T, device=dev, dtype=torch.int32)
        Lt = input_ids.size(1) if input_ids is not None else 0
        Li = img_feat.size(1) if img_feat is not None else 0
        if input_ids is not None:
            input_ids = input_ids.contiguous()
            position_ids = position_ids.contiguous()
        if img_masks is not None:
            img_masks = img_masks.to(torch.uint8).contiguous()
        a = _lib.EmbedPrepArgs(
            pack_idx=meta["pack_idx"].data_ptr(),
            gather_index=gather_index.contiguous().data_ptr() if mode == 0 else None,
            input_ids=_lib.ptr(input_ids), position_ids=_lib.ptr(position_ids),
            txt_type_ids=_lib.ptr(txt_type_ids.contiguous() if txt_type_ids is not None else None),
            img_type_ids=_lib.ptr(img_type_ids.contiguous() if img_type_ids is not None else None),
            img_masks=_lib.ptr(img_masks), T=T, L=L, Lt=Lt, Li=Li,
            pos_rows=position_ids.size(0) if position_ids is not None else 1, mode=mode,
            kind=idx[0].data_ptr(), word_id=idx[1].data_ptr(), pos_id=idx[2].data_ptr(),
            type_id=idx[3].data_ptr(), img_src=idx[4].data_ptr(), mask_flag=idx[5].data_ptr())
        _lib.check(lib.ub200_embed_prep(C.byref(a), stream))
        A = G = pos_feat = None
        if mode != 1:
            if img_feat.dtype not in (torch.float32, dtype):
                img_feat = img_feat.to(dtype)
            img_feat = img_feat.contiguous()
            D = img_feat.size(-1)
            A = torch.empty(T, D, device=dev, dtype=dtype)
            mask_row = ie.mask_embedding.weight[1].contiguous()
            _lib.check(lib.ub200_embed_gather_cast(
                img_feat.data_ptr(), 1 if img_feat.dtype == torch.float32 else 0, idx[4].data_ptr(),
                idx[5].data_ptr(), mask_row.data_ptr(), A.data_ptr(), T, D, dt, stream))
            G = ops.gemm(A, ie.img_linear.weight, bias=ie.img_linear.bias)   # img_linear on the wgmma core
            pos_feat = img_pos_feat.float().contiguous().view(-1, img_pos_feat.size(-1))
            assert pos_feat.size(1) == 7
        x = torch.empty(T, H, device=dev, dtype=dtype)
        u = torch.empty_like(x)
        ppre = torch.empty_like(x)
        seed, offset, rng_dev = _next_rng(dev)
        rng_stream = (offset << 20) | (0xFFFF << 4) | 4
        r = _lib.EmbedRowsArgs(
            kind=idx[0].data_ptr(), word_id=idx[1].data_ptr(), pos_id=idx[2].data_ptr(),
            type_id=idx[3].data_ptr(), img_src=idx[4].data_ptr(),
            word_emb=word_w.data_ptr(), pos_emb=pos_w.data_ptr(), type_emb=type_w.data_ptr(),
            ln_txt_g=te.LayerNorm.weight.data_ptr(), ln_txt_b=te.LayerNorm.bias.data_ptr(),
            img_linear_out=_lib.ptr(G), pos_feat=_lib.ptr(pos_feat),
            w_pos=ie.pos_linear.weight.contiguous().data_ptr(), b_pos=ie.pos_linear.bias.data_ptr(),
            ln_img_g=ie.img_layer_norm.weight.data_ptr(), ln_img_b=ie.img_layer_norm.bias.data_ptr(),
            ln_pos_g=ie.pos_layer_norm.weight.data_ptr(), ln_pos_b=ie.pos_layer_norm.bias.data_ptr(),
            ln_out_g=ie.LayerNorm.weight.data_ptr(), ln_out_b=ie.LayerNorm.bias.data_ptr(),
            x=x.data_ptr(), u=u.data_ptr(), ppre=ppre.data_ptr(), T=T, hidden=H, dtype=dt,
            dropout_p=float(dropout_p), rng_seed=seed, rng_stream=rng_stream, rng_offset_dev=rng_dev)
        _lib.check(lib.ub200_embed_rows_fwd(C.byref(r), stream))
        ctx.model = model
        ctx.mode, ctx.dropout_p, ctx.seed, ctx.rng_stream, ctx.rng_dev = mode, float(dropout_p), seed, rng_stream, rng_dev
        ctx.has_masks = img_masks is not None
        ctx.save_for_backward(idx, A, G, u, ppre, pos_feat)
        return x

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, dx):
        """Row-kind masked LayerNorm backward (x4), img_linear wgrad on the wgmma GEMM, then the
        table gradients in three launches (ub200_embed_bwd_scatter / _colsums); every small fp32
        gradient lives in ONE staging buffer whose layout equals the arena's front-end small section,
        so one launch converts (or accumulates) all of them into the parameters' .grad views."""
        from . import ops
        lib = _bind()
        model = ctx.model
        idx, A, G, u, ppre, pos_feat = ctx.saved_tensors
        te, ie = model.embeddings, model.img_embeddings
        arena, ep = model._ensure_arena()
        dx = dx.contiguous()
        T, H = dx.shape
        dtype, dev = dx.dtype, dx.device
        dt = _lib.dtype_code(dtype)
        stream = _lib.current_stream()
        kind, word_id, pos_id, type_id, img_src, mask_flag = (idx[i] for i in range(6))
        kw = dict(dropout_p=ctx.dropout_p, rng_seed=ctx.seed, rng_stream=ctx.rng_stream,
                  row_kind=kind, dropout_on_dy=ctx.dropout_p > 0, rng_offset_dev=ctx.rng_dev)
        has_txt, has_img = ctx.mode != 2, ctx.mode != 1
        # ---- one fp32 staging buffer for every small gradient (accumulated by the kernels)
        fs = ep["front_small"]                      # name -> (offset, numel) inside the small section
        S = torch.zeros(ep["front_small_n"], device=dev, dtype=torch.float32)
        sec = {k: S[o:o + n] for k, (o, n) in fs.items()}

        du = torch.empty_like(dx)        # every packed row is text or image: fully written below
        if has_txt:
            ops.layernorm_bwd(dx, u, te.LayerNorm.weight, kind=0, dx=du, want_dbias=False,
                              dgamma=sec["lnt_g"], dbeta=sec["lnt_b"], **kw)
        if has_img:
            ops.layernorm_bwd(dx, u, ie.LayerNorm.weight, kind=1, dx=du, want_dbias=False,
                              dgamma=sec["lnf_g"], dbeta=sec["lnf_b"], **kw)
        if has_txt:
            word = te.word_embeddings.weight
            d_word = arena.view(word)
            if not arena.claim([word]):      # first writer of this step: the scatter is additive
                d_word.zero_()
            _lib.check(lib.ub200_embed_bwd_scatter(du.data_ptr(), kind.data_ptr(), word_id.data_ptr(),
                                                   pos_id.data_ptr(), d_word.data_ptr(),
                                                   sec["pos"].data_ptr(), T, H, dt, stream))
        type_w = te.token_type_embeddings.weight
        ca = _lib.EmbedColsumArgs(x=du.data_ptr(), type_id=type_id.data_ptr(), out=sec["type"].data_ptr(),
                                  T=T, hidden=H, mode=0, type_vocab=type_w.size(0), dtype=dt)
        _lib.check(lib.ub200_embed_bwd_colsums(C.byref(ca), stream))
        if has_img:
            dG = torch.empty_like(dx)    # text rows are zeroed by the kernel (zero_inactive)
            dP = torch.empty_like(dx)
            ops.layernorm_bwd(du, G, ie.img_layer_norm.weight, row_kind=kind, kind=1, dx=dG, zero_inactive=True,
                              dgamma=sec["lni_g"], dbeta=sec["lni_b"], dbias=sec["img_b"])
            ops.layernorm_bwd(du, ppre, ie.pos_layer_norm.weight, row_kind=kind, kind=1, dx=dP, zero_inactive=True,
                              dgamma=sec["lnp_g"], dbeta=sec["lnp_b"], dbias=sec["posl_b"])
            # img_linear.weight [H, D] = dG^T A   (wgrad form: both operands read un-transposed)
            img_w = ie.img_linear.weight
            acc = arena.claim([img_w])
            ops.gemm(dG, A, a_major=1, b_major=1, out=arena.view(img_w), accumulate=acc)
            # pos_linear.weight [H, 7] = dP^T box  (K = T reduction with 7 weights per row)
            ca = _lib.EmbedColsumArgs(x=dP.data_ptr(), kind=kind.data_ptr(), img_src=img_src.data_ptr(),
                                      pos_feat=pos_feat.data_ptr(), out=sec["posl_w"].data_ptr(),
                                      T=T, hidden=H, mode=1, type_vocab=0, dtype=dt)
            _lib.check(lib.ub200_embed_bwd_colsums(C.byref(ca), stream))
            mask_w = ie.mask_embedding.weight
            if ctx.has_masks and mask_w.requires_grad:
                dA = ops.gemm(dG, img_w, b_major=1)                                 # [T, D]
                row = (dA.float() * (mask_flag != 0).unsqueeze(1)).sum(0).to(dtype)
                d_mask = arena.view(mask_w)
                if arena.claim([mask_w]):
                    d_mask[1].add_(row)
                else:
                    d_mask.zero_()
                    d_mask[1].copy_(row)
        # ---- fp32 -> model dtype straight into the arena's small section, one launch.  The section is
        # ordered [text-only | token_type | image-only], so the parameters a mode touches are one
        # contiguous range (text-only: prefix, image-only: suffix) and the others are left alone.
        names = ep["front_small_order"]
        first = 0 if has_txt else names.index("type")
        last = len(names) - 1 if has_img else names.index("type")
        used = ep["front_small_params"][first:last + 1]
        acc = arena.claim(used)
        r_lo = fs[names[first]][0]
        r_hi = fs[names[last]][0] + fs[names[last]][1]
        lo, _ = ep["segments"]["front_small"]
        dst = arena.flat[lo + r_lo:lo + r_hi]
        _lib.check(lib.ub200_cvt_from_f32_strided(S[r_lo:].data_ptr(), dst.data_ptr(), r_hi - r_lo, 1, 0, 0,
                                                  1 if acc else 0, dt, stream))
        return (None,) * 13


class _EncoderStack(torch.autograd.Function):
    """NL x BertLayer over packed tokens: one C-ABI call forward, one backward."""

    @staticmethod
    @_lib.forward_in_mode(
        lambda ctx, x, anchor, model, meta, want_all, need_grad: meta["max_seqlen"] if need_grad else None)
    def forward(ctx, x, anchor, model, meta, want_all, need_grad):
        lib = _bind()
        cfg = model.config
        T, H = x.shape
        NL = cfg.num_hidden_layers
        training = model.training
        p_hidden = float(model.encoder.layer[0].output.dropout.p) if training else 0.0
        p_attn = float(model.encoder.layer[0].attention.self.dropout.p) if training else 0.0
        seed, offset, rng_dev = _next_rng(x.device)
        desc = _EncoderDesc(
            hidden=H, intermediate=cfg.intermediate_size, num_heads=cfg.num_attention_heads,
            num_layers=NL, dtype=_lib.dtype_code(x.dtype), batch=meta["batch"], total_tokens=T,
            max_seqlen=meta["max_seqlen"], cu_seqlens=meta["cu_seqlens"].data_ptr(),
            hidden_dropout_p=p_hidden, attn_dropout_p=p_attn,
            rng_seed=seed, rng_offset=offset, rng_offset_dev=rng_dev)
        weights = model._weight_table()
        act_bytes = lib.ub200_encoder_act_bytes_per_layer(C.byref(desc))
        act = torch.empty((NL if need_grad else 1) * act_bytes, device=x.device, dtype=torch.uint8)
        outs = torch.empty(NL, T, H, device=x.device, dtype=x.dtype)
        out_ptrs = (C.c_void_p * NL)(*[outs[l].data_ptr() for l in range(NL)])
        x = x.contiguous()
        _lib.check(lib.ub200_encoder_fwd(C.byref(desc), weights, x.data_ptr(), out_ptrs,
                                         act.data_ptr(), 1 if need_grad else 0,
                                         _lib.current_stream()))
        if need_grad:
            model._fwd_since_reduce = getattr(model, "_fwd_since_reduce", 0) + 1
        ctx.model = model
        ctx.desc = desc
        ctx.meta = meta
        ctx.want_all = want_all
        ctx.save_for_backward(x, outs, act)
        ctx.out_ptrs = out_ptrs
        if want_all:
            return outs
        return outs[NL - 1]

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, grad_out):
        lib = _bind()
        model = ctx.model
        x, outs, act = ctx.saved_tensors
        desc = ctx.desc
        NL = desc.num_layers
        T, H = x.shape
        grad_out = grad_out.contiguous()
        arena, ep = model._ensure_arena()
        grads = ep["gtable"]
        ep["small32"].zero_()
        weights = model._weight_table()
        scratch = torch.empty(lib.ub200_encoder_bwd_scratch_bytes(C.byref(desc)), device=x.device,
                              dtype=torch.uint8)
        act_bytes = lib.ub200_encoder_act_bytes_per_layer(C.byref(desc))
        stream = _lib.current_stream()
        hook = getattr(model, "_bwd_chunk_hook", None)
        nchunks = max(1, min(NL, int(getattr(model, "_bwd_chunks", 1)))) if hook is not None else 1
        bounds = [round(i * NL / nchunks) for i in range(nchunks + 1)]
        # the backward is issued in chunks of layers (top chunk first) so that a data-parallel
        # reducer can start all-reducing a chunk's gradients while the next chunk is computing
        dtop = grad_out[NL - 1] if ctx.want_all else grad_out
        for ci in range(nchunks - 1, -1, -1):
            lo, hi = bounds[ci], bounds[ci + 1]
            n = hi - lo
            accumulate = arena.claim([q for lp in ep["layer_params"][lo:hi] for q in lp])
            d = _EncoderDesc.from_buffer_copy(desc)
            d.num_layers, d.layer_offset = n, lo
            d_ptrs = (C.c_void_p * n)()
            if ctx.want_all:
                for l in range(lo, hi - 1):
                    d_ptrs[l - lo] = grad_out[l].data_ptr()
            d_ptrs[n - 1] = dtop.data_ptr()
            x_in = x if lo == 0 else outs[lo - 1]
            dx = torch.empty_like(x)
            out_ptrs = (C.c_void_p * n)(*[outs[l].data_ptr() for l in range(lo, hi)])
            _lib.check(lib.ub200_encoder_bwd(
                C.byref(d), C.byref(weights[lo]), C.byref(grads[lo]), x_in.data_ptr(), out_ptrs,
                act.data_ptr() + lo * act_bytes, d_ptrs, dx.data_ptr(), scratch.data_ptr(),
                1 if accumulate else 0, stream))
            if lo > 0 and ctx.want_all:
                dx = dx + grad_out[lo - 1]
            dtop = dx
            model._finish_grads(accumulate, lo, hi)
            if hook is not None:
                hook(model, lo, hi)
        return dtop, None, None, None, None, None


# ============================================================================ the model
class UniterModel(UniterPreTrainedModel):
    """Joint vision-language encoder — same constructor / forward as model/model.py:295-367."""

    def __init__(self, config, img_dim):
        super().__init__(config)
        if config.hidden_size != 64 * config.num_attention_heads:
            raise ValueError("libub200 attention kernels need head_dim 64 (hidden_size=%d, heads=%d)"
                             % (config.hidden_size, config.num_attention_heads))
        self.embeddings = UniterTextEmbeddings(config)
        self.img_embeddings = UniterImageEmbeddings(config, img_dim)
        self.encoder = UniterEncoder(config)
        self.pooler = BertPooler(config)
        self.apply(self.init_weights)
        self._packed_key = None
        self._wtable = None
        self._arena = None

    # ------------------------------------------------------------------ parameter / gradient arenas
    _BIG = ("wqkv", "wo", "w1", "w2")

    def _layer_params(self, layer):
        a, o = layer.attention, layer.output
        return dict(q_w=a.self.query.weight, k_w=a.self.key.weight, v_w=a.self.value.weight,
                    q_b=a.self.query.bias, k_b=a.self.key.bias, v_b=a.self.value.bias,
                    wo=a.output.dense.weight, bo=a.output.dense.bias,
                    ln1_g=a.output.LayerNorm.weight, ln1_b=a.output.LayerNorm.bias,
                    w1=layer.intermediate.dense.weight, b1=layer.intermediate.dense.bias,
                    w2=o.dense.weight, b2=o.dense.bias, ln2_g=o.LayerNorm.weight,
                    ln2_b=o.LayerNorm.bias)

    def _weight_table(self):
        """ctypes array of per-layer weight pointers.  query/key/value are re-homed (once, and
        again after any ``.half()`` / ``.to()`` that re-allocates them) as views of one [3H, H]
        and one [3H] buffer so the fused QKV projection reads them in place."""
        layers = self.encoder.layer
        key = tuple(l.attention.self.query.weight.data_ptr() for l in layers) + \
            tuple(l.output.dense.weight.data_ptr() for l in layers)
        if self._wtable is not None and key == self._packed_key:
            return self._wtable
        H = self.config.hidden_size
        table = (_LayerWeights * len(layers))()
        p0 = layers[0].attention.self.query.weight
        if not p0.is_cuda or p0.dtype not in (torch.float16, torch.bfloat16):
            raise RuntimeError("UniterModel (libub200) needs fp16/bf16 parameters on a CUDA device "
                               "(got %s on %s); call .cuda().half() or .bfloat16() — there is no "
                               "fp32 / CPU fallback" % (p0.dtype, p0.device))
        for i, layer in enumerate(layers):
            P = self._layer_params(layer)
            qw, kw, vw = P["q_w"], P["k_w"], P["v_w"]
            nb = qw.numel() * qw.element_size()
            contiguous = (kw.data_ptr() == qw.data_ptr() + nb and vw.data_ptr() == kw.data_ptr() + nb)
            if not contiguous:
                buf = torch.cat([qw.data, kw.data, vw.data], 0)  # [3H, H]
                qw.data, kw.data, vw.data = buf[:H], buf[H:2 * H], buf[2 * H:]
            qb, kb, vb = P["q_b"], P["k_b"], P["v_b"]
            nb = qb.numel() * qb.element_size()
            if not (kb.data_ptr() == qb.data_ptr() + nb and vb.data_ptr() == kb.data_ptr() + nb):
                buf = torch.cat([qb.data, kb.data, vb.data], 0)
                qb.data, kb.data, vb.data = buf[:H], buf[H:2 * H], buf[2 * H:]
            t = table[i]
            t.wqkv, t.bqkv = qw.data_ptr(), qb.data_ptr()
            for name in ("wo", "bo", "ln1_g", "ln1_b", "w1", "b1", "w2", "b2", "ln2_g", "ln2_b"):
                if not P[name].is_contiguous():
                    P[name].data = P[name].data.contiguous()
                setattr(t, name, P[name].data_ptr())
        self._wtable = table
        self._packed_key = tuple(l.attention.self.query.weight.data_ptr() for l in layers) + \
            tuple(l.output.dense.weight.data_ptr() for l in layers)
        return table

    # The gradient arena (uniter_b200.arena.GradArena) owns ONE flat buffer for every parameter of
    # the root module it was attached to; the encoder contributes its library layout to the plan.
    def _plan_arena(self, off):
        """Element offsets of this model's parameters inside a GradArena starting at `off`."""
        lib = _bind()
        cfg = self.config
        H, I, NL = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
        plan, seg = [], {}

        def put(p, o):
            plan.append((p, o, p.numel()))

        def a8(n):
            return (n + 7) // 8 * 8
        # ---- pooler (its backward runs before the encoder's)
        lo = off
        for p in self.pooler.parameters():
            put(p, off)
            off += a8(p.numel())
        seg["pooler"] = (lo, off)
        # ---- encoder layers, library layout (ub200_layer_grads)
        small_n = lib.ub200_encoder_small_grad_count(H, I)
        big_n = 3 * H * H + H * H + I * H + H * I
        per_layer = a8(big_n + small_n)
        layer0 = off
        layer_params = []
        for i, layer in enumerate(self.encoder.layer):
            P = self._layer_params(layer)
            o = layer0 + i * per_layer
            put(P["q_w"], o); put(P["k_w"], o + H * H); put(P["v_w"], o + 2 * H * H); o += 3 * H * H
            put(P["wo"], o); o += H * H
            put(P["w1"], o); o += I * H
            put(P["w2"], o); o += H * I
            for name, n in (("q_b", H), ("k_b", H), ("v_b", H), ("bo", H), ("ln1_g", H), ("ln1_b", H),
                            ("b1", I), ("b2", H), ("ln2_g", H), ("ln2_b", H)):
                put(P[name], o)
                o += n
            layer_params.append([P[k] for k in ("q_w", "k_w", "v_w", "wo", "w1", "w2", "q_b", "k_b", "v_b",
                                                "bo", "ln1_g", "ln1_b", "b1", "b2", "ln2_g", "ln2_b")])
        off = layer0 + NL * per_layer
        seg["layers"] = (layer0, off)
        # ---- embedding front-end: big tables, then the small section in staging-buffer order
        te, ie = self.embeddings, self.img_embeddings
        lo = off
        for p in (te.word_embeddings.weight, ie.img_linear.weight, ie.mask_embedding.weight):
            put(p, off)
            off += a8(p.numel())
        small_lo = off
        order = [("pos", te.position_embeddings.weight), ("lnt_g", te.LayerNorm.weight),
                 ("lnt_b", te.LayerNorm.bias), ("type", te.token_type_embeddings.weight),
                 ("lnf_g", ie.LayerNorm.weight), ("lnf_b", ie.LayerNorm.bias),
                 ("lni_g", ie.img_layer_norm.weight), ("lni_b", ie.img_layer_norm.bias),
                 ("lnp_g", ie.pos_layer_norm.weight), ("lnp_b", ie.pos_layer_norm.bias),
                 ("img_b", ie.img_linear.bias), ("posl_b", ie.pos_linear.bias),
                 ("posl_w", ie.pos_linear.weight)]
        front_small = {}
        for name, p in order:       # H % 8 == 0 for every entry (H * 7 included): no padding inside
            put(p, off)
            front_small[name] = (off - small_lo, p.numel())
            off += p.numel()
        front_small_n = off - small_lo
        off = a8(off)
        seg["front"] = (lo, off)
        seg["front_small"] = (small_lo, small_lo + front_small_n)
        return dict(plan=plan, segments=seg, end=off, per_layer=per_layer, layer0=layer0, big_n=big_n,
                    small_n=small_n, layer_params=layer_params, front_small=front_small,
                    front_small_n=front_small_n, front_small_params=[p for _, p in order],
                    front_small_order=[n for n, _ in order])

    def _bind_arena(self, arena, ep):
        """Called by GradArena once its flat buffer exists: pointer tables for the C ABI."""
        NL = self.config.num_hidden_layers
        H, I = self.config.hidden_size, self.config.intermediate_size
        flat = arena.flat
        es = flat.element_size()
        small32 = torch.zeros(NL * ep["small_n"], device=flat.device, dtype=torch.float32)
        gtable = (_LayerGrads * NL)()
        for i in range(NL):
            base = flat.data_ptr() + (ep["layer0"] + i * ep["per_layer"]) * es
            g = gtable[i]
            g.dwqkv = base
            g.dwo = base + 3 * H * H * es
            g.dw1 = g.dwo + H * H * es
            g.dw2 = g.dw1 + I * H * es
            g.small = small32[i * ep["small_n"]:(i + 1) * ep["small_n"]].data_ptr()
        ep["gtable"], ep["small32"] = gtable, small32
        te, ie = self.embeddings, self.img_embeddings
        managed = [q for lp in ep["layer_params"] for q in lp] + ep["front_small_params"] + \
            [te.word_embeddings.weight, ie.img_linear.weight, ie.mask_embedding.weight] + \
            list(self.pooler.parameters())
        arena.mark_managed(managed)
        self._arena = (arena, ep)

    def _ensure_arena(self):
        """(arena, this model's plan).  Built lazily over this model alone unless a larger root was
        attached with GradArena.attach(root) (bench / GraphedStep / GradientReducer do that so that
        the task head's gradients live in the same flat buffer)."""
        from .arena import GradArena
        if self.encoder.layer[0].attention.self.query.weight.is_cuda:
            self._weight_table()           # (CPU: host-side bookkeeping only, e.g. the gloo / arena tests)
        if self._arena is None or not self._arena[0]._still_valid():
            self._arena = None
            GradArena(self)                      # binds itself through _bind_arena
        return self._arena

    def grad_arena(self):
        """The flat gradient buffer this model's parameters live in (what gets all-reduced)."""
        return self._ensure_arena()[0].flat

    def _finish_grads(self, accumulate, lo=0, hi=None):
        """fp32 -> 16-bit for the small (bias / LayerNorm) gradients of layers [lo, hi)."""
        lib = _bind()
        arena, ep = self._arena
        NL = self.config.num_hidden_layers
        hi = NL if hi is None else hi
        flat, small32, n = arena.flat, ep["small32"], ep["small_n"]
        dt = _lib.dtype_code(flat.dtype)
        dst0 = flat[ep["layer0"] + lo * ep["per_layer"] + ep["big_n"]:]
        _lib.check(lib.ub200_cvt_from_f32_strided(small32[lo * n:].data_ptr(), dst0.data_ptr(), n, hi - lo,
                                                  n, ep["per_layer"], 1 if accumulate else 0, dt,
                                                  _lib.current_stream()))

    def arena_slice(self, lo, hi):
        """Flat gradient slice of encoder layers [lo, hi) (contiguous)."""
        arena, ep = self._ensure_arena()
        return arena.flat[ep["layer0"] + lo * ep["per_layer"]:ep["layer0"] + hi * ep["per_layer"]]

    # ------------------------------------------------------------------ embeddings (reference API)
    def _compute_txt_embeddings(self, input_ids, position_ids, txt_type_ids=None):
        return self.embeddings(input_ids, position_ids, txt_type_ids)

    def _compute_img_embeddings(self, img_feat, img_pos_feat, img_masks=None, img_type_ids=None):
        if img_type_ids is None:
            img_type_ids = torch.ones_like(img_feat[:, :, 0].long())
        img_type_embeddings = self.embeddings.token_type_embeddings(img_type_ids)
        return self.img_embeddings(img_feat, img_pos_feat, img_type_embeddings, img_masks)

    def _compute_img_txt_embeddings(self, input_ids, position_ids, img_feat, img_pos_feat,
                                    gather_index, img_masks=None, txt_type_ids=None,
                                    img_type_ids=None):
        """Padded [B, L, H] result with the reference's semantics (model/model.py:321-334); the
        forward pass below never materialises it (it gathers straight into packed rows)."""
        txt_emb = self._compute_txt_embeddings(input_ids, position_ids, txt_type_ids)
        img_emb = self._compute_img_embeddings(img_feat, img_pos_feat, img_masks, img_type_ids)
        cat = torch.cat([txt_emb, img_emb], dim=1)
        B, Lc, H = cat.shape
        flat_idx = (gather_index + torch.arange(B, device=cat.device).unsqueeze(1) * Lc).reshape(-1)
        out = _GatherRows.apply(cat.reshape(B * Lc, H), flat_idx.to(torch.int32).contiguous(), B * Lc, None)
        return out.view(B, gather_index.size(1), H)

    # ------------------------------------------------------------------ packing metadata
    @staticmethod
    def _pack_meta(attention_mask):
        """Valid-token bookkeeping from the [B, L] attention mask (prefix masks in every reference
        collate, but any 0/1 pattern is honoured: valid tokens are packed in order).

        Needs the per-sample lengths on the host (they size the launches).  They come from, in
        order: lengths registered by `register_lengths` (the host-side loader knows them before
        the H2D copy — no sync), a cache hit on the same mask tensor (e.g. the 400-pair eval +
        32-pair train forwards of model/itm.py:82-88 reuse it), or one small device->host read
        (the reference itself syncs every step, train_vqa.py:201)."""
        B, L = attention_mask.shape
        hit = _meta_lookup(attention_mask)
        if hit is not None and "cu_seqlens" in hit:
            return hit
        dev = attention_mask.device
        registered = hit is not None
        if registered and hit.get("prefix"):
            # prefix masks with host-known lengths: the whole bookkeeping (cu_seqlens, pack and
            # unpack indices) is integer arithmetic done on the HOST and shipped in one small H2D
            # copy — no device reads, no index kernels
            lens_h = hit["lens_host"]
            host, offs, T = _prefix_pack_host(lens_h, L)
            devbuf = _META_RING.upload(host, dev)
            meta = _meta_from_buffer(devbuf, offs, B, L, T, max(lens_h) if lens_h else 0, lens_h, False)
            _meta_store(attention_mask, meta)
            return meta
        else:
            am = attention_mask != 0
            lens = am.sum(1)
            if registered:
                lens_h = hit["lens_host"]             # registered by the loader: no sync
            else:
                lens_h = lens.tolist()                # host sync (B integers)
            T = int(sum(lens_h))
            cu = torch.zeros(B + 1, device=dev, dtype=torch.int32)
            cu[1:] = torch.cumsum(lens, 0)
            # [T] -> b*L+j ; size is known from the host-side lengths, so no second sync
            pack_idx = torch.nonzero_static(am.reshape(-1), size=T).squeeze(1).to(torch.int32)
        unpack_ext = torch.full((B * L + 1,), -1, device=dev, dtype=torch.int32)
        unpack_ext[pack_idx.long()] = torch.arange(T, device=dev, dtype=torch.int32)
        meta = dict(batch=B, L=L, total=T, max_seqlen=max(lens_h) if lens_h else 0,
                    cu_seqlens=cu, pack_idx=pack_idx, pack_inv=pack_idx, unpack_idx=unpack_ext[:B * L],
                    unpack_ext=unpack_ext, lens_host=lens_h, n_batch=B)
        _meta_store(attention_mask, meta)
        return meta

    # ------------------------------------------------------------------ forward
    def encode_packed(self, input_ids, position_ids, img_feat, img_pos_feat, attention_mask,
                      gather_index=None, img_masks=None, output_all_encoded_layers=False,
                      txt_type_ids=None, img_type_ids=None):
        """Same computation as forward() but returns the PACKED result and its bookkeeping:
        (out, meta) with out [T, H] (or [NL, T, H]) over the valid tokens only and
        meta["unpack_idx"] mapping a flat position b * L + j of the reference's [B, L] view to its
        packed row (-1 at masked positions).  Heads that only read a few rows (MLM / MRM masked
        positions, model/pretrain.py:129-133; the pooler's [:, 0]) gather them from here instead
        of materialising the padded [B, L, H] tensor."""
        self._weight_table()  # validates dtype/device, packs q/k/v
        meta = self._pack_meta(attention_mask)
        if meta["total"] == 0:
            raise ValueError("attention_mask selects no tokens")
        B, L = meta["n_batch"], meta["L"]
        # ---- embeddings (model/model.py:347-360) computed straight into PACKED rows by libub200
        if input_ids is None:
            mode = 2
            if img_feat.size(1) != L:
                raise ValueError("attention_mask length %d != number of regions %d" % (L, img_feat.size(1)))
        elif img_feat is None:
            mode = 1
            if input_ids.size(1) != L:
                raise ValueError("attention_mask length %d != text length %d" % (L, input_ids.size(1)))
        else:
            mode = 0
            if gather_index is None or gather_index.shape != (B, L):
                raise ValueError("gather_index must be [B, L] like attention_mask")
        te, ie = self.embeddings, self.img_embeddings
        if self.training and te.dropout.p != ie.dropout.p:
            raise NotImplementedError("text / image embedding dropout probabilities differ")
        if img_masks is not None:
            ie.mask_embedding.weight.data[0, :].fill_(0)          # model/model.py:263
        if not hasattr(self, "_anchor") or self._anchor.device != attention_mask.device:
            self._anchor = torch.zeros(1, device=attention_mask.device, requires_grad=True)
        x = _EmbedFront.apply(
            self._anchor, self, meta, mode, input_ids, position_ids, img_feat, img_pos_feat, gather_index,
            img_masks, txt_type_ids, img_type_ids, te.dropout.p if self.training else 0.0)  # [T, H] packed

        # ---- encoder stack on packed tokens
        # (grad mode is always off inside Function.forward, so decide here whether the backward
        #  will need the per-layer activations)
        out = _EncoderStack.apply(x, self._anchor, self, meta, bool(output_all_encoded_layers),
                                  torch.is_grad_enabled())
        return out, meta

    def forward(self, input_ids, position_ids, img_feat, img_pos_feat, attention_mask,
                gather_index=None, img_masks=None, output_all_encoded_layers=True,
                txt_type_ids=None, img_type_ids=None):
        out, meta = self.encode_packed(input_ids, position_ids, img_feat, img_pos_feat, attention_mask,
                                       gather_index, img_masks, output_all_encoded_layers,
                                       txt_type_ids, img_type_ids)
        B, L = meta["n_batch"], meta["L"]
        H = self.config.hidden_size
        # ---- back to the reference's padded [B, L, H] view (zeros at masked positions)
        if output_all_encoded_layers:
            return [_GatherRows.apply(out[l], meta["unpack_idx"], meta["total"],
                                      meta["pack_inv"]).view(B, L, H) for l in range(out.size(0))]
        return _GatherRows.apply(out, meta["unpack_idx"], meta["total"], meta["pack_inv"]).view(B, L, H)


def gather_packed_rows(packed, rows):
    """packed[rows] with zeros where rows < 0 (int32 [n]); differentiable.  The backward is itself
    a row gather through the inverse map, so neither direction needs atomics or a sync.
    `rows` must not contain a packed row twice (true for MLM / MRM positions and [CLS] rows): the
    inverse map keeps one entry per packed row, a duplicate's gradient would be dropped — use
    `_GatherRows.apply(packed, rows, T, None)` (scatter-add backward) for arbitrary index lists."""
    T = packed.size(0)
    n = rows.numel()
    inv = torch.full((T + 1,), -1, device=packed.device, dtype=torch.int32)
    slot = torch.where(rows >= 0, rows, torch.full_like(rows, T)).long()
    inv[slot] = torch.arange(n, device=packed.device, dtype=torch.int32)
    return _GatherRows.apply(packed, rows.contiguous(), T, inv[:T].contiguous())
