"""Callers of the hot path: the reference's task heads on top of the drop-in `UniterModel`.

Parameter names and module trees follow the reference so its checkpoints load
(`uniter.*`, `cls.predictions.*`, `vqa_output.*`, `itm_output.*`, `rank_output.*`):

* ``UniterForMLM`` — the MLM branch of ``UniterForPretraining`` (model/pretrain.py:50-60,
  107-133).  SURVEY.md §8f-1: the head runs on libub200 — masked rows are gathered straight from
  the PACKED encoder output, ``BertPredictionHeadTransform`` (model/layer.py:188-203) is the
  wgmma GEMM with the bias+GELU epilogue + the LayerNorm kernel, the tied decoder
  (model/layer.py:206-222) is the same GEMM over the un-padded [V, H] embedding table
  (``n_valid``), and the cross-entropy is one fused kernel per direction; the decoder's dgrad
  (few output tiles, K = V = 28996) runs split-K.
* ``UniterForVisualQuestionAnswering`` (model/vqa.py:16-52) and ``UniterForImageTextRetrieval``
  (model/itm.py:14-59): pooler + small classifier, plain torch on top of the encoder — they are
  here so the parity tests can check head-level logits against the reference's goldens.
* ``UniterForReferringExpressionComprehension`` (model/re.py): the region rows gathered from the
  packed output, scored and turned into the per-sample loss by one fused kernel per direction.
* ``UniterForVisualCommonsenseReasoning`` (model/vcr.py): the [CLS] rows gathered from the packed output,
  the library pooler, LibTransform(act="relu") at twice the hidden size and LibLinear with N = 2.
"""
import random
from collections import defaultdict

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import _lib, ops
from .model import LibLinear, UniterModel, UniterPreTrainedModel, gather_packed_rows


class GELU(nn.Module):
    """model/layer.py:40-42 (erf form)."""

    def forward(self, x):
        return F.gelu(x)


def gelu(x):
    return F.gelu(x)  # erf form, == model/layer.py:31-37


class BertPredictionHeadTransform(nn.Module):
    """model/layer.py:188-203 (parameter container; the fused head reads the weights by pointer)."""

    def __init__(self, config):
        super().__init__()
        self.dense = nn.Linear(config.hidden_size, config.hidden_size)
        self.LayerNorm = nn.LayerNorm(config.hidden_size, eps=1e-12)


class BertLMPredictionHead(nn.Module):
    """model/layer.py:206-222 — decoder weight tied to the word embeddings."""

    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.transform = BertPredictionHeadTransform(config)
        self.decoder = nn.Linear(bert_model_embedding_weights.size(1),
                                 bert_model_embedding_weights.size(0), bias=False)
        self.decoder.weight = bert_model_embedding_weights
        self.bias = nn.Parameter(torch.zeros(bert_model_embedding_weights.size(0)))


class BertOnlyMLMHead(nn.Module):
    def __init__(self, config, bert_model_embedding_weights):
        super().__init__()
        self.predictions = BertLMPredictionHead(config, bert_model_embedding_weights)


_PAD_LOGIT = -30000.0   # finite in fp16 and bf16; exp(pad - max) underflows to exactly 0


class _MlmHead(torch.autograd.Function):
    """scores = decoder(LayerNorm(gelu(dense(h)))) + bias ; loss = cross_entropy(scores, targets)
    on libub200.  Returns the per-row loss (fp32) or, with ``want_scores``, the [n, V] scores.
    Rows whose target is outside [0, V) (padding of a fixed-size index list) get loss 0 and
    contribute no gradient.  The head's parameters are read by pointer and their gradients are
    written straight into the gradient arena (the tied decoder / word-embedding gradient is one
    buffer that the decoder wgrad writes first and the embedding scatter adds to later)."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, h, module, targets, want_scores):
        p = module.cls.predictions
        dense_w, dense_b = p.transform.dense.weight, p.transform.dense.bias
        ln_g, ln_b = p.transform.LayerNorm.weight, p.transform.LayerNorm.bias
        word_w, dec_bias = p.decoder.weight, p.bias
        n, H = h.shape
        V = word_w.size(0)
        Vp = (V + 7) // 8 * 8
        dtype = h.dtype
        t, pre = ops.gemm(h, dense_w, bias=dense_b, gelu=True)        # model/layer.py:199-200
        z = ops.layernorm_fwd(t, ln_g, ln_b)                         # :201
        if Vp != V:
            bias_p = torch.full((Vp,), _PAD_LOGIT, device=h.device, dtype=dtype)
            bias_p[:V] = dec_bias
        else:
            bias_p = dec_bias
        logits = torch.empty(n, Vp, device=h.device, dtype=dtype)
        ops.gemm(z, word_w, bias=bias_p, out=logits, n_valid=V if Vp != V else 0)   # :220-221
        if want_scores:           # validation path (compute_loss=False): forward only
            scores = logits[:, :V]
            ctx.mark_non_differentiable(scores)
            return scores
        targets = targets.contiguous()
        loss, lse = ops.ce_fwd(logits, targets, V)                    # model/pretrain.py:122-125
        ctx.save_for_backward(h, pre, t, z, logits, lse, targets)
        ctx.V = V
        ctx.module = module
        return loss

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, dloss):
        from .arena import GradArena
        h, pre, t, z, logits, lse, targets = ctx.saved_tensors
        module = ctx.module
        p = module.cls.predictions
        dense_w, dense_b = p.transform.dense.weight, p.transform.dense.bias
        ln_g, ln_b = p.transform.LayerNorm.weight, p.transform.LayerNorm.bias
        word_w, dec_bias = p.decoder.weight, p.bias
        arena = GradArena.for_params(module, dense_w)
        arena.mark_managed([dense_w, dense_b, ln_g, ln_b, dec_bias])
        V = ctx.V
        dtype = h.dtype
        # the scores are dead after this point: the gradient overwrites them
        dlog = ops.ce_bwd_(logits, targets, lse, dloss.contiguous().float(), V)
        dlv = dlog[:, :V]                                             # [n, V], row pitch Vp
        # dz = dlog W_dec: 2 x (H / 128) output tiles, K = V -> split-K over the SMs (fp32 atomics)
        dz = ops.cvt_from_f32(ops.gemm(dlv, word_w, b_major=1, k_splits=-1), dtype)
        acc = arena.claim([word_w])
        ops.gemm(dlv, z, a_major=1, b_major=1, out=arena.view(word_w), accumulate=acc)   # [V, H] = dlog^T z
        dt, _, dg, db, _ = ops.layernorm_bwd(dz, t, ln_g, want_dbias=False)
        dpre = ops.dgelu_mul(dt, pre)
        dh = ops.gemm(dpre, dense_w, b_major=1)
        acc = arena.claim([dense_w, dense_b, ln_g, ln_b, dec_bias])
        ops.gemm(dpre, h, a_major=1, b_major=1, out=arena.view(dense_w), accumulate=acc)
        ops.cvt_from_f32(ops.colsum(dpre), dtype, out=arena.view(dense_b), accumulate=acc)
        ops.cvt_from_f32(dg, dtype, out=arena.view(ln_g), accumulate=acc)
        ops.cvt_from_f32(db, dtype, out=arena.view(ln_b), accumulate=acc)
        ops.cvt_from_f32(ops.colsum(dlog)[:V], dtype, out=arena.view(dec_bias), accumulate=acc)
        return dh, None, None, None


class UniterForMLM(UniterPreTrainedModel):
    """The MLM branch of UniterForPretraining (model/pretrain.py:50-60, 107-133)."""

    def __init__(self, config, img_dim):
        super().__init__(config)
        self.uniter = UniterModel(config, img_dim)
        self.cls = BertOnlyMLMHead(config, self.uniter.embeddings.word_embeddings.weight)
        self.apply(self.init_weights)

    def forward(self, batch, compute_loss=True):
        """Per-masked-token loss [n] (fp32), or the scores [n, V].  With loader-provided
        `mlm_index` (flat positions b * L + j; entries equal to B * L and targets of -1 are PADDING
        of a fixed-size list: zero rows, zero loss, no gradient) nothing here depends on data on
        the device, so the step can be captured in a CUDA graph."""
        batch = defaultdict(lambda: None, batch)
        input_ids = batch["input_ids"]
        packed, meta = self.uniter.encode_packed(
            input_ids, batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False,
            txt_type_ids=batch["txt_type_ids"])
        L = meta["L"]
        if batch["mlm_index"] is not None:
            # loader-provided flat positions (b * L + j) of the masked tokens: static shapes, no sync
            flat, targets = batch["mlm_index"], batch["mlm_targets"]
        else:
            # model/pretrain.py:115-118,129-133: text part only, rows where txt_labels != -1
            txt_labels = batch["txt_labels"]
            pos = (txt_labels != -1).nonzero(as_tuple=False)           # device sync, like the reference
            flat = pos[:, 0] * L + pos[:, 1]
            targets = txt_labels[pos[:, 0], pos[:, 1]]
        if flat.numel() == 0:
            V = self.uniter.config.vocab_size
            return packed.new_zeros(0, dtype=torch.float32) if compute_loss else packed.new_zeros(0, V)
        rows = meta["unpack_ext"][flat]                                # packed row of each masked token
        masked_output = gather_packed_rows(packed, rows)               # [n, H]
        return _MlmHead.apply(masked_output, self, targets, not compute_loss)


class LibTransform(torch.autograd.Function):
    """z = LayerNorm(act(h W^T + b)) on libub200, with act = "gelu" (default) or "relu".

    gelu: BertPredictionHeadTransform (model/layer.py:188-203) and the `net.0 / net.1 / net.2` prefix of
    RegionFeatureRegression / RegionClassification (model/pretrain.py:19-47): GEMM with the bias + GELU
    epilogue, LayerNorm kernels, dGELU kernel, dgrad / wgrad GEMMs.
    relu: the `vcr_output.0 / .1 / .2` prefix of the VCR head (model/vcr.py:27-32), Linear(H, 2H) ->
    ReLU -> LayerNorm(2H): GEMM with the plain bias epilogue, then the LayerNorm kernels with the ReLU
    applied as they load `pre`; their backward also writes dpre = dx o (pre > 0) and its column sums
    (the Linear's bias gradient).

    Gradients of parameters that live in a gradient arena are written there directly."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, h, dense_w, dense_b, ln_g, ln_b, act="gelu"):
        if act not in ("gelu", "relu"):
            raise ValueError("LibTransform: act must be 'gelu' or 'relu', got %r" % (act,))
        h = h.contiguous()
        if act == "relu":
            pre = ops.gemm(h, dense_w, bias=dense_b)
            t = pre
            z = ops.layernorm_fwd(pre, ln_g, ln_b, relu=True)
        else:
            t, pre = ops.gemm(h, dense_w, bias=dense_b, gelu=True)
            z = ops.layernorm_fwd(t, ln_g, ln_b)
        ctx.save_for_backward(h, pre, t)
        ctx.params = (dense_w, dense_b, ln_g, ln_b)
        ctx.act = act
        return z

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, dz):
        h, pre, t = ctx.saved_tensors
        dense_w, dense_b, ln_g, ln_b = ctx.params
        dtype = h.dtype
        if ctx.act == "relu":
            _, dpre, dg, db, dbias = ops.layernorm_bwd(dz.contiguous(), pre, ln_g, relu=True)
        else:
            dt, _, dg, db, _ = ops.layernorm_bwd(dz.contiguous(), t, ln_g, want_dbias=False)
            dpre = ops.dgelu_mul(dt, pre)
            dbias = None
        dh = ops.gemm(dpre, dense_w, b_major=1) if ctx.needs_input_grad[0] else None
        arena = getattr(dense_w, "_ub_arena", None)
        if arena is not None and arena._still_valid() and all(id(q) in arena._views for q in ctx.params):
            arena.mark_managed(ctx.params)
            acc = arena.claim(list(ctx.params))
            ops.gemm(dpre, h, a_major=1, b_major=1, out=arena.view(dense_w), accumulate=acc)
            ops.cvt_from_f32(ops.colsum(dpre) if dbias is None else dbias, dtype, out=arena.view(dense_b),
                             accumulate=acc)
            ops.cvt_from_f32(dg, dtype, out=arena.view(ln_g), accumulate=acc)
            ops.cvt_from_f32(db, dtype, out=arena.view(ln_b), accumulate=acc)
            return dh, None, None, None, None, None
        return (dh, ops.gemm(dpre, h, a_major=1, b_major=1),
                ops.cvt_from_f32(ops.colsum(dpre) if dbias is None else dbias, dtype),
                ops.cvt_from_f32(dg, dtype), ops.cvt_from_f32(db, dtype), None)


class RegionFeatureRegression(nn.Module):
    """model/pretrain.py:19-32 (MRFR head): LN(gelu(dense(h))) @ img_linear.weight + bias — the
    output projection is TIED to the image embedding's input projection, read as a [K, N] operand."""

    def __init__(self, hidden_size, feat_dim, img_linear_weight):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(hidden_size, hidden_size), GELU(),
                                 nn.LayerNorm(hidden_size, eps=1e-12))
        self.weight = img_linear_weight
        self.bias = nn.Parameter(torch.zeros(feat_dim))

    def forward(self, input_):
        hidden = LibTransform.apply(input_, self.net[0].weight, self.net[0].bias, self.net[2].weight,
                                    self.net[2].bias)
        return LibLinear.apply(hidden, self.weight, self.bias, True, False)


class RegionClassification(nn.Module):
    """model/pretrain.py:35-47 (MRC / MRC-kl head)."""

    def __init__(self, hidden_size, label_dim):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(hidden_size, hidden_size), GELU(),
                                 nn.LayerNorm(hidden_size, eps=1e-12), nn.Linear(hidden_size, label_dim))

    def forward(self, input_):
        hidden = LibTransform.apply(input_, self.net[0].weight, self.net[0].bias, self.net[2].weight,
                                    self.net[2].bias)
        return LibLinear.apply(hidden, self.net[3].weight, self.net[3].bias, False, False)


def _masked_rows(packed, meta, mask2d, index):
    """Rows of the packed encoder output selected by a [B, L] boolean mask (model/pretrain.py:129-133,
    `_compute_masked_hidden`) — or by a loader-provided flat index list (b * L + j; entries equal to
    B * L are padding of a fixed-size list -> zero rows), which needs no device read."""
    if index is None:
        pos = mask2d.nonzero(as_tuple=False)                   # device sync, like the reference
        index = pos[:, 0] * meta["L"] + pos[:, 1]
    return gather_packed_rows(packed, meta["unpack_ext"][index])


class _WraDist(torch.autograd.Function):
    """Word-region alignment distance of every pair (model/ot.py:optimal_transport_dist over the pair's
    text and region rows, rounded to the encoder's 16-bit type like `.to(txt_emb)`) in one kernel per
    direction (ub200_wra_*).  The transport plan is a constant for autograd; the backward writes one
    gradient row per packed row, zero on the rows of the padding sequence."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, packed, cu_seqlens, txt_len, batch, max_m, max_n):
        ws = ops.wra_workspace(batch, max_m, max_n, packed.device)
        dist = ops.wra_fwd(packed, cu_seqlens, txt_len, batch, max_m, max_n, ws)
        ctx.save_for_backward(packed, cu_seqlens, txt_len, ws)
        ctx.shape = (batch, max_m, max_n)
        return dist.to(packed.dtype)

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, d_dist):
        packed, cu_seqlens, txt_len, ws = ctx.saved_tensors
        d_packed = ops.wra_bwd(packed, cu_seqlens, txt_len, *ctx.shape, ws, d_dist.float().contiguous())
        return d_packed, None, None, None, None, None


class UniterForPretraining(UniterPreTrainedModel):
    """model/pretrain.py:50-229 with every head on libub200: MLM (fused head + cross-entropy), MRFR,
    MRC / MRC-kl (LibTransform + LibLinear over the masked REGION rows gathered straight from the
    packed encoder output) and ITM (library pooler + LibLinear).  Same parameter names, weight tying
    (cls.predictions.decoder <-> word_embeddings, feat_regress.weight <-> img_linear.weight) and
    forward(batch, task, compute_loss) contract.  ITM with `ot_inputs` (data/itm.py:itm_ot_collate) adds
    word-region alignment (model/pretrain.py:166-193): the IPOT distance between each pair's text rows
    and region rows, read straight from the packed encoder output (_WraDist, ub200_wra_*), returned as
    (itm_loss or itm_scores, (ot_pos, ot_neg)).  `ot_scatter` / `scatter_max` are not read; the pads may
    be uint8 or bool.

    Fixed-shape (CUDA-graph friendly) variants of the reference's data-dependent row selections are
    taken from the batch when the loader provides them: `mlm_index` / `mlm_targets`, `mrm_index`, and for
    WRA `ot_txt_lens` (int32 [B] text lengths) with `ot_pos_index` / `ot_neg_index` (int64 positions of
    the positive / negative pairs).  With those the ITM step reads nothing from the device; without them
    the text lengths come from one read of the pads and ot_pos / ot_neg from masked_select, as the
    reference reads them.  Where `txt_lens` / `num_bbs` are known on the host, a pair whose text and
    region counts do not add up to its valid tokens is a ValueError before any launch."""

    def __init__(self, config, img_dim, img_label_dim):
        super().__init__(config)
        self.uniter = UniterModel(config, img_dim)
        self.cls = BertOnlyMLMHead(config, self.uniter.embeddings.word_embeddings.weight)
        self.feat_regress = RegionFeatureRegression(config.hidden_size, img_dim,
                                                    self.uniter.img_embeddings.img_linear.weight)
        self.region_classifier = RegionClassification(config.hidden_size, img_label_dim)
        self.itm_output = nn.Linear(config.hidden_size, 2)
        self.apply(self.init_weights)

    def _encode(self, batch, img_masks=None):
        return self.uniter.encode_packed(
            batch["input_ids"], batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False,
            img_masks=img_masks, txt_type_ids=batch["txt_type_ids"])

    def forward(self, batch, task, compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        if task == "mlm":
            return self.forward_mlm(batch, compute_loss)
        if task == "mrfr":
            return self.forward_mrfr(batch, compute_loss)
        if task == "itm":
            return self.forward_itm(batch, compute_loss)
        if task.startswith("mrc"):
            return self.forward_mrc(batch, task, compute_loss)
        raise ValueError("invalid task")

    def forward_mlm(self, batch, compute_loss=True):                      # model/pretrain.py:107-127
        packed, meta = self._encode(batch)
        L = meta["L"]
        if batch["mlm_index"] is not None:
            flat, targets = batch["mlm_index"], batch["mlm_targets"]
        else:
            txt_labels = batch["txt_labels"]
            pos = (txt_labels != -1).nonzero(as_tuple=False)
            flat = pos[:, 0] * L + pos[:, 1]
            targets = txt_labels[pos[:, 0], pos[:, 1]]
        masked_output = gather_packed_rows(packed, meta["unpack_ext"][flat])
        return _MlmHead.apply(masked_output, self, targets, not compute_loss)

    def forward_mrfr(self, batch, compute_loss=True):                     # model/pretrain.py:135-154
        packed, meta = self._encode(batch, img_masks=batch["img_masks"])
        masked_output = _masked_rows(packed, meta, batch["img_mask_tgt"], batch["mrm_index"])
        prediction_feat = self.feat_regress(masked_output)
        if compute_loss:
            return F.mse_loss(prediction_feat, batch["feat_targets"].to(prediction_feat.dtype),
                              reduction="none")
        return prediction_feat

    def _wra_lengths(self, batch, ot_inputs):
        """(int32 text lengths on the device, max_m, max_n) of the WRA pairs, checked on the host where
        the lengths are known there.  max_m / max_n are the padded text and region extents."""
        max_m, max_n = batch["input_ids"].size(1), batch["img_feat"].size(1)
        if max_m * max_n > _lib.WRA_MAX_MN:
            raise ValueError("word-region alignment supports max text length x max regions <= %d, got %d x %d"
                             % (_lib.WRA_MAX_MN, max_m, max_n))
        dev = batch["attn_masks"].device
        txt_lens, num_bbs, txt_len = batch["txt_lens"], batch["num_bbs"], batch["ot_txt_lens"]
        if txt_len is None and (txt_lens is None or num_bbs is None):
            txt_pad, img_pad = ot_inputs["txt_pad"], ot_inputs["img_pad"]
            counts = torch.cat([txt_pad.size(1) - (txt_pad != 0).sum(1),
                                img_pad.size(1) - (img_pad != 0).sum(1)]).tolist()     # one device read
            txt_lens, num_bbs = counts[:txt_pad.size(0)], counts[txt_pad.size(0):]
        if txt_lens is not None and num_bbs is not None:
            seq = self.uniter._pack_meta(batch["attn_masks"])["lens_host"]
            for b, (m, n) in enumerate(zip(txt_lens, num_bbs)):
                if not (1 <= m <= max_m and 1 <= n <= max_n) or (seq is not None and m + n != seq[b]):
                    raise ValueError("pair %d: %d text tokens and %d regions do not fill its %s valid tokens "
                                     "(padded extents %d x %d)" % (b, m, n, seq[b] if seq else "?", max_m, max_n))
        if txt_len is None:
            txt_len = torch.tensor(list(txt_lens), dtype=torch.int32)
        return txt_len.to(dev, torch.int32).contiguous(), max_m, max_n

    def forward_itm(self, batch, compute_loss=True):                      # model/pretrain.py:156-199
        ot_inputs = batch["ot_inputs"]
        if ot_inputs is not None:
            txt_len, max_m, max_n = self._wra_lengths(batch, ot_inputs)
        packed, meta = self._encode(batch)
        B, L = meta["n_batch"], meta["L"]
        cls_rows = meta["unpack_ext"][::L][:B]          # packed row of position (b, 0): the [CLS] token
        pooled = self.uniter.pooler(gather_packed_rows(packed, cls_rows.contiguous()))
        itm_scores = LibLinear.apply(pooled, self.itm_output.weight, self.itm_output.bias, False, False)
        ot_loss = None
        if ot_inputs is not None:
            # the pairs' text rows then region rows, in the packed layout of the prefix masks
            ot_dist = _WraDist.apply(packed, meta["cu_seqlens"], txt_len, B, max_m, max_n)
            targets = batch["targets"]
            if batch["ot_pos_index"] is not None and batch["ot_neg_index"] is not None:
                dev = ot_dist.device
                ot_loss = (ot_dist.index_select(0, batch["ot_pos_index"].to(dev)),
                           ot_dist.index_select(0, batch["ot_neg_index"].to(dev)))
            else:
                ot_loss = (ot_dist.masked_select(targets == 1), ot_dist.masked_select(targets == 0))
        if compute_loss:
            return F.cross_entropy(itm_scores.float(), batch["targets"], reduction="none"), ot_loss
        return itm_scores, ot_loss

    def forward_mrc(self, batch, task, compute_loss=True):                # model/pretrain.py:201-229
        packed, meta = self._encode(batch, img_masks=batch["img_masks"])
        masked_output = _masked_rows(packed, meta, batch["img_mask_tgt"], batch["mrm_index"])
        prediction_soft_label = self.region_classifier(masked_output)
        if not compute_loss:
            return prediction_soft_label
        label_targets = batch["label_targets"]
        if "kl" in task:
            logp = F.log_softmax(prediction_soft_label.float(), dim=-1)
            return F.kl_div(logp, label_targets.float(), reduction="none")
        label_targets = torch.max(label_targets[:, 1:], dim=-1)[1] + 1   # background is never a target
        return F.cross_entropy(prediction_soft_label.float(), label_targets, ignore_index=0, reduction="none")


class UniterForVisualQuestionAnswering(UniterPreTrainedModel):
    """model/vqa.py:16-52."""

    def __init__(self, config, img_dim, num_answer):
        super().__init__(config)
        self.uniter = UniterModel(config, img_dim)
        self.vqa_output = nn.Sequential(
            nn.Linear(config.hidden_size, config.hidden_size * 2),
            GELU(),
            nn.LayerNorm(config.hidden_size * 2, eps=1e-12),
            nn.Linear(config.hidden_size * 2, num_answer))
        self.apply(self.init_weights)

    def forward(self, batch, compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        # pooler(sequence_output) (model/vqa.py:36-43) from the packed encoder output: only the [CLS]
        # rows are gathered, the padded [B, L, H] tensor is never materialised
        packed, meta = self.uniter.encode_packed(
            batch["input_ids"], batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False)
        B, L = meta["n_batch"], meta["L"]
        cls_rows = meta["unpack_ext"][::L][:B].contiguous()
        pooled_output = self.uniter.pooler(gather_packed_rows(packed, cls_rows))
        answer_scores = self.vqa_output(pooled_output)
        if compute_loss:
            return F.binary_cross_entropy_with_logits(answer_scores, batch["targets"], reduction="none")
        return answer_scores


class UniterForImageTextRetrieval(UniterPreTrainedModel):
    """model/itm.py:14-59 (ITM classifier of model/pretrain.py:159-176 shares ``itm_output``)."""

    def __init__(self, config, img_dim, margin=0.2):
        super().__init__(config)
        self.uniter = UniterModel(config, img_dim)
        self.itm_output = nn.Linear(config.hidden_size, 2)
        self.rank_output = nn.Linear(config.hidden_size, 1)
        self.margin = margin
        self.apply(self.init_weights)

    def init_output(self):
        """need to be called after from pretrained (model/itm.py:26-29)"""
        self.rank_output.weight.data = self.itm_output.weight.data[1:, :]
        self.rank_output.bias.data = self.itm_output.bias.data[1:]

    def pooled(self, batch):
        """pooler(sequence_output) (model/itm.py:36-42) without materialising the padded [B, L, H]
        tensor: the [CLS] rows are gathered straight from the packed encoder output."""
        batch = defaultdict(lambda: None, batch)
        packed, meta = self.uniter.encode_packed(
            batch["input_ids"], batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False)
        B, L = meta["n_batch"], meta["L"]
        cls_rows = meta["unpack_ext"][::L][:B].contiguous()      # packed row of position (b, 0)
        return self.uniter.pooler(gather_packed_rows(packed, cls_rows))

    def itm_scores(self, batch):
        """model/pretrain.py:163-164: itm_output(pooler(sequence_output))."""
        return LibLinear.apply(self.pooled(batch), self.itm_output.weight, self.itm_output.bias, False, False)

    def forward(self, batch, compute_loss=True):
        rank_scores = LibLinear.apply(self.pooled(batch), self.rank_output.weight, self.rank_output.bias,
                                      False, False)
        if compute_loss:
            scores = torch.sigmoid(rank_scores).contiguous().view(-1, batch["sample_size"])
            pos, neg = scores[:, :1], scores[:, 1:]
            return torch.clamp(self.margin + neg - pos, 0)
        return rank_scores


class UniterForImageTextRetrievalHardNeg(UniterForImageTextRetrieval):
    """model/itm.py:57-147 — in-batch hard-negative mining: score all N candidate pairs of one
    text (sample_from='t') or one image ('i') without gradients in eval mode, keep the positive
    (row 0) and the `hard_size` best-scoring negatives, and train on those."""

    def __init__(self, config, img_dim, margin=0.2, hard_size=16):
        super().__init__(config, img_dim, margin)
        self.hard_size = hard_size

    def forward(self, batch, sample_from="t", compute_loss=True):
        n_pairs = batch["attn_masks"].size(0)
        if sample_from == "t":                       # one text shared by every pair
            if batch["input_ids"].size(0) == 1:
                batch["input_ids"] = batch["input_ids"].expand(n_pairs, -1)
        elif sample_from == "i":                     # one image shared by every pair
            for key in ("img_feat", "img_pos_feat"):
                if batch[key].size(0) == 1:
                    batch[key] = batch[key].expand(n_pairs, -1, -1)
        else:
            raise ValueError()
        if not (self.training and compute_loss):
            return super().forward(batch, compute_loss)
        with torch.no_grad():
            self.eval()
            scores = super().forward(batch, compute_loss=False)
            hard_batch = self._get_hard_batch(batch, scores, sample_from)
            self.train()
        return super().forward(hard_batch, compute_loss=True)

    def _get_hard_batch(self, batch, scores, sample_from="t"):
        """Row selection of model/itm.py:92-147 (pure index logic, pinned bit-exactly against the
        reference in tests/test_heads_optim_cpu.py)."""
        batch = defaultdict(lambda: None, batch)
        k = self.hard_size
        neg = scores.squeeze(-1)[1:].topk(k, sorted=False)[1] + 1          # positive is row 0
        rows = torch.cat([neg.new_zeros(1), neg])
        masks = batch["attn_masks"].index_select(0, rows)
        gather = batch["gather_index"].index_select(0, rows)
        pos = batch["position_ids"]
        if pos.size(0) != 1:
            pos = pos[:k + 1]
        ids, feat, box = batch["input_ids"], batch["img_feat"], batch["img_pos_feat"]
        # host-known lengths of the candidate pairs (our collates provide them): the lengths of the
        # mined rows are then known after ONE small read of the top-k indices, and the train forward
        # packs without reading the device again (the reference syncs here too, model/itm.py:113)
        lens_all = None
        if batch["txt_lens"] is not None and batch["num_bbs"] is not None:
            lens_all = [a + b for a, b in zip(batch["txt_lens"], batch["num_bbs"])]
            rows_h = rows.tolist()
            lens_sel = [lens_all[r] for r in rows_h]
        if sample_from == "t":
            longest = max(lens_sel) if lens_all is not None else masks.sum(dim=1).max().item()   # cut to minimum padding
            n_img = longest - ids.size(1)
            masks, gather = masks[:, :longest], gather[:, :longest]
            feat = feat.index_select(0, rows)[:, :n_img, :]
            box = box.index_select(0, rows)[:, :n_img, :]
            ids = ids[:k + 1]
        elif sample_from == "i":
            ids = ids.index_select(0, rows)
            feat, box = feat[:k + 1], box[:k + 1]
        else:
            raise ValueError()
        if lens_all is not None:
            from .model import register_lengths
            masks = masks.contiguous()
            register_lengths(masks, lens_sel, prefix=True)
        return {"sample_size": k + 1, "input_ids": ids, "position_ids": pos, "img_feat": feat,
                "img_pos_feat": box, "attn_masks": masks, "gather_index": gather}


# ============================================================================ referring expressions
def re_neg_plan(targets, num_bbs, hard_ratio, np_random=None, py_random=None):
    """The negative of each sample of the ranking loss, drawn like model/re.py:102-127 (sample_neg_ix):
    per sample one np.random.uniform(0, 1, 1) draw decides hard (< hard_ratio) or easy; an easy sample
    draws random.randint(0, num_bb - 1) until it differs from the target.  Returns a list with -1 for a
    hard negative (the kernel picks the best-scoring other region on the device) and the drawn index for
    an easy one.  By default the draws come from the same global generators as the reference's, so a
    run seeded like train_re.py makes the same decisions; np_random / py_random replace them."""
    nr = np_random if np_random is not None else np.random
    pr = py_random if py_random is not None else random
    plan = []
    for t, nbb in zip(targets, num_bbs):
        t, nbb = int(t), int(nbb)
        if nbb < 2 or not 0 <= t < nbb:
            raise ValueError("the ranking loss needs num_bb >= 2 and 0 <= target < num_bb, got target %d of %d"
                             % (t, nbb))
        if nr.uniform(0, 1, 1) < hard_ratio:
            plan.append(-1)
        else:
            ix = pr.randint(0, nbb - 1)
            while ix == t:
                ix = pr.randint(0, nbb - 1)
            plan.append(ix)
    return plan


class _RegionScoreHead(torch.autograd.Function):
    """re_output (Linear(H, 1)) over the region rows, masked_fill(obj_masks, -1e4) and the per-sample
    loss (model/re.py:69-96) in one kernel per direction (ub200_region_score_*).  Returns the loss [B]
    fp32, or the masked scores [B, S] for mode RE_SCORES.  The weight and bias gradients are summed in
    sample order and written into the gradient arena when the parameters live in one."""

    @staticmethod
    @_lib.forward_in_mode()
    def forward(ctx, rows, weight, bias, seg, obj_masks, targets, neg_plan, mode, margin):
        w = weight.reshape(-1)
        if w.data_ptr() % 16:
            w = w.clone()
        scores, loss, lse, neg = ops.region_score_fwd(rows, w, bias, seg, obj_masks, targets, neg_plan,
                                                      mode, margin)
        if mode == _lib.RE_SCORES:
            ctx.mark_non_differentiable(scores)
            return scores
        ctx.save_for_backward(rows, w, seg, obj_masks, targets, scores, lse, neg)
        ctx.mode, ctx.margin, ctx.params = mode, margin, (weight, bias)
        return loss

    @staticmethod
    @_lib.backward_in_mode
    def backward(ctx, dloss):
        rows, w, seg, obj_masks, targets, scores, lse, neg = ctx.saved_tensors
        weight, bias = ctx.params
        d_rows, dw, db = ops.region_score_bwd(rows, w, seg, obj_masks, targets, scores, lse, neg,
                                              dloss.contiguous().float(), ctx.mode, ctx.margin)
        dtype = rows.dtype
        arena = getattr(weight, "_ub_arena", None)
        params = [weight, bias]
        if arena is not None and arena._still_valid() and all(id(p) in arena._views for p in params):
            arena.mark_managed(params)
            acc = arena.claim(params)
            ops.cvt_from_f32(dw, dtype, out=arena.view(weight), accumulate=acc)
            ops.cvt_from_f32(db, dtype, out=arena.view(bias), accumulate=acc)
            return d_rows, None, None, None, None, None, None, None, None
        return (d_rows, ops.cvt_from_f32(dw, dtype).view_as(weight), ops.cvt_from_f32(db, dtype).view_as(bias),
                None, None, None, None, None, None)


class UniterForReferringExpressionComprehension(UniterPreTrainedModel):
    """model/re.py:18-100 on the packed path.  Same parameter names (`re_output.weight / bias`, or
    `re_output.{0,2,3}.*` for mlp=2) and forward(batch, compute_loss) contract: the per-sample loss [B]
    (fp32; cross-entropy for loss="cls", the ranking hinge for "rank") when training with
    compute_loss, else the masked scores [B, max_num_bb].

    The region rows are gathered straight from the packed encoder output (no padded [B, L, H] tensor,
    no per-sample slicing); region k of sample b is padded position b * L + txt_lens[b] + k.  The batch
    may carry, as batching.re_collate makes them, `re_index` (those flat positions, padded with B * L)
    and `re_seg` (int32 [2, B]: start and length of each sample's rows); otherwise they are formed on
    the host from `txt_lens` / `num_bbs`.  The ranking loss reads the plan of negatives from
    `re_neg_plan` (int64 [B], see re_neg_plan) or, without one, draws it from the targets (one device
    read, as model/re.py:112 does).  With all three keys the step reads nothing from the device and can
    be captured by GraphedStep.  obj_masks may be uint8 (what data/re.py builds) or bool."""

    def __init__(self, config, img_dim, loss="cls", margin=0.2, hard_ratio=0.3, mlp=1):
        super().__init__(config)
        self.uniter = UniterModel(config, img_dim)
        H = config.hidden_size
        if mlp == 1:
            self.re_output = nn.Linear(H, 1)
        elif mlp == 2:
            self.re_output = nn.Sequential(nn.Linear(H, H), GELU(), nn.LayerNorm(H, eps=1e-12), nn.Linear(H, 1))
        else:
            raise ValueError("MLP restricted to be 1 or 2 layers.")
        self.loss = loss
        assert self.loss in ("cls", "rank")
        if self.loss == "rank":
            self.margin = margin
            self.hard_ratio = hard_ratio
        self.mlp = mlp
        self.apply(self.init_weights)

    def forward(self, batch, compute_loss=True):
        from .batching import re_region_index
        batch = defaultdict(lambda: None, batch)
        packed, meta = self.uniter.encode_packed(
            batch["input_ids"], batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False)
        dev = packed.device
        num_bbs = batch["num_bbs"]
        if num_bbs is not None and min(num_bbs) < 1:
            raise ValueError("every sample needs at least one region, got num_bbs %s" % list(num_bbs))
        index, seg = batch["re_index"], batch["re_seg"]
        if index is None or seg is None:
            if batch["txt_lens"] is None or num_bbs is None:
                raise ValueError("the batch needs re_index and re_seg, or txt_lens and num_bbs")
            index, seg = re_region_index(batch["txt_lens"], num_bbs, meta["L"])
            index, seg = index.to(dev), seg.to(dev)
        rows = gather_packed_rows(packed, meta["unpack_ext"][index])     # model/re.py:63-65
        head = self.re_output
        if self.mlp == 2:
            rows = LibTransform.apply(rows, head[0].weight, head[0].bias, head[2].weight, head[2].bias)
            head = head[3]
        obj_masks = batch["obj_masks"]
        if obj_masks.dtype not in (torch.uint8, torch.bool):
            obj_masks = obj_masks != 0
        obj_masks = obj_masks.contiguous()
        if not compute_loss:
            return _RegionScoreHead.apply(rows, head.weight, head.bias, seg, obj_masks, None, None,
                                          _lib.RE_SCORES, 0.0)
        targets = batch["targets"].reshape(-1)
        if not targets.is_cuda and num_bbs is not None:
            for t, nbb in zip(targets.tolist(), num_bbs):
                if not 0 <= t < nbb:
                    raise ValueError("target %d outside [0, %d)" % (t, nbb))
        targets = targets.to(dev).contiguous()
        if self.loss == "cls":
            return _RegionScoreHead.apply(rows, head.weight, head.bias, seg, obj_masks, targets, None,
                                          _lib.RE_CLS, 0.0)
        plan = batch["re_neg_plan"]
        if plan is None:
            if num_bbs is None:
                raise ValueError("the ranking loss needs re_neg_plan or num_bbs")
            plan = torch.tensor(re_neg_plan(targets.tolist(), num_bbs, self.hard_ratio), dtype=torch.long)
        plan = plan.to(dev).contiguous()
        return _RegionScoreHead.apply(rows, head.weight, head.bias, seg, obj_masks, targets, plan,
                                      _lib.RE_RANK, float(self.margin))


# ============================================================================ visual commonsense reasoning
class UniterForVisualCommonsenseReasoning(UniterPreTrainedModel):
    """model/vcr.py on the packed path.  Same parameter names (`vcr_output.{0,2,3}.*`), the same
    forward(batch, compute_loss) contract (the mean cross-entropy over the batch, a scalar, with
    compute_loss; else scores[:, 1:], shape [B, 1]) and the same init_type_embedding /
    init_word_embedding semantics.

    The [CLS] rows are gathered from the packed encoder output (as VQA and ITM do), the pooler is the
    library's, and vcr_output runs as LibTransform(act="relu") — Linear(H, 2H) -> ReLU -> LayerNorm(2H)
    with the ReLU fused into the LayerNorm kernels — then LibLinear(2H, 2).  txt_type_ids (values 0-3
    after init_type_embedding) reach the embedding front-end.  With the host-known lengths registered
    (batching.vcr_collate provides txt_lens / num_bbs) a step reads nothing from the device, so
    GraphedStep captures it."""

    def __init__(self, config, img_dim):
        super().__init__(config, img_dim)
        self.uniter = UniterModel(config, img_dim)
        H = config.hidden_size
        self.vcr_output = nn.Sequential(
            nn.Linear(H, H * 2),
            nn.ReLU(),
            nn.LayerNorm(H * 2, eps=1e-12),
            nn.Linear(H * 2, 2))
        self.apply(self.init_weights)

    def _replace_table(self, name, new_emb):
        """Install new_emb (built and initialised on the CPU in fp32, as the reference does) as
        uniter.embeddings.<name> on the old table's device and dtype, and retire every gradient arena
        planned over the old parameter set."""
        from .arena import GradArena
        te = self.uniter.embeddings
        old = getattr(te, name).weight
        new_emb = new_emb.to(device=old.device, dtype=old.dtype)
        new_emb.weight.requires_grad_(old.requires_grad)
        stale = {id(a): a for a in (getattr(old, "_ub_arena", None), GradArena.of(self),
                                    self.uniter._arena[0] if self.uniter._arena is not None else None)
                 if a is not None}
        for a in stale.values():
            a.invalidate()
        self.uniter._arena = None
        setattr(te, name, new_emb)

    def init_type_embedding(self):
        """model/vcr.py:34-44: a 4-row token-type table, init_weights-initialised; rows 0 and 1 copied
        from the old table, rows 2 and 3 copies of old row 0.  Consumes the global torch RNG like the
        reference (the new table is built on the CPU in fp32 whatever the model's device)."""
        old = self.uniter.embeddings.token_type_embeddings.weight.data.float().cpu()
        new_emb = nn.Embedding(4, self.uniter.config.hidden_size)
        new_emb.apply(self.init_weights)
        for i in [0, 1]:
            new_emb.weight.data[i, :].copy_(old[i, :])
        new_emb.weight.data[2, :].copy_(old[0, :])
        new_emb.weight.data[3, :].copy_(old[0, :])
        self._replace_table("token_type_embeddings", new_emb)

    def init_word_embedding(self, num_special_tokens):
        """model/vcr.py:46-53: an nn.Embedding(V + num_special_tokens, H) with no padding_idx,
        init_weights-initialised, its first V rows copied from the old table (train_vcr.py adds 81)."""
        old = self.uniter.embeddings.word_embeddings.weight.data.float().cpu()
        orig_word_num = old.size(0)
        new_emb = nn.Embedding(orig_word_num + num_special_tokens, self.uniter.config.hidden_size)
        new_emb.apply(self.init_weights)
        new_emb.weight.data[:orig_word_num, :].copy_(old)
        self._replace_table("word_embeddings", new_emb)

    def forward(self, batch, compute_loss=True):
        batch = defaultdict(lambda: None, batch)
        packed, meta = self.uniter.encode_packed(
            batch["input_ids"], batch["position_ids"], batch["img_feat"], batch["img_pos_feat"],
            batch["attn_masks"], batch["gather_index"], output_all_encoded_layers=False,
            txt_type_ids=batch["txt_type_ids"])
        B, L = meta["n_batch"], meta["L"]
        cls_rows = meta["unpack_ext"][::L][:B].contiguous()       # packed row of position (b, 0)
        pooled_output = self.uniter.pooler(gather_packed_rows(packed, cls_rows))
        head = self.vcr_output
        hidden = LibTransform.apply(pooled_output, head[0].weight, head[0].bias, head[2].weight, head[2].bias,
                                    "relu")
        rank_scores = LibLinear.apply(hidden, head[3].weight, head[3].bias, False, False)
        if compute_loss:
            targets = batch["targets"]
            return F.cross_entropy(rank_scores.float(), targets.squeeze(-1), reduction="mean")
        return rank_scores[:, 1:]
