"""ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product path.

CPU fp32 restatement of the reference's encoder hot path (ChenRocks/UNITER), written from the
algorithm in SURVEY.md §8a.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import this module; the
product (``uniter_b200``) never does.

Pinning: the reference ships NO tests or golden vectors for this path ("parity unpinned" by the
reference's own suite).  This restatement is therefore pinned against outputs of the reference
itself: ``tests/golden/make_goldens.py`` imports the reference's ``model/`` (apex FusedLayerNorm
shimmed to torch.nn.LayerNorm — the only apex symbol the model code uses) and stores its
outputs; ``tests/test_oracle_golden.py`` checks this file against them.

Every function takes the model as a flat ``state`` dict of fp32 tensors keyed exactly like the
reference ``UniterModel.state_dict()`` (SURVEY.md §8b), so it is independent of any nn.Module
class of ours or theirs.  Autograd works through it (plain torch ops), which is how gradient
goldens are checked.

Third-party arithmetic pinned here (not in the reference): apex FusedLayerNorm (NGC 19.05
image, no version pin) = biased variance, eps inside the sqrt, fp32 statistics; Horovod 0.16.4
allreduce = mean over ranks.
"""
import math

import torch


# ----------------------------------------------------------------------------- elementwise
def gelu_erf(x):
    """model/layer.py:31-37 — exact erf GELU (not the tanh approximation)."""
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def layer_norm(x, weight, bias, eps=1e-12):
    """apex FusedLayerNorm as used at model/layer.py:108,149 and model/model.py:228,254-259:
    mean / biased variance over the last dim, eps added inside the sqrt, affine.  16-bit inputs keep
    fp32 statistics and round once, as apex does for half inputs (torch's native layer_norm has the
    same contract)."""
    if x.dtype in (torch.float16, torch.bfloat16):
        return torch.nn.functional.layer_norm(x, (x.size(-1),), weight, bias, eps)
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * weight + bias


def linear(x, w, b=None):
    y = x @ w.t()
    return y if b is None else y + b


def dropout(x, keep=None, inv_keep=1.0):
    """nn.Dropout with a given keep mask (bool, broadcasting against x): x * keep * inv_keep, computed
    in at least fp32 and rounded once to x's dtype as torch's dropout does; identity without a mask."""
    if keep is None:
        return x
    w = torch.promote_types(x.dtype, torch.float32)
    return (x.to(w) * (keep.to(w) * inv_keep)).to(x.dtype)


# ----------------------------------------------------------------------------- embeddings
def text_embeddings(state, input_ids, position_ids, token_type_ids=None, prefix="embeddings.",
                    keep=None, inv_keep=1.0, taps=None):
    """model/model.py:232-245 — dropout(LN(word[ids] + pos[position_ids] + type[tt])), the dropout
    given as a keep mask (none: p = 0).  position_ids is [1, Lt] and broadcasts over the batch.
    taps["u"]: the sum before the LayerNorm."""
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    e = (state[prefix + "word_embeddings.weight"][input_ids]
         + state[prefix + "position_embeddings.weight"][position_ids]
         + state[prefix + "token_type_embeddings.weight"][token_type_ids])
    if taps is not None:
        taps["u"] = e
    return dropout(layer_norm(e, state[prefix + "LayerNorm.weight"], state[prefix + "LayerNorm.bias"]),
                   keep, inv_keep)


def image_embeddings(state, img_feat, img_pos_feat, img_type_ids=None, img_masks=None,
                     prefix="img_embeddings.", keep=None, inv_keep=1.0, taps=None):
    """model/model.py:311-319 + :261-272 — dropout(LN( LN(img_linear(f)) + LN(pos_linear(p)) + type )),
    the dropout given as a keep mask (none: p = 0).  With img_masks, row 1 of mask_embedding is added
    to masked regions (row 0 is forced to 0).  taps["u"]: the sum before the last LayerNorm,
    taps["ppre"]: the pos_linear output."""
    if img_type_ids is None:
        img_type_ids = torch.ones(img_feat.shape[:2], dtype=torch.long)
    type_emb = state["embeddings.token_type_embeddings.weight"][img_type_ids]
    if img_masks is not None:
        mw = state[prefix + "mask_embedding.weight"].clone()
        mw[0] = 0  # model/model.py:263
        img_feat = img_feat + mw[img_masks.long()]
    t_im = layer_norm(linear(img_feat, state[prefix + "img_linear.weight"],
                             state[prefix + "img_linear.bias"]),
                      state[prefix + "img_layer_norm.weight"], state[prefix + "img_layer_norm.bias"])
    ppre = linear(img_pos_feat, state[prefix + "pos_linear.weight"], state[prefix + "pos_linear.bias"])
    t_pos = layer_norm(ppre, state[prefix + "pos_layer_norm.weight"], state[prefix + "pos_layer_norm.bias"])
    u = t_im + t_pos + type_emb
    if taps is not None:
        taps["u"], taps["ppre"] = u, ppre
    return dropout(layer_norm(u, state[prefix + "LayerNorm.weight"], state[prefix + "LayerNorm.bias"]),
                   keep, inv_keep)


def gather_embeddings(txt_emb, img_emb, gather_index):
    """model/model.py:321-334 — x[b, j] = cat([txt, img], 1)[b, gather_index[b, j]]."""
    cat = torch.cat([txt_emb, img_emb], dim=1)
    idx = gather_index.unsqueeze(-1).expand(-1, -1, cat.size(-1))
    return torch.gather(cat, 1, idx)


# ----------------------------------------------------------------------------- encoder layer
def self_attention(state, prefix, x, ext_mask, num_heads, taps=None):
    """model/layer.py:75-101.  x [B, L, H]; ext_mask [B, 1, 1, L] additive (0 / -10000)."""
    B, L, H = x.shape
    d = H // num_heads

    def split(t):  # transpose_for_scores, :70-73
        return t.view(B, L, num_heads, d).permute(0, 2, 1, 3)

    q = split(linear(x, state[prefix + "query.weight"], state[prefix + "query.bias"]))
    k = split(linear(x, state[prefix + "key.weight"], state[prefix + "key.bias"]))
    v = split(linear(x, state[prefix + "value.weight"], state[prefix + "value.bias"]))
    scores = q @ k.transpose(-1, -2) / math.sqrt(d) + ext_mask
    probs = torch.softmax(scores, dim=-1)
    ctx = (probs @ v).permute(0, 2, 1, 3).contiguous().view(B, L, H)
    if taps is not None:
        taps["q"], taps["k"], taps["v"], taps["ctx"] = q, k, v, ctx
    return ctx


def bert_layer(state, prefix, x, ext_mask, num_heads, taps=None):
    """model/layer.py:159-170 (BertLayer) = BertAttention (:118-127: self + BertSelfOutput
    :111-115) -> BertIntermediate (:139-142) -> BertOutput (:152-156).  Post-LN, eps 1e-12."""
    ctx = self_attention(state, prefix + "attention.self.", x, ext_mask, num_heads, taps)
    a = layer_norm(linear(ctx, state[prefix + "attention.output.dense.weight"],
                          state[prefix + "attention.output.dense.bias"]) + x,
                   state[prefix + "attention.output.LayerNorm.weight"],
                   state[prefix + "attention.output.LayerNorm.bias"])
    f = gelu_erf(linear(a, state[prefix + "intermediate.dense.weight"],
                        state[prefix + "intermediate.dense.bias"]))
    out = layer_norm(linear(f, state[prefix + "output.dense.weight"],
                            state[prefix + "output.dense.bias"]) + a,
                     state[prefix + "output.LayerNorm.weight"], state[prefix + "output.LayerNorm.bias"])
    if taps is not None:
        taps["attn_out"], taps["ffn1"], taps["layer_out"] = a, f, out
    return out


def pooler(state, seq_out, prefix="pooler."):
    """model/layer.py:179-185 — tanh(dense(x[:, 0]))."""
    return torch.tanh(linear(seq_out[:, 0], state[prefix + "dense.weight"],
                             state[prefix + "dense.bias"]))


# ----------------------------------------------------------------------------- whole model
def uniter_forward(state, num_layers, num_heads, input_ids, position_ids, img_feat, img_pos_feat,
                   attention_mask, gather_index=None, img_masks=None,
                   output_all_encoded_layers=True, txt_type_ids=None, img_type_ids=None,
                   taps=None):
    """model/model.py:336-367 (UniterModel.forward), padded [B, L] rectangle exactly as the
    reference computes it, including its garbage at masked query rows."""
    pdtype = next(iter(state.values())).dtype           # :343-344 "fp16 compatibility": param dtype
    ext_mask = (1.0 - attention_mask[:, None, None, :].to(pdtype)) * -10000.0         # :342-345
    if input_ids is None:                                                              # :348-351
        x = image_embeddings(state, img_feat, img_pos_feat, img_type_ids, img_masks)
    elif img_feat is None:                                                             # :352-355
        x = text_embeddings(state, input_ids, position_ids, txt_type_ids)
    else:                                                                              # :356-360
        txt = text_embeddings(state, input_ids, position_ids, txt_type_ids)
        img = image_embeddings(state, img_feat, img_pos_feat, img_type_ids, img_masks)
        x = gather_embeddings(txt, img, gather_index)
    if taps is not None:
        taps["embedding_output"] = x
    outs = []
    for i in range(num_layers):                                                        # :286-289
        x = bert_layer(state, "encoder.layer.%d." % i, x, ext_mask, num_heads,
                       taps if (taps is not None and i == 0) else None)
        if output_all_encoded_layers:
            outs.append(x)
    return outs if output_all_encoded_layers else x


def mlm_head(state, masked_hidden, prefix="cls.predictions."):
    """model/layer.py:188-222 — LN(gelu(dense(h))) @ word_embeddings^T + bias (tied decoder,
    model/pretrain.py:55-56)."""
    h = layer_norm(gelu_erf(linear(masked_hidden, state[prefix + "transform.dense.weight"],
                                   state[prefix + "transform.dense.bias"])),
                   state[prefix + "transform.LayerNorm.weight"], state[prefix + "transform.LayerNorm.bias"])
    return h @ state["uniter.embeddings.word_embeddings.weight"].t() + state[prefix + "bias"]


def mlm_forward(state, num_layers, num_heads, batch):
    """UniterForPretraining.forward_mlm (model/pretrain.py:107-133): per-masked-token CE loss."""
    enc = {k[len("uniter."):]: v for k, v in state.items() if k.startswith("uniter.")}
    seq = uniter_forward(enc, num_layers, num_heads, batch["input_ids"], batch["position_ids"],
                         batch["img_feat"], batch["img_pos_feat"], batch["attn_masks"],
                         batch["gather_index"], output_all_encoded_layers=False)
    seq = seq[:, :batch["input_ids"].size(1), :]
    mask = batch["txt_labels"] != -1
    scores = mlm_head(state, seq[mask])
    return torch.nn.functional.cross_entropy(scores, batch["txt_labels"][mask], reduction="none")


def vqa_head(state, pooled, prefix="vqa_output."):
    """model/vqa.py:23-28,44 — Linear(H, 2H) -> GELU -> LayerNorm(2H) -> Linear(2H, answers)."""
    h = gelu_erf(linear(pooled, state[prefix + "0.weight"], state[prefix + "0.bias"]))
    h = layer_norm(h, state[prefix + "2.weight"], state[prefix + "2.bias"])
    return linear(h, state[prefix + "3.weight"], state[prefix + "3.bias"])


def itm_head(state, pooled, prefix="itm_output."):
    """model/pretrain.py:163-164 / model/itm.py:20 — Linear(H, 2) on the pooled output."""
    return linear(pooled, state[prefix + "weight"], state[prefix + "bias"])


# ----------------------------------------------------------------------------- optimizer
def clip_grad_norm(grads, max_norm):
    """torch.nn.utils.clip_grad_norm_ as called at train_vqa.py:223-226: total 2-norm over all
    gradients; coef = max_norm / (total + 1e-6); gradients are scaled only if coef < 1.
    Returns (clipped grads, total_norm)."""
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads)).float()
    coef = max_norm / (total + 1e-6)
    if coef < 1:
        grads = [g * coef for g in grads]
    return grads, total


def adamw_step(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-6, weight_decay=0.0,
               correct_bias=True):
    """optim/adamw.py:62-101, one parameter tensor, fp32: returns (p, m, v) after step `step`
    (1-based).  m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; denom = sqrt(v) + eps;
    step_size = lr * sqrt(1-b2^t) / (1-b1^t); p -= step_size * m / denom; then the decoupled
    decay p -= lr * wd * p on the UPDATED p (:99-100)."""
    m = m * beta1 + (1.0 - beta1) * g
    v = v * beta2 + (1.0 - beta2) * g * g
    denom = v.sqrt() + eps
    step_size = lr
    if correct_bias:
        step_size = step_size * math.sqrt(1.0 - beta2 ** step) / (1.0 - beta1 ** step)
    p = p - step_size * (m / denom)
    if weight_decay > 0.0:
        p = p - lr * weight_decay * p
    return p, m, v


# ----------------------------------------------------------------------------- host-side index logic
def get_gather_index(txt_lens, num_bbs, batch_size, max_len, out_size):
    """data/data.py:271-279 — canonical compaction index (pure integer logic)."""
    assert len(txt_lens) == len(num_bbs) == batch_size
    gi = torch.arange(0, out_size, dtype=torch.long).unsqueeze(0).repeat(batch_size, 1)
    for i, (tl, nbb) in enumerate(zip(txt_lens, num_bbs)):
        gi[i, tl:tl + nbb] = torch.arange(max_len, max_len + nbb, dtype=torch.long)
    return gi


def allreduce_mean(grads_per_rank):
    """utils/distributed.py:16-43 with Horovod 0.16.4 `allreduce_(average=True)`: every rank ends
    with the mean over ranks of the flattened gradient buffer (rescale_denom = 1 at call sites)."""
    n = len(grads_per_rank)
    mean = sum(grads_per_rank) / float(n)
    return [mean.clone() for _ in range(n)]
