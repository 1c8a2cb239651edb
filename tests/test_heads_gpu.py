"""GPU: the task heads on top of the drop-in encoder (SURVEY.md §8c G6, §8f-1).

Head-level logits through OUR modules vs the goldens the reference's own heads produced
(north star: logits within 1e-2 in fp16), the fused MLM head (wgmma GEMMs with n_valid /
split-K, fused cross-entropy) vs the CPU oracle including gradients, and the CE kernels alone."""
import pytest
import torch

from oracle import encoder_oracle as orc
from tests import util

pytestmark = pytest.mark.gpu


def _cuda(batch):
    return util.batch_to(batch, "cuda")


def test_vqa_logits_match_reference_golden_fp16():
    from uniter_b200.heads import UniterForVisualQuestionAnswering
    g = util.load_golden("heads_tiny")
    mod = UniterForVisualQuestionAnswering(util.tiny_config(), 64, 17)
    mod.load_state_dict(util.head_state(mod, seed=3), strict=True)
    mod = mod.cuda().half().eval()
    logits = mod(_cuda(util.heads_batch()), compute_loss=False)
    err = (logits.float().cpu() - torch.from_numpy(g["vqa_logits"])).abs().max().item()
    assert err <= 1e-2, err


@pytest.mark.parametrize("use_index", [True, False])
def test_mlm_scores_match_reference_golden_fp16(use_index):
    from uniter_b200.heads import UniterForMLM
    g = util.load_golden("heads_tiny")
    mod = UniterForMLM(util.tiny_config(), 64)
    mod.load_state_dict(util.head_state(mod, seed=4, ties=util.PRETRAIN_TIES), strict=True)
    mod = mod.cuda().half().eval()
    batch = util.heads_batch()
    if not use_index:            # the reference's own boolean-mask path (model/pretrain.py:129-133)
        batch = {k: v for k, v in batch.items() if k not in ("mlm_index", "mlm_targets")}
    with torch.no_grad():
        scores = mod(_cuda(batch), compute_loss=False)
    ref = torch.from_numpy(g["mlm_scores"])
    assert scores.shape == ref.shape
    err = (scores.float().cpu() - ref).abs().max().item()
    assert err <= 1e-2, err


def test_itm_scores_match_reference_golden_fp16():
    from uniter_b200.heads import UniterForImageTextRetrieval
    g = util.load_golden("heads_tiny")
    mod = UniterForImageTextRetrieval(util.tiny_config(), 64)
    st = util.head_state(mod, seed=4, ties=(util.PRETRAIN_TIES[1],))
    # the golden ran inside UniterForPretraining, where word embeddings carry the decoder alias
    from uniter_b200.synth import seeded_state
    st["uniter.embeddings.word_embeddings.weight"] = seeded_state(
        {"cls.predictions.decoder.weight": (2000, 128)}, seed=4)["cls.predictions.decoder.weight"]
    mod.load_state_dict(st, strict=True)
    mod = mod.cuda().half().eval()
    scores = mod.itm_scores(_cuda(util.heads_batch()))
    err = (scores.float().cpu() - torch.from_numpy(g["itm_scores"])).abs().max().item()
    assert err <= 1e-2, err


@pytest.mark.parametrize("dtype,vocab", [(torch.float16, 2004), (torch.bfloat16, 2004), (torch.bfloat16, 2000)])
def test_mlm_loss_and_gradients_vs_oracle(dtype, vocab):
    """Vocabulary NOT a multiple of 8 (like BERT's 28996): padded score columns must not leak into
    the loss or any gradient; tied decoder / embedding gradient accumulates both uses."""
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.model import UniterConfig
    from uniter_b200.synth import synth_batch
    cfg = UniterConfig(vocab, hidden_size=128, num_hidden_layers=2, num_attention_heads=2,
                       intermediate_size=512, max_position_embeddings=64)
    mod = UniterForMLM(cfg, 64)
    st = util.head_state(mod, seed=9)
    st["cls.predictions.decoder.weight"] = st["uniter.embeddings.word_embeddings.weight"]
    mod.load_state_dict(st, strict=True)
    mod = mod.to("cuda", dtype).eval()
    batch = synth_batch(5, 6, 14, 3, 9, seed=21, img_dim=64, vocab_size=vocab, mlm_prob=0.4)
    loss = mod(_cuda(batch))
    rs = {k: v.to(dtype).float().requires_grad_(True) for k, v in st.items()
          if k != "cls.predictions.decoder.weight"}
    b16 = dict(batch)
    b16["img_feat"] = batch["img_feat"].to(dtype).float()
    b16["img_pos_feat"] = batch["img_pos_feat"].to(dtype).float()
    ref = orc.mlm_forward(rs, 2, 2, b16)
    assert loss.dtype == torch.float32 and loss.shape == ref.shape
    tol = 2e-2 if dtype == torch.float16 else 8e-2
    assert (loss.cpu() - ref.detach()).abs().max().item() <= tol
    (loss.mean() * 64).backward()
    (ref.mean() * 64).backward()
    params = dict(mod.named_parameters())
    worst = ("", 0.0)
    for name in ("cls.predictions.transform.dense.weight", "cls.predictions.transform.dense.bias",
                 "cls.predictions.transform.LayerNorm.weight", "cls.predictions.transform.LayerNorm.bias",
                 "cls.predictions.bias", "uniter.embeddings.word_embeddings.weight",
                 "uniter.embeddings.position_embeddings.weight", "uniter.embeddings.token_type_embeddings.weight",
                 "uniter.img_embeddings.pos_linear.weight", "uniter.img_embeddings.img_linear.weight",
                 "uniter.encoder.layer.1.output.dense.weight", "uniter.encoder.layer.0.attention.self.value.weight"):
        got = params[name].grad.float().cpu()
        want = rs[name].grad
        rel = ((got - want).norm() / (want.norm() + 1e-12)).item()
        if rel > worst[1]:
            worst = (name, rel)
    assert worst[1] <= (3e-2 if dtype == torch.float16 else 6e-2), worst


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n,V", [(190, 28996), (3, 2000), (17, 1001)])
def test_cross_entropy_kernels_vs_torch(dtype, n, V):
    from uniter_b200 import ops
    torch.manual_seed(n + V)
    Vp = (V + 7) // 8 * 8
    logits = torch.full((n, Vp), -30000.0, device="cuda", dtype=dtype)
    logits[:, :V] = (torch.randn(n, V, device="cuda") * 3).to(dtype)
    targets = torch.randint(0, V, (n,), device="cuda")
    targets[0] = -1                                  # ignored row: loss 0, gradient 0
    x = logits[:, :V].float().requires_grad_(True)
    keep = targets >= 0
    ref = torch.zeros(n, device="cuda")
    ref[keep] = torch.nn.functional.cross_entropy(x[keep], targets[keep], reduction="none")
    loss, lse = ops.ce_fwd(logits, targets, V)
    assert (loss - ref.detach()).abs().max().item() <= 2e-3
    dloss = torch.rand(n, device="cuda") + 0.5
    (ref * dloss).sum().backward()
    d = ops.ce_bwd_(logits, targets, lse, dloss, V)
    assert d.data_ptr() == logits.data_ptr()
    assert (d[:, V:] == 0).all() and (d[0] == 0).all()
    err = (d[:, :V].float() - x.grad).abs().max().item()
    assert err <= (2e-3 if dtype == torch.float16 else 1e-2), err


def test_embedding_table_gradient_kernels_vs_torch():
    """ub200_embed_bwd_scatter / _colsums against index_add_ / matmul restatements."""
    import ctypes as C
    from uniter_b200 import _lib
    lib = _lib.load()
    torch.manual_seed(5)
    T, H, V, P, Ty, R = 777, 768, 300, 40, 3, 500
    for dtype in (torch.bfloat16, torch.float16):
        du = (torch.randn(T, H, device="cuda") * 0.1).to(dtype)
        kind = (torch.rand(T, device="cuda") < 0.6).int()          # 1 = image row
        word_id = torch.randint(0, V, (T,), device="cuda", dtype=torch.int32)
        pos_id = torch.randint(0, P, (T,), device="cuda", dtype=torch.int32)
        type_id = torch.randint(0, Ty, (T,), device="cuda", dtype=torch.int32)
        img_src = torch.where(kind == 1, torch.randint(0, R, (T,), device="cuda", dtype=torch.int32),
                              torch.full((T,), -1, device="cuda", dtype=torch.int32))
        pos_feat = torch.rand(R, 7, device="cuda")
        d_word = torch.zeros(V, H, device="cuda", dtype=dtype)
        d_pos = torch.zeros(P, H, device="cuda")
        dt = _lib.dtype_code(dtype)
        s = _lib.current_stream()
        _lib.check(lib.ub200_embed_bwd_scatter(du.data_ptr(), kind.data_ptr(), word_id.data_ptr(),
                                               pos_id.data_ptr(), d_word.data_ptr(), d_pos.data_ptr(),
                                               T, H, dt, s))
        txt = (kind == 0)
        ref_w = torch.zeros(V, H, device="cuda").index_add_(0, word_id[txt].long(), du[txt].float())
        ref_p = torch.zeros(P, H, device="cuda").index_add_(0, pos_id[txt].long(), du[txt].float())
        assert (d_pos - ref_p).abs().max().item() <= 1e-4
        tol = 4e-2 if dtype == torch.bfloat16 else 6e-3               # 16-bit atomic accumulation
        assert (d_word.float() - ref_w).abs().max().item() <= tol * max(1.0, ref_w.abs().max().item())
        d_type = torch.zeros(Ty, H, device="cuda")
        a = _lib.EmbedColsumArgs(x=du.data_ptr(), type_id=type_id.data_ptr(), out=d_type.data_ptr(),
                                 T=T, hidden=H, mode=0, type_vocab=Ty, dtype=dt)
        _lib.check(lib.ub200_embed_bwd_colsums(C.byref(a), s))
        ref_t = torch.zeros(Ty, H, device="cuda").index_add_(0, type_id.long(), du.float())
        assert (d_type - ref_t).abs().max().item() <= 2e-3
        d_wpos = torch.zeros(H, 7, device="cuda")
        a = _lib.EmbedColsumArgs(x=du.data_ptr(), kind=kind.data_ptr(), img_src=img_src.data_ptr(),
                                 pos_feat=pos_feat.data_ptr(), out=d_wpos.data_ptr(), T=T, hidden=H,
                                 mode=1, type_vocab=0, dtype=dt)
        _lib.check(lib.ub200_embed_bwd_colsums(C.byref(a), s))
        F = pos_feat[img_src.clamp(min=0).long()].to(dtype).float() * (kind == 1).unsqueeze(1)
        ref_wp = du.float().t() @ F
        assert (d_wpos - ref_wp).abs().max().item() <= 2e-3 * max(1.0, ref_wp.abs().max().item())


def test_collate_prefetch_pipeline_matches_plain_batches():
    """Host batching -> pinned side-stream H2D -> registered lengths (no device sync in forward)
    gives the same losses as feeding the same collated batch without any registration."""
    from tests.golden.make_goldens import batching_samples
    from uniter_b200 import batching
    from uniter_b200.heads import UniterForMLM
    torch.manual_seed(1)
    mod = UniterForMLM(util.tiny_config(), 16).to("cuda", torch.float16).eval()
    samples = batching_samples(41, 24, True)
    lens = [s[3].numel() for s in samples]
    import random
    sampler = batching.TokenBucketSampler(lens, bucket_size=16, batch_size=160, rng=random.Random(0))
    host_batches = [batching.mlm_collate([samples[i] for i in ids]) for ids in iter(sampler)]
    assert len(host_batches) >= 2 and sum(len(b["txt_lens"]) for b in host_batches) == 24
    got = []
    with torch.no_grad():
        for batch in batching.DevicePrefetcher(host_batches):
            assert batch["attn_masks"].is_cuda
            got.append(mod(batch).float().cpu())
        for hb, g in zip(host_batches, got):
            plain = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in hb.items()
                     if k not in ("mlm_index", "mlm_targets")}
            ref = mod(plain).float().cpu()
            assert ref.shape == g.shape and torch.allclose(ref, g, atol=1e-3, rtol=0)
