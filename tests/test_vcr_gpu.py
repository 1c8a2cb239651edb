"""GPU: VCR fine-tuning (uniter_b200.heads.UniterForVisualCommonsenseReasoning) and the ReLU / wide
LayerNorm kernels under its head.

* The kernels against float64 (tests/vcr_check.py, tests/rowops_check.py) in fp16 and bf16: ReLU rows at
  W = 768, 1536 and 2048 and plain rows at 1536 and 2048; 1, 3, 64 and 257 rows whose `pre` holds
  negatives, exact zeros and an all-negative row; both library modes, the deterministic one giving the
  same bits across runs and under two SM reserves.
* The model against the UNMODIFIED reference class (model/vcr.py, staged into oracle/_ref by build())
  over the drop-in encoder, after both init methods, at UNITER-base (1 layer: a 1536-wide head) with one
  sequence longer than 128 tokens, and at UNITER-large (a 2048-wide head).
* A GraphedStep replay of a VCR step equals the eager step; two graphed fp16 steps with the loss scaler
  and FusedAdamW under torch.use_deterministic_algorithms give the same bits (sequences <= 128 tokens;
  a longer batch is refused under the flag).
* A gradient arena built before init_type_embedding / init_word_embedding is replaced, not written into.
"""
import pytest
import torch

from oracle import ref_loader
from tests import rowops_check as rc
from tests import util, vcr_check

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="reference sources not staged")

N_SPECIAL = 81


@pytest.fixture(autouse=True)
def torch_flags():
    from uniter_b200 import _lib
    saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    yield
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])
    _lib.load().ub200_set_sm_reserve(0)


# ----------------------------------------------------------------------------- kernels vs float64
def _ln_run(pre, gamma, beta, dy, relu):
    from uniter_b200 import ops
    y = ops.layernorm_fwd(pre, gamma, beta, relu=relu)
    dx, dpre, dg, db, dbias = ops.layernorm_bwd(dy, pre, gamma, relu=relu)
    torch.cuda.synchronize()
    return dict(y=y, dx=dx, dpre=dpre, dgamma=dg, dbeta=db, dbias=dbias)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("W,relu", [(768, True), (1536, True), (2048, True), (1536, False), (2048, False)])
@pytest.mark.parametrize("deterministic", [False, True])
def test_layernorm_kernels_match_float64(dtype, W, relu, deterministic):
    from uniter_b200 import _lib
    torch.use_deterministic_algorithms(deterministic)
    lib = _lib.load()
    for rows in (1, 3, 64, 257):
        pre, gamma, beta, dy = vcr_check.relu_ln_case(rows, W, dtype, seed=rows * 7 + W, device="cuda")
        out = _ln_run(pre, gamma, beta, dy, relu)
        base = vcr_check.relu_ln_baseline(dy, pre, gamma, beta, relu)
        if relu:
            fails = vcr_check.check_fwd(out["y"], vcr_check.relu_ln_fwd_reference(pre, gamma, beta), base["y"], dtype)
        else:
            assert out["dpre"] is None
            fails = vcr_check.check_fwd(out["y"], rc.ln_fwd_reference(pre, gamma, beta), base["y"], dtype)
        fails += vcr_check.check_bwd(out, vcr_check.relu_ln_bwd_reference(dy, pre, gamma, relu), base, pre, dtype,
                                     relu)
        assert not fails, (rows, fails)
        if deterministic:
            for reserve in (0, 8):
                lib.ub200_set_sm_reserve(reserve)
                again = _ln_run(pre, gamma, beta, dy, relu)
                for k, v in out.items():
                    if v is not None:
                        assert torch.equal(again[k], v), (rows, reserve, k)
            lib.ub200_set_sm_reserve(0)


def test_relu_layernorm_rejects_what_it_does_not_cover():
    from uniter_b200 import ops
    x = torch.randn(4, 2056, device="cuda", dtype=torch.float16)
    g = torch.ones(2056, device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="H <= 2048"):
        ops.layernorm_fwd(x, g, g, relu=True)
    x, g = x[:, :1536].contiguous(), g[:1536].contiguous()
    with pytest.raises(RuntimeError, match="dropout_p must be 0"):
        ops.layernorm_bwd(x, x, g, relu=True, dropout_p=0.1)


# ----------------------------------------------------------------------------- batches
def vcr_samples(seed, n_questions, vocab, D, txt=(6, 20), nbb=(4, 12), long_txt=None):
    """Per-question tuples of 4 choices shaped like VcrDataset's (qa type ids for even questions, qar
    for odd ones); every question uses a few of the 81 added tokens (ids >= vocab).  long_txt: the text
    length of question 0's first choice (to make one sequence longer than 128 tokens)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n_questions):
        nb = int(torch.randint(nbb[0], nbb[1] + 1, (1,), generator=g))
        feat, pos = torch.randn(nb, D, generator=g), torch.rand(nb, 7, generator=g)
        choices = []
        for c in range(4):
            tl = long_txt if (long_txt and i == 0 and c == 0) else int(torch.randint(txt[0], txt[1] + 1, (1,),
                                                                                        generator=g))
            ids = torch.randint(1000, vocab, (tl,), generator=g)
            ids[0] = 101
            ids[tl // 2] = vocab + int(torch.randint(0, N_SPECIAL, (1,), generator=g))
            q = tl // 3
            types = torch.tensor([0] * (q + 1) + [2] * (tl - q - 1)) if i % 2 == 0 else \
                torch.tensor([0] * (q + 1) + [2] * q + [3] * (tl - 2 * q - 1))
            choices.append((ids, types, feat, pos, torch.ones(tl + nb, dtype=torch.long),
                            torch.tensor([1 if c == 0 else 0])))
        out.append(tuple(choices))
    return out


def _on_device(batch):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}


def _zero_dropout(mod):
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return mod


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-6)).item()


def _config(geo):
    from uniter_b200.model import UniterConfig
    return UniterConfig(geo["vocab_size"], **{k: v for k, v in geo.items() if k not in ("vocab_size", "img_dim")})


# ----------------------------------------------------------------------------- model vs the reference
def _against_reference(geo, long_txt):
    from tests.test_reference_heads_gpu import _swap
    from uniter_b200.batching import vcr_collate
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    from uniter_b200.synth import seeded_state
    rm, rvcr = ref_loader.load("model.model", "model.vcr")
    rcfg = rm.UniterConfig(geo["vocab_size"], **{k: v for k, v in geo.items() if k not in ("vocab_size", "img_dim")})
    with _swap(rvcr):
        ref = rvcr.UniterForVisualCommonsenseReasoning(rcfg, geo["img_dim"])
    ours = UniterForVisualCommonsenseReasoning(_config(geo), geo["img_dim"])
    for m in (ref, ours):
        m.init_type_embedding()
        m.init_word_embedding(N_SPECIAL)
    st = seeded_state({k: tuple(v.shape) for k, v in ref.state_dict().items()}, seed=17)
    ref.load_state_dict(st, strict=True)
    ours.load_state_dict(st, strict=True)
    ref, ours = _zero_dropout(ref.cuda().half()), _zero_dropout(ours.cuda().half())
    host = vcr_collate(vcr_samples(5, 2, geo["vocab_size"], geo["img_dim"], long_txt=long_txt))
    if long_txt:
        assert max(a + b for a, b in zip(host["txt_lens"], host["num_bbs"])) > 128
    b = _on_device(host)
    with torch.no_grad():
        ref.eval(), ours.eval()
        want = ref(b, compute_loss=False)
        got = ours(b, compute_loss=False)
    assert got.shape == want.shape == (8, 1)
    assert (got.float() - want.float()).abs().max().item() <= 1e-2
    ref.train(), ours.train()
    lr = ref(b, compute_loss=True)
    lo = ours(b, compute_loss=True)
    assert lo.dim() == 0 and lo.dtype == torch.float32
    assert abs(lo.item() - lr.float().item()) <= 2e-2 * abs(lr.float().item()) + 1e-3
    (lr.float() * 64).backward()
    (lo * 64).backward()
    gr, go = dict(ref.named_parameters()), dict(ours.named_parameters())
    names = [n for n in go if n.startswith("vcr_output.")] + [
        "uniter.pooler.dense.weight", "uniter.encoder.layer.0.attention.self.query.weight",
        "uniter.encoder.layer.0.intermediate.dense.weight"]
    for n in names:
        assert go[n].grad is not None and gr[n].grad is not None, n
        assert _rel(go[n].grad, gr[n].grad) <= 2e-2, (n, _rel(go[n].grad, gr[n].grad))
    tt = "uniter.embeddings.token_type_embeddings.weight"
    assert _rel(go[tt].grad[2:4], gr[tt].grad[2:4]) <= 2e-2
    assert gr[tt].grad[2:4].float().norm() > 0
    ww = "uniter.embeddings.word_embeddings.weight"
    special = torch.unique(host["input_ids"][host["input_ids"] >= geo["vocab_size"]]).cuda()
    assert special.numel() > 0
    assert _rel(go[ww].grad[special], gr[ww].grad[special]) <= 2e-2


@needs_reference
def test_model_matches_the_unmodified_reference_base():
    _against_reference(util.BASE_L1, long_txt=150)


@needs_reference
def test_model_matches_the_unmodified_reference_large():
    _against_reference(util.LARGE_L1, long_txt=None)


# ----------------------------------------------------------------------------- graphed steps
def _vcr_model(dtype=torch.float16):
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    torch.manual_seed(0)
    mod = UniterForVisualCommonsenseReasoning(util.tiny_config(), 64)
    mod.init_type_embedding()
    mod.init_word_embedding(N_SPECIAL)
    mod.load_state_dict(util.head_state(mod, seed=19), strict=True)
    return _zero_dropout(mod.to("cuda", dtype).train())


def _graph_host(seed, long_txt=None):
    from uniter_b200.batching import vcr_collate
    b = vcr_collate(vcr_samples(seed, 3, util.TINY["vocab_size"], 64, long_txt=long_txt))
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    tensors = {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}
    return tensors, lens


def test_graphed_vcr_step_equals_the_eager_step():
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.model import register_lengths
    mod = _vcr_model()
    loss_fn = lambda b: mod(b)                      # noqa: E731
    host, lens = _graph_host(81)
    b = {k: v.cuda() for k, v in host.items()}
    register_lengths(b["attn_masks"], lens, prefix=True)
    mod.zero_grad(set_to_none=True)
    eager = loss_fn(b)
    eager.backward()
    eager = eager.detach()
    ref_g = {n: p.grad.detach().clone() for n, p in mod.named_parameters() if p.grad is not None}
    assert "uniter.embeddings.token_type_embeddings.weight" in ref_g and "vcr_output.0.weight" in ref_g
    step = GraphedStep(mod, loss_fn, token_bucket=64)
    for _ in range(2):
        loss = step(host, lens)
        torch.cuda.synchronize()
        assert torch.equal(loss, eager), (loss.item(), eager.item())
        got = {n: p.grad for n, p in mod.named_parameters()}
        for n, g in ref_g.items():
            d = (got[n].float() - g.float()).norm().item()
            assert d <= 4e-3 * g.float().norm().item() + 1e-6, (n, d)
    assert step.captures == 1
    w = mod.vcr_output[0].weight
    assert w.grad.data_ptr() == step.arena.view(w).data_ptr()


def test_graphed_fp16_vcr_steps_are_bit_reproducible(monkeypatch):
    from tests.test_reproducible_step_gpu import _assert_identical, _graphed_run
    from uniter_b200.optim import DynamicLossScaler
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    mod = _vcr_model()
    init = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    calls = [(_graph_host(s)[0], _graph_host(s)[1], {}) for s in (91, 92)]
    assert max(max(c[1]) for c in calls) <= 128
    loss_fn = lambda b: mod(b)                      # noqa: E731
    torch.use_deterministic_algorithms(True)
    runs = []
    for _ in range(2):
        snap, _ = _graphed_run(mod, init, loss_fn, calls, scaler=DynamicLossScaler(init_scale=2.**12))
        runs.append(snap)
    _assert_identical(runs, ["first", "second"])
    assert not torch.equal(runs[0]["weight vcr_output.0.weight"], init["vcr_output.0.weight"])


def test_long_vcr_batch_is_refused_under_the_deterministic_flag():
    from uniter_b200.model import register_lengths
    mod = _vcr_model()
    host, lens = _graph_host(93, long_txt=120)
    assert max(lens) > 128
    b = {k: v.cuda() for k, v in host.items()}
    register_lengths(b["attn_masks"], lens, prefix=True)
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="deterministic"):
        mod(b).backward()


# ----------------------------------------------------------------------------- stale arena
def test_init_after_a_warmup_step_uses_a_fresh_arena():
    """A warm-up step before init_* builds an arena over the 2-row type table and the V-row word table;
    the step after init_* must write into a fresh arena that holds the new tables, with the same
    gradients as a model that was initialised before any step.  A GraphedStep built before the init
    refuses to run.  (Deterministic mode: the two runs are compared bit for bit.)"""
    from uniter_b200.arena import GradArena
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    from uniter_b200.model import register_lengths

    def build(warmup):
        torch.manual_seed(0)
        mod = _zero_dropout(UniterForVisualCommonsenseReasoning(util.tiny_config(), 64).to("cuda", torch.float16))
        mod.train()
        step = None
        if warmup:
            host, lens = _graph_host(71)          # ids < V and type ids < 2 are all a 2-row table takes
            host = dict(host, input_ids=host["input_ids"] % util.TINY["vocab_size"],
                        txt_type_ids=host["txt_type_ids"].clamp(max=1))
            b = {k: v.cuda() for k, v in host.items()}
            register_lengths(b["attn_masks"], lens, prefix=True)
            mod(b).backward()
            step = GraphedStep(mod, lambda bb: mod(bb), token_bucket=64)
        old = GradArena.of(mod) if warmup else None
        torch.manual_seed(1)
        mod.init_type_embedding()
        mod.init_word_embedding(N_SPECIAL)
        return mod, old, step

    torch.use_deterministic_algorithms(True)
    host, lens = _graph_host(72)
    grads = []
    for warmup in (True, False):
        mod, old, step = build(warmup)
        mod.zero_grad(set_to_none=True)
        b = {k: v.cuda() for k, v in host.items()}
        register_lengths(b["attn_masks"], lens, prefix=True)
        mod(b).backward()
        torch.cuda.synchronize()
        te = mod.uniter.embeddings
        arena = mod.uniter._ensure_arena()[0]
        assert arena._still_valid()
        for p in (te.word_embeddings.weight, te.token_type_embeddings.weight):
            assert p.grad is not None and p.grad.data_ptr() == arena.view(p).data_ptr()
        if warmup:
            assert old is not arena and not old._still_valid()
            with pytest.raises(RuntimeError, match="replaced"):
                step(host, lens)
        grads.append({n: p.grad.detach().clone() for n, p in mod.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys()
    for n in grads[1]:
        assert torch.equal(grads[0][n], grads[1][n]), n
