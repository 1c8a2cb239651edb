"""GPU: the referring-expression head (ub200_region_score_*, uniter_b200.heads.
UniterForReferringExpressionComprehension).

* The kernels against float64 (tests/re_check.py) in fp16 and bf16 at H = 768 and 1024: segments of 1,
  2, 37 and 100 regions with padding rows between and after them, interior obj_masks, both losses, hard
  and easy negatives, a hinge exactly at 0 and a tie between two hard negatives; the same bits from
  two runs and under two SM reserves.
* The model against the UNMODIFIED reference class (model/re.py, staged into oracle/_ref by build())
  over the drop-in encoder with the same seeded weights, mlp 1 and 2, both losses, the same negatives.
* A GraphedStep replay of an RE step equals the eager step, and two graphed fp16 steps with the loss
  scaler and FusedAdamW under torch.use_deterministic_algorithms give the same bits.
"""
import os
import random
import sys

import numpy as np
import pytest
import torch

from oracle import ref_loader
from tests import re_check, util

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="reference sources not staged")

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_re_goldens  # noqa: E402


@pytest.fixture(autouse=True)
def torch_flags():
    import torch.utils.deterministic as tud
    from uniter_b200 import _lib
    saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
             tud.fill_uninitialized_memory)
    yield
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])
    tud.fill_uninitialized_memory = saved[2]
    _lib.load().ub200_set_sm_reserve(0)


# ----------------------------------------------------------------------------- kernels vs float64
def _kernel_case(dtype, H, mode):
    """Six samples with padding rows before, between and after them.  cls: lengths 1, 2, 37, 100, 5, 9;
    rank: 2, 3, 37, 100, 5, 9.  Sample 4's negative has the target's row (equal scores: the hinge is
    exactly the margin); sample 5's two best regions have identical rows (a tie for the hard negative)."""
    g = torch.Generator().manual_seed(H + mode)
    lens = [1, 2, 37, 100, 5, 9] if mode == re_check.CLS else [2, 3, 37, 100, 5, 9]
    starts, r = [], 2
    for n in lens:
        starts.append(r)
        r += n + 1
    R = r + 7
    rows = torch.randn(R, H, generator=g)
    w = torch.randn(H, generator=g) * (2.0 / H ** 0.5)
    st4, st5 = starts[4], starts[5]
    rows[st4 + 1] = rows[st4]
    rows[st5 + 2] = w * 2.0
    rows[st5 + 6] = rows[st5 + 2]
    rows, w = rows.to(dtype).cuda(), w.to(dtype).cuda()
    b = torch.tensor([-0.3]).to(dtype).cuda()
    seg = torch.tensor([starts, lens], dtype=torch.int32).cuda()
    S = max(lens)
    om = torch.zeros(len(lens), S, dtype=torch.uint8)
    for i, n in enumerate(lens):
        om[i, n:] = 1
    om[2, 3] = om[2, 10] = om[3, 50] = 1
    targets = torch.tensor([0, 1, 4, 77, 0, 0]).cuda()
    plan = torch.tensor([-1, 0, -1, 12, 1, -1]).cuda()
    dloss = (torch.rand(len(lens), generator=g) + 0.5).cuda()
    return rows, w, b, seg, om.cuda(), targets, plan, dloss


def _kernel_run(rows, w, b, seg, om, targets, plan, dloss, mode, margin):
    from uniter_b200 import ops
    scores, loss, lse, neg = ops.region_score_fwd(rows, w, b, seg, om, targets, plan, mode, margin)
    d_rows, dw, db = ops.region_score_bwd(rows, w, seg, om, targets, scores, lse, neg, dloss, mode, margin)
    torch.cuda.synchronize()
    return {"scores": scores, "loss": loss, "neg": neg, "d_rows": d_rows, "dw": dw, "db": db}


CASES = [(re_check.CLS, 0.0), (re_check.RANK, 0.2), (re_check.RANK, 0.0)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H", [768, 1024])
@pytest.mark.parametrize("mode,margin", CASES)
def test_region_score_kernels_match_float64(dtype, H, mode, margin):
    from uniter_b200 import _lib, ops
    case = _kernel_case(dtype, H, mode)
    rows, w, b, seg, om, targets, plan, dloss = case
    out = _kernel_run(*case, mode, margin)
    if mode == re_check.CLS:
        out["neg"] = None
    ref = re_check.reference(rows, w, b, seg, om, out["scores"], targets, plan, mode, margin, dloss)
    base = re_check.baseline(rows, w, b, seg, om, targets, ref["neg"].clamp(min=0), mode, margin, dloss)
    re_check.check(out, ref, dtype, base)
    if mode == re_check.RANK:
        assert out["neg"].tolist()[5] == 2                          # the tie goes to the lower index
        if margin == 0.0:                                           # hinge exactly 0: the gradient passes
            assert float(out["loss"][4]) == 0.0 and float(ref["dscore"][4].abs().sum()) > 0
    # eval scores are the same bits; every output repeats bit for bit, whatever the SM reserve
    scores_only, _, _, _ = ops.region_score_fwd(rows, w, b, seg, om)
    assert torch.equal(scores_only, out["scores"])
    lib = _lib.load()
    for reserve in (0, 0, 8):
        lib.ub200_set_sm_reserve(reserve)
        again = _kernel_run(*case, mode, margin)
        for k, v in out.items():
            if v is not None:
                assert torch.equal(again[k], v), (reserve, k)
    lib.ub200_set_sm_reserve(0)


# ----------------------------------------------------------------------------- model vs the reference
def _re_batch(seed, n=6):
    from uniter_b200.batching import re_collate
    return re_collate(make_re_goldens.re_samples(seed, n, D=64))


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


@needs_reference
@pytest.mark.parametrize("mlp", [1, 2])
@pytest.mark.parametrize("loss", ["cls", "rank"])
def test_model_matches_the_unmodified_reference_head(mlp, loss):
    from tests.test_reference_heads_gpu import _swap, _tiny_ref_config
    from uniter_b200.heads import UniterForReferringExpressionComprehension, re_neg_plan
    from uniter_b200.synth import seeded_state
    rm, rre = ref_loader.load("model.model", "model.re")
    with _swap(rre):
        ref = rre.UniterForReferringExpressionComprehension(_tiny_ref_config(rm), 64, loss=loss, mlp=mlp)
    ours = UniterForReferringExpressionComprehension(util.tiny_config(), 64, loss=loss, mlp=mlp)
    st = seeded_state({k: tuple(v.shape) for k, v in ref.state_dict().items()}, seed=12)
    ref.load_state_dict(st, strict=True)
    ours.load_state_dict(st, strict=True)
    ref, ours = _zero_dropout(ref.cuda().half()), _zero_dropout(ours.cuda().half())
    host = _re_batch(71)
    b = _on_device(host)
    b_ref = dict(b, obj_masks=b["obj_masks"].bool())
    with torch.no_grad():
        ref.eval(), ours.eval()
        want = ref(b_ref, compute_loss=False)
        got = ours(b, compute_loss=False)
    assert got.shape == want.shape
    assert (got.float() - want.float()).abs().max().item() <= 1e-2
    ref.train(), ours.train()
    np_state, py_state = np.random.get_state(), random.getstate()
    try:
        if loss == "rank":
            np.random.seed(5)
            random.seed(5)
            plan = re_neg_plan(host["targets"].view(-1).tolist(), host["num_bbs"], ours.hard_ratio)
            b["re_neg_plan"] = torch.tensor(plan).cuda()
            np.random.seed(5)
            random.seed(5)
        lr = ref(b_ref, compute_loss=True)
    finally:
        np.random.set_state(np_state)
        random.setstate(py_state)
    lo = ours(b, compute_loss=True)
    assert lo.shape == lr.shape and lo.dtype == torch.float32
    assert (lo - lr.float()).norm().item() <= 2e-2 * lr.float().norm().item() + 1e-3
    (lr.float().sum() * 64).backward()
    (lo.sum() * 64).backward()
    gr, go = dict(ref.named_parameters()), dict(ours.named_parameters())
    names = [n for n in go if n.startswith("re_output.")] + [
        "uniter.img_embeddings.img_linear.weight", "uniter.encoder.layer.0.attention.self.query.weight"]
    for n in names:
        assert go[n].grad is not None and gr[n].grad is not None, n
        if gr[n].grad.float().norm() == 0:
            assert go[n].grad.float().norm() == 0, n
            continue
        assert _rel(go[n].grad, gr[n].grad) <= 2e-2, (n, _rel(go[n].grad, gr[n].grad))


# ----------------------------------------------------------------------------- graphed steps
def _re_model(loss="rank", mlp=1, dtype=torch.float16):
    from uniter_b200.heads import UniterForReferringExpressionComprehension
    torch.manual_seed(0)
    mod = UniterForReferringExpressionComprehension(util.tiny_config(), 64, loss=loss, mlp=mlp)
    mod.load_state_dict(util.head_state(mod, seed=13), strict=True)
    return _zero_dropout(mod.to("cuda", dtype).train())


def _graph_host(seed):
    from uniter_b200.heads import re_neg_plan
    b = _re_batch(seed, n=8)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    b["re_neg_plan"] = torch.tensor(re_neg_plan(b["targets"].view(-1).tolist(), b["num_bbs"], 0.3,
                                                np_random=np.random.RandomState(seed),
                                                py_random=random.Random(seed)))
    tensors = {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}
    return b, tensors, lens


def test_graphed_re_step_equals_the_eager_step():
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.model import register_lengths
    mod = _re_model()
    loss_fn = lambda b: mod(b).sum()                    # noqa: E731
    full, host, lens = _graph_host(81)
    # eager, from the index keys, and from the host lists alone: the same loss bits
    b = {k: v.cuda() for k, v in host.items()}
    register_lengths(b["attn_masks"], lens, prefix=True)
    mod.zero_grad(set_to_none=True)
    eager = loss_fn(b)
    eager.backward()
    eager = eager.detach()          # frees the autograd graph: its AccumulateGrad nodes belong to this stream
    ref_g = {n: p.grad.detach().clone() for n, p in mod.named_parameters() if p.grad is not None}
    lists = {k: v for k, v in _on_device(full).items() if k not in ("re_index", "re_seg")}
    with torch.no_grad():
        assert torch.equal(mod(lists).sum(), eager)
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
    w = mod.re_output.weight
    assert w.grad.data_ptr() == step.arena.view(w).data_ptr()


@pytest.mark.parametrize("mlp", [1, 2])
def test_graphed_fp16_re_steps_are_bit_reproducible(monkeypatch, mlp):
    from tests.test_reproducible_step_gpu import _assert_identical, _graphed_run
    from uniter_b200.optim import DynamicLossScaler
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    mod = _re_model(loss="cls", mlp=mlp)
    init = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    calls = [(_graph_host(s)[1], _graph_host(s)[2], {}) for s in (91, 92)]
    loss_fn = lambda b: mod(b).sum() / b["targets"].numel()     # noqa: E731
    torch.use_deterministic_algorithms(True)
    runs = []
    for _ in range(2):
        snap, _ = _graphed_run(mod, init, loss_fn, calls, scaler=DynamicLossScaler(init_scale=2.**12))
        runs.append(snap)
    _assert_identical(runs, ["first", "second"])
    assert not torch.equal(runs[0]["weight re_output.3.weight" if mlp == 2 else "weight re_output.weight"],
                           init["re_output.3.weight" if mlp == 2 else "re_output.weight"])
