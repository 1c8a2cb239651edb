"""GPU: word-region alignment (ub200_wra_*, UniterForPretraining.forward_itm with ot_inputs).

* The kernels against float64 (tests/wra_check.py) in fp16 and bf16 at H = 768 and 1024: C4's length
  draws, the pre-training configs' maximum of 62 text rows x 100 regions, pairs with m = 1 or n = 1, the
  largest supported max_m * max_n, and rows of a padding sequence after the pairs; the same bits twice.
* One text length above the supported extent is a ValueError before any launch.
* The library's forward_itm with ot_inputs against the reference's outputs stored in tests/golden/wra.npz.
* The UNMODIFIED reference UniterForPretraining (model/ot.py's `trace` replaced by the diagonal sum, pads
  passed as bool) over the drop-in encoder, against the library.
* A GraphedStep replay of an ITM + WRA step equals the eager step, and graphed fp16 ITM + WRA steps with
  the loss scaler and FusedAdamW under torch.use_deterministic_algorithms give the same bits.
"""
import os
import sys

import pytest
import torch

from oracle import ref_loader
from tests import util, wra_check

pytestmark = pytest.mark.gpu
needs_reference = pytest.mark.skipif(not ref_loader.available(), reason="reference sources not staged")

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_wra_goldens  # noqa: E402

ITM_OT_LAMBDA = make_wra_goldens.ITM_OT_LAMBDA


@pytest.fixture(autouse=True)
def torch_flags():
    import torch.utils.deterministic as tud
    saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
             tud.fill_uninitialized_memory)
    yield
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])
    tud.fill_uninitialized_memory = saved[2]


# ----------------------------------------------------------------------------- kernels vs float64
def _geometry(case):
    g = torch.Generator().manual_seed(17)
    if case == "c4":
        return [(int(torch.randint(12, 29, (1,), generator=g)), int(torch.randint(26, 47, (1,), generator=g)))
                for _ in range(8)]
    if case == "config_max":
        return [(62, 100), (40, 100), (62, 73)]
    if case == "m1_n1":
        return [(1, 9), (7, 1), (1, 1), (13, 30)]
    if case == "limit":
        return [(88, 128), (5, 3)]
    raise ValueError(case)


def _inputs(case, H, dtype, pad_rows=11):
    geo = _geometry(case)
    g = torch.Generator().manual_seed(5)
    T = sum(m + n for m, n in geo)
    packed = (torch.randn(T + pad_rows, H, generator=g) + 0.05 * torch.randn(1, H, generator=g)).to(dtype)
    cu = [0]
    for m, n in geo:
        cu.append(cu[-1] + m + n)
    tl = [m for m, _ in geo]
    dg = torch.randn(len(geo), generator=g).to(dtype).float()
    return packed, cu, tl, dg, max(m for m, _ in geo), max(n for _, n in geo)


def _kernel_run(packed, cu, tl, dg, max_m, max_n):
    from uniter_b200 import ops
    dev_p = packed.cuda()
    cu_d = torch.tensor(cu, dtype=torch.int32, device="cuda")
    tl_d = torch.tensor(tl, dtype=torch.int32, device="cuda")
    B = len(tl)
    ws = ops.wra_workspace(B, max_m, max_n, dev_p.device)
    dist = ops.wra_fwd(dev_p, cu_d, tl_d, B, max_m, max_n, ws)
    d = ops.wra_bwd(dev_p, cu_d, tl_d, B, max_m, max_n, ws, dg.cuda())
    torch.cuda.synchronize()
    return {"dist": dist, "d_packed": d}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("H", [768, 1024])
@pytest.mark.parametrize("case", ["c4", "config_max", "m1_n1", "limit"])
def test_kernels_match_float64(case, H, dtype):
    from uniter_b200 import _lib
    packed, cu, tl, dg, max_m, max_n = _inputs(case, H, dtype)
    if case == "limit":
        assert max_m * max_n == _lib.WRA_MAX_MN
    out = _kernel_run(packed, cu, tl, dg, max_m, max_n)
    ref = wra_check.reference(packed, cu, tl, dg)
    base = wra_check.baseline(packed.cuda(), cu, tl, dg)
    wra_check.check(out, ref, dtype, base)
    again = _kernel_run(packed, cu, tl, dg, max_m, max_n)
    assert torch.equal(again["dist"], out["dist"]) and torch.equal(again["d_packed"], out["d_packed"])


def _tiny_pretraining(dtype=torch.float16):
    from uniter_b200.heads import UniterForPretraining
    from uniter_b200.synth import seeded_state
    mod = UniterForPretraining(util.tiny_config(), 64, 11)
    st = seeded_state({k: tuple(v.shape) for k, v in mod.state_dict().items()}, seed=make_wra_goldens.WRA_STATE_SEED)
    mod.load_state_dict(st, strict=True)
    return mod.to("cuda", dtype), st


def _itm_batch(seed=81, n=6, tl_max=None):
    from uniter_b200.batching import itm_ot_collate
    return itm_ot_collate(make_wra_goldens.wra_samples(seed, n, D=64))


def _on_device(batch):
    out = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch.items()}
    out["ot_inputs"] = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in batch["ot_inputs"].items()}
    return out


def _combined(itm_loss, ot):
    pos, neg = ot
    return itm_loss.float().mean() + ITM_OT_LAMBDA * (pos.float().sum() - neg.float().sum()) / (pos.numel() + neg.numel())


def test_extent_above_the_limit_is_a_value_error_before_any_launch():
    import ctypes
    from uniter_b200 import _lib
    from uniter_b200.batching import itm_ot_collate
    mod, _ = _tiny_pretraining()
    g = torch.Generator().manual_seed(3)
    samples = [(torch.randint(1000, 1999, (m,), generator=g), torch.randn(n, 64, generator=g), torch.rand(n, 7, generator=g),
                torch.ones(m + n, dtype=torch.long), torch.tensor([1])) for m, n in ((89, 128), (4, 6))]
    b = _on_device(itm_ot_collate(samples))
    lib = _lib.load()
    lib.ub200_launch_count.restype = ctypes.c_ulonglong
    n0 = lib.ub200_launch_count()
    with pytest.raises(ValueError):
        mod(b, "itm")
    assert lib.ub200_launch_count() == n0
    # a pair whose text and region counts do not fill its valid tokens
    b = _on_device(_itm_batch())
    b["txt_lens"] = [t + 1 for t in b["txt_lens"]]
    with pytest.raises(ValueError):
        mod(b, "itm")
    assert lib.ub200_launch_count() == n0


# ----------------------------------------------------------------------------- model vs the reference
def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-6)).item()


@pytest.mark.parametrize("keys", ["host_keys", "pads_only"])
def test_forward_itm_matches_the_stored_reference(keys):
    from tests.golden.make_goldens import state_checksum
    g = util.load_golden("wra")
    mod, st = _tiny_pretraining()
    assert abs(state_checksum(st) - float(g["itm/checksum"])) <= 1e-6 * abs(float(g["itm/checksum"]))
    mod.eval()
    b = _on_device(_itm_batch())
    if keys == "pads_only":        # the reference's batch: the pads (bool here) are read once
        for k in ("txt_lens", "num_bbs", "ot_txt_lens", "ot_pos_index", "ot_neg_index"):
            del b[k]
        b["ot_inputs"] = dict(b["ot_inputs"], txt_pad=b["ot_inputs"]["txt_pad"].bool())
    itm_loss, ot = mod(b, "itm")
    loss = _combined(itm_loss, ot)
    for name, got in (("itm_loss", itm_loss), ("ot_pos", ot[0]), ("ot_neg", ot[1]), ("loss", loss)):
        want = torch.from_numpy(g["itm/" + name]).float()
        assert got.shape == want.shape, name
        assert (got.float().cpu() - want).abs().max().item() <= 1e-2, name
    (loss * 64).backward()
    params = dict(mod.named_parameters())
    for k in make_wra_goldens.GRAD_KEYS:
        want = torch.from_numpy(g["itm/grad/" + k]) * 64
        assert _rel(params[k].grad, want) <= 2e-2, (k, _rel(params[k].grad, want))
    with torch.no_grad():
        scores, ot2 = mod(b, "itm", compute_loss=False)
    assert scores.shape == (6, 2) and torch.equal(ot2[0], ot[0]) and torch.equal(ot2[1], ot[1])


@needs_reference
def test_unmodified_reference_over_the_drop_in_encoder():
    from tests.test_reference_heads_gpu import _swap, _tiny_ref_config
    from uniter_b200.heads import UniterForPretraining
    from uniter_b200.synth import seeded_state
    rm, rpre, rot = ref_loader.load("model.model", "model.pretrain", "model.ot")
    saved_trace = rot.trace
    rot.trace = make_wra_goldens.trace_diag
    try:
        with _swap(rpre):
            ref = rpre.UniterForPretraining(_tiny_ref_config(rm), 64, 11)
        ours = UniterForPretraining(util.tiny_config(), 64, 11)
        st = seeded_state({k: tuple(v.shape) for k, v in ref.state_dict().items()}, seed=31)
        ref.load_state_dict(st, strict=True)
        ours.load_state_dict(st, strict=True)
        ref, ours = ref.cuda().half().eval(), ours.cuda().half().eval()
        b = _on_device(_itm_batch(85, 8))
        b_ref = dict(b, ot_inputs=dict(b["ot_inputs"], txt_pad=b["ot_inputs"]["txt_pad"].bool(),
                                       img_pad=b["ot_inputs"]["img_pad"].bool()))
        lr, otr = ref(b_ref, task="itm", compute_loss=True)
        lo, oto = ours(b, "itm")
        for x, y in ((lo, lr), (oto[0], otr[0]), (oto[1], otr[1]), (_combined(lo, oto), _combined(lr, otr))):
            assert x.shape == y.shape
            assert (x.float() - y.float()).abs().max().item() <= 1e-2
        (_combined(lr, otr) * 64).backward()
        (_combined(lo, oto) * 64).backward()
    finally:
        rot.trace = saved_trace
    gr, go = dict(ref.named_parameters()), dict(ours.named_parameters())
    for n in make_wra_goldens.GRAD_KEYS:
        assert _rel(go[n].grad, gr[n].grad) <= 2e-2, (n, _rel(go[n].grad, gr[n].grad))


# ----------------------------------------------------------------------------- graphed steps
def _wra_loss(mod):
    def loss_fn(b):
        # a graphed step sees the batch's tensors only: ot_txt_lens / ot_pos_index / ot_neg_index carry WRA
        itm_loss, ot = mod(dict(b, ot_inputs={}), "itm")
        return _combined(itm_loss, ot)
    return loss_fn


def _graph_host(seed, n=8):
    b = _itm_batch(seed, n)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    tensors = {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}
    return tensors, lens


def test_graphed_itm_wra_step_equals_the_eager_step():
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.model import register_lengths
    mod, _ = _tiny_pretraining()
    mod.train()
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    loss_fn = _wra_loss(mod)
    host, lens = _graph_host(87)
    b = {k: v.cuda() for k, v in host.items()}
    register_lengths(b["attn_masks"], lens, prefix=True)
    mod.zero_grad(set_to_none=True)
    eager = loss_fn(b)
    eager.backward()
    eager = eager.detach()
    ref_g = {n: p.grad.detach().clone() for n, p in mod.named_parameters() if p.grad is not None}
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


def test_graphed_fp16_itm_wra_steps_are_bit_reproducible(monkeypatch):
    from tests.test_reproducible_step_gpu import _assert_identical, _graphed_run
    from uniter_b200.optim import DynamicLossScaler
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    mod, _ = _tiny_pretraining()
    mod.train()
    init = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    calls = [_graph_host(s) + ({},) for s in (91, 92)]
    torch.use_deterministic_algorithms(True)
    runs = []
    for _ in range(2):
        snap, _ = _graphed_run(mod, init, _wra_loss(mod), calls, scaler=DynamicLossScaler(init_scale=2.**12))
        runs.append(snap)
    _assert_identical(runs, ["first", "second"])
    assert not torch.equal(runs[0]["weight itm_output.weight"], init["itm_output.weight"])
