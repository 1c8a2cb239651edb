"""GPU: dynamic fp16 loss scaling on the device (ub200_adam_prep_scaled + ub200_adamw_step_scaled,
uniter_b200.optim.DynamicLossScaler, GraphedStep(loss_scaler=...)).

  * the prep kernel against the host policy (oracle/loss_scaler.py), bit for bit, over a long stream
    of finite / inf / NaN norms with three loss ids;
  * the optimizer trajectory with gradients carrying the current scale, against the AdamW oracle on
    the unscaled gradients with the overflowed steps skipped;
  * a captured fp16 step against the same steps run eagerly: the same scale / skip trajectory, one
    capture, no host read inside the replay;
  * one scaler per pre-training task, accumulation windows, and resuming from state_dict().
"""
import math

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as orc
from oracle.loss_scaler import LossScaler, ScaledStepState
from tests import util

pytestmark = pytest.mark.gpu

INF, NAN = float("inf"), float("nan")


def _row(table, k):
    """(scale, unskipped, inv_scale) of entry k of a ub200_loss_scaler table (host copy)."""
    t = table.cpu()
    return float(t[k, 0]), int(t.view(torch.int32)[k, 1]), float(t[k, 2])


def _is_pow2(x):
    m, _ = math.frexp(x)
    return x > 0 and m == 0.5


# ------------------------------------------------------------------------------ kernel vs oracle
def _prep_stream():
    """(loss_id, sumsq) pairs.  id 0: apex defaults, two overflows then > 2000 clean steps (one
    doubling); id 1: starts at 2^23, doubles to the 2^24 cap after 2000 clean steps and stays there
    when the next window completes, then a NaN; id 2: window 3 with a floor of 1, frequent overflows
    of every kind (inf, -inf, NaN, a finite sum above the 3e38 limit)."""
    rng = np.random.default_rng(7)
    clean = lambda n: list(rng.uniform(1e-3, 1e6, n))
    per_id = {
        0: clean(10) + [INF] + clean(9) + [NAN] + clean(2100) + [INF] + clean(30),
        1: clean(4100) + [NAN] + clean(40),
        2: [],
    }
    bad = [INF, -INF, NAN, 3.2e38]
    for _ in range(300):
        per_id[2].append(bad[rng.integers(4)] if rng.random() < 0.4 else float(rng.uniform(0, 1e3)))
    seq, pos = [], {k: 0 for k in per_id}
    while any(pos[k] < len(v) for k, v in per_id.items()):
        live = [k for k, v in per_id.items() if pos[k] < len(v)]
        k = live[rng.integers(len(live))]
        seq.append((k, per_id[k][pos[k]]))
        pos[k] += 1
    return seq


def test_prep_kernel_matches_the_host_policy_bit_for_bit():
    from uniter_b200 import _lib
    from uniter_b200.optim import DynamicLossScaler, scaler_table
    lib = _lib.load()
    policies = [(2.**16, 2000, 2.**24, None), (2.**23, 2000, 2.**24, None), (2.0, 3, 2.**24, 1.0)]
    sc = DynamicLossScaler(num_losses=3)
    sc.table.copy_(scaler_table([(s, 0, w, mx, mn) for s, w, mx, mn in policies]))
    orc_state = ScaledStepState([LossScaler(s, w, mx, mn) for s, w, mx, mn in policies])
    seq = _prep_stream()
    n = len(seq)
    assert n > 6000
    sums = torch.tensor([v for _, v in seq], dtype=torch.float32, device="cuda")
    state = torch.zeros(4, dtype=torch.int32, device="cuda")
    rec_tab = torch.empty(n, 8, dtype=torch.float32, device="cuda")
    rec_st = torch.empty(n, 4, dtype=torch.int32, device="cuda")
    stream = _lib.current_stream()
    for i, (k, _) in enumerate(seq):
        _lib.check(lib.ub200_adam_prep_scaled(sums.data_ptr() + 4 * i, state.data_ptr(), sc.table.data_ptr(),
                                              k, stream))
        rec_tab[i].copy_(sc.table[k])
        rec_st[i].copy_(state)
    tab, st = rec_tab.cpu(), rec_st.cpu()
    tab_i = tab.view(torch.int32)
    seen_cap = seen_floor = False
    prev = [float(p[0]) for p in policies]
    for i, (k, v) in enumerate(seq):
        inv = orc_state.prep(v, k)
        o = orc_state.scalers[k]
        got = (float(tab[i, 0]), int(tab_i[i, 1]), float(tab[i, 2]))
        assert got == (float(o.scale), o.unskipped, float(inv)), (i, k, v, got)
        assert (int(st[i, 0]), int(st[i, 1]), int(st[i, 2])) == (orc_state.step, orc_state.found_inf,
                                                                  orc_state.skipped), (i, k, v)
        assert _is_pow2(got[0]) and _is_pow2(1.0 / got[2])
        # a window completed AT the cap: the counter restarts, the scale stays
        seen_cap |= k == 1 and prev[1] == 2.**24 and got[:2] == (2.**24, 0) and orc_state.found_inf == 0
        seen_floor |= k == 2 and prev[2] == 1.0 and got[0] == 1.0 and orc_state.found_inf == 1
        prev[k] = got[0]
    assert seen_cap and seen_floor
    # entries are independent: the final table is the three oracles', entry for entry
    for k in range(3):
        o = orc_state.scalers[k]
        assert _row(sc.table, k)[:2] == (float(o.scale), o.unskipped)
    assert orc_state.scalers[0].scale == 2.**14                # halved twice, doubled once, halved once
    assert orc_state.scalers[1].scale == 2.**23                # at the cap, then one NaN


# ------------------------------------------------------------------------------ optimizer trajectory
def test_fused_adamw_with_the_device_scaler_follows_the_oracle():
    """fp16 parameters, scale starting at 2^24 (the first steps overflow): masters follow
    orc.adamw_step on the UNSCALED gradients with the overflowed steps skipped, the clip uses the
    unscaled norm, and the model weights are round(master) after every step."""
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    gen = torch.Generator().manual_seed(11)
    shapes = [(300, 64), (64,), (4097,), (2, 3, 8)]
    wd = [0.01, 0.0, 0.01, 0.0]
    p0 = [(torch.randn(s, generator=gen) * 0.05).half() for s in shapes]
    params = [torch.nn.Parameter(x.clone().cuda()) for x in p0]
    opt = FusedAdamW([{"params": [params[0], params[2]], "weight_decay": 0.01},
                      {"params": [params[1], params[3]], "weight_decay": 0.0}], lr=1e-3)
    sc = DynamicLossScaler(init_scale=2.**24, scale_window=3)
    host = LossScaler(init_scale=2.**24, scale_window=3)
    max_norm = 1.0
    P = [x.float() for x in p0]
    M = [torch.zeros_like(x) for x in P]
    V = [torch.zeros_like(x) for x in P]
    t, overflows, clipped, scales = 0, 0, 0, []
    for it in range(16):
        scale = float(host.scale)
        assert sc.loss_scale() == scale
        scales.append(scale)
        grads16 = [(torch.randn(s, generator=gen) * 0.01 * scale).half() for s in shapes]
        for p, gr in zip(params, grads16):
            p.grad = gr.cuda()
        opt.step(grad_scale=sc, max_grad_norm=max_norm)
        ovf = not all(bool(torch.isfinite(gr).all()) for gr in grads16)
        inv = float(host.update(ovf))
        assert _row(sc.table, 0) == (float(host.scale), host.unskipped, inv)
        assert int(opt.found_inf.item()) == int(ovf)
        if ovf:
            overflows += 1
        else:
            t += 1
            un = [gr.float() * inv for gr in grads16]
            un, total = orc.clip_grad_norm(un, max_norm)
            total = float(total)
            assert abs(math.sqrt(opt.last_sumsq.item()) * inv - total) <= 1e-4 * total
            clipped += total > max_norm
            for i in range(len(P)):
                P[i], M[i], V[i] = orc.adamw_step(P[i], un[i], M[i], V[i], t, 1e-3, weight_decay=wd[i])
        for i in range(len(P)):
            master = opt.state[id(params[i])]["master"].cpu()
            np.testing.assert_allclose(master.numpy(), P[i].numpy(), atol=1e-6, rtol=1e-5)
            assert torch.equal(params[i].detach().cpu(), master.half())
    assert opt._applied_steps() == t and opt.skipped_steps() == overflows
    assert overflows >= 3 and t >= 6 and clipped >= 1
    assert any(b == 2 * a for a, b in zip(scales, scales[1:]))       # the window doubled the scale


# ------------------------------------------------------------------------------ model helpers
def _mlm_model(seed=9):
    from uniter_b200.heads import UniterForMLM
    torch.manual_seed(0)
    mod = UniterForMLM(util.tiny_config(), 64)
    mod.load_state_dict(util.head_state(mod, seed=seed), strict=False)
    mod = mod.to("cuda", torch.float16).train()
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    return mod


def _mlm_batch(seed, tl, nb):
    from uniter_b200.synth import pad_mlm_index, synth_batch
    b = synth_batch(len(tl), 0, 0, 0, 0, seed=seed, img_dim=64, vocab_size=2000, mlm_prob=0.3,
                    txt_lens=tl, num_bbs=nb)
    b = pad_mlm_index(b, 16)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    return {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens


# 128 tokens: the graph's token bucket holds the batch exactly, so the captured step launches the
# same kernels with the same shapes as the eager one
TL_128, NB_128 = [12, 10, 7, 9, 12, 8], [9, 13, 14, 9, 11, 14]


def _mlm_loss(mod):
    return lambda b: (mod(b).sum() * b["mlm_inv_n"]).squeeze()


def _params(mod):
    return {n: p.detach().clone() for n, p in mod.named_parameters()}


# ------------------------------------------------------------------------------ graph vs eager
def test_graphed_fp16_step_with_the_scaler_equals_the_eager_steps():
    """The scale and the skipped-step count follow the same trajectory, step for step, and the first
    loss is bit-identical.  Losses and weights after that agree to the run-to-run noise of the
    backward's fp32 atomics (DESIGN.md §2b: two runs of the same step differ in the last bits of
    some gradients), which Adam's normalised update carries into the weights."""
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.model import register_lengths
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    n_steps = 12
    hb, lens = _mlm_batch(51, TL_128, NB_128)
    assert sum(lens) == 128

    # eager: scaler.scale(loss).backward(); opt.step(grad_scale=scaler)
    mod = _mlm_model()
    opt = FusedAdamW(mod.parameters(), lr=1e-3)
    sc = DynamicLossScaler(init_scale=2.**24, scale_window=3)
    b = {k: v.cuda() for k, v in hb.items()}
    register_lengths(b["attn_masks"], lens, prefix=True)
    eager = []
    for _ in range(n_steps):
        opt.zero_grad()
        loss = _mlm_loss(mod)(b)
        sc.scale(loss).backward()
        opt.step(grad_scale=sc)
        eager.append((loss.detach().clone(), sc.loss_scale(), opt.skipped_steps()))
    eager_params = _params(mod)

    # graph: the same steps replayed from one capture
    mod2 = _mlm_model()
    opt2 = FusedAdamW(mod2.parameters(), lr=1e-3)
    sc2 = DynamicLossScaler(init_scale=2.**24, scale_window=3)
    step = GraphedStep(mod2, _mlm_loss(mod2), token_bucket=128, optimizer=opt2, loss_scaler=sc2)
    graphed = []
    for _ in range(n_steps):
        bk = step.stage(hb, lens)
        torch.cuda.set_sync_debug_mode("error")       # any device -> host read inside replay() raises
        try:
            loss = step.replay(bk)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        graphed.append((loss.clone(), sc2.loss_scale(), opt2.skipped_steps()))
    assert step.captures == 1

    scales = [e[1] for e in eager]
    assert [g[1:] for g in graphed] == [e[1:] for e in eager], (scales, [g[1] for g in graphed])
    assert torch.equal(graphed[0][0], eager[0][0])
    for i, (g, e) in enumerate(zip(graphed, eager)):
        assert math.isfinite(g[0].item())           # the returned loss is the unscaled one
        assert abs(g[0].item() - e[0].item()) <= 1e-3 * abs(e[0].item()), (i, g[0].item(), e[0].item())
    # the two runs' weights differ by a small fraction of how far the steps moved them
    got = _params(mod2)
    p0 = _params(_mlm_model())
    moved = sum(((p.float() - p0[n].float()) ** 2).sum().item() for n, p in eager_params.items()) ** 0.5
    apart = sum(((got[n].float() - p.float()) ** 2).sum().item() for n, p in eager_params.items()) ** 0.5
    assert moved > 0 and apart <= 0.05 * moved, (apart, moved)
    # the trajectory exercised the policy: overflows, halvings and a doubling
    assert eager[-1][2] >= 3 and len(set(scales)) >= 3
    assert any(b == 2 * a for a, b in zip(scales, scales[1:]))
    assert opt2._applied_steps() == n_steps - eager[-1][2] > 0


# ------------------------------------------------------------------------------ per-task scalers
def _pretrain_batches():
    from uniter_b200.synth import pad_mlm_index, synth_batch, synth_mrm
    mlm = pad_mlm_index(synth_batch(6, 5, 12, 3, 9, seed=61, img_dim=64, vocab_size=2000, mlm_prob=0.3), 16)
    mrfr = synth_mrm(synth_batch(6, 5, 12, 3, 9, seed=62, img_dim=64, vocab_size=2000), 0.3, 11, seed=3,
                     pad_multiple=16)
    for k in ("img_mask_tgt", "label_targets"):
        mrfr.pop(k)
    out = {}
    for task, b in (("mlm", mlm), ("mrfr", mrfr)):
        lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
        out[task] = ({k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens)
    return out


def test_one_scaler_per_pretraining_task():
    """mlm and mrfr cycled under loss ids 0 and 1; id 1 starts at a scale that overflows every
    mrfr step: its scale halves each time, id 0's scale and counter do not move on those steps,
    and the overflowed steps are skipped."""
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForPretraining
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    torch.manual_seed(0)
    mod = UniterForPretraining(util.tiny_config(), 64, 11)
    mod.load_state_dict(util.head_state(mod, seed=4, ties=util.PRETRAIN_TIES), strict=True)
    mod = mod.to("cuda", torch.float16).train()
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0

    def opt_state():
        return [st[k].clone() for st in opt.state.values() for k in ("master", "exp_avg", "exp_avg_sq")]

    def loss_fn(b, task):
        if task == "mlm":
            return (mod(b, "mlm").sum() * b["mlm_inv_n"]).squeeze()
        l = mod(b, "mrfr").float()
        return ((l * b["mrm_valid"].unsqueeze(1)).sum() * b["mrm_inv_n"] / l.size(1)).squeeze()

    opt = FusedAdamW(mod.parameters(), lr=1e-3)
    sc = DynamicLossScaler(num_losses=2, init_scale=2.**8)
    sc.load_state_dict({"loss_scaler0": {"loss_scale": 2.**8, "unskipped": 0},
                        "loss_scaler1": {"loss_scale": 2.**40, "unskipped": 0}})
    step = GraphedStep(mod, loss_fn, token_bucket=64, optimizer=opt, loss_scaler=sc,
                       loss_ids={"mlm": 0, "mrfr": 1})
    batches = _pretrain_batches()
    host = ScaledStepState([LossScaler(2.**8), LossScaler(2.**40)])
    for task in ("mlm", "mrfr", "mlm", "mrfr", "mlm"):
        lid = 0 if task == "mlm" else 1
        other = _row(sc.table, 1 - lid)
        before = opt_state()
        loss = step(*batches[task], tag=task)
        torch.cuda.synchronize()
        assert math.isfinite(loss.item()), task
        ovf = task == "mrfr"
        host.prep(INF if ovf else 1.0, lid)
        assert int(opt.found_inf.item()) == int(ovf), task
        o = host.scalers[lid]
        assert _row(sc.table, lid)[:2] == (float(o.scale), o.unskipped), task
        assert _row(sc.table, 1 - lid)[:2] == other[:2], task          # the other task's scaler
        if ovf:          # skipped: masters and moments untouched
            assert all(torch.equal(a, b) for a, b in zip(opt_state(), before)), task
    assert sc.loss_scale(1) == 2.**38 and sc.unskipped(1) == 0
    assert sc.loss_scale(0) == 2.**8 and sc.unskipped(0) == 3
    assert opt._applied_steps() == 3 and opt.skipped_steps() == 2
    assert step.captures == 2


# ------------------------------------------------------------------------------ accumulation
def test_accumulation_window_keeps_one_scale_and_steps_once():
    """Three micro-batches per optimizer step (accumulate=True after the first, the optimizer in the
    last one's graph only).  A window whose second micro-batch overflows is skipped as a whole and
    halves the scale once; the clean windows each count one step."""
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    mod = _mlm_model()
    opt = FusedAdamW(mod.parameters(), lr=1e-3)
    sc = DynamicLossScaler(init_scale=2.**10)
    # b["boost"] multiplies the loss: 2^30 makes the scaled gradients of that micro-batch overflow
    step = GraphedStep(mod, lambda b: (mod(b).sum() * b["mlm_inv_n"] * b["boost"]).squeeze(),
                       token_bucket=64, optimizer=opt, loss_scaler=sc)
    hb, lens = _mlm_batch(71, TL_128, NB_128)

    def window(boosts):
        for j, bst in enumerate(boosts):
            b = dict(hb, boost=torch.tensor([bst], dtype=torch.float32).pin_memory())
            step(b, lens, accumulate=j > 0, step_optimizer=j == len(boosts) - 1)
        torch.cuda.synchronize()

    window([1.0, 1.0, 1.0])
    assert (sc.loss_scale(), sc.unskipped(), opt._applied_steps(), opt.skipped_steps()) == (2.**10, 1, 1, 0)
    assert step.captures == 3
    p1 = _params(mod)
    window([1.0, 2.**30, 1.0])
    assert int(opt.found_inf.item()) == 1
    assert (sc.loss_scale(), sc.unskipped(), opt._applied_steps(), opt.skipped_steps()) == (2.**9, 0, 1, 1)
    assert all(torch.equal(p, p1[n]) for n, p in _params(mod).items())
    window([1.0, 1.0, 1.0])
    assert (sc.loss_scale(), sc.unskipped(), opt._applied_steps(), opt.skipped_steps()) == (2.**9, 1, 2, 1)
    assert step.captures == 3


# ------------------------------------------------------------------------------ resume
def test_resume_from_state_dict_is_bit_identical():
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    gen = torch.Generator().manual_seed(21)
    shapes = [(130, 8), (33,), (4100,)]
    p0 = [(torch.randn(s, generator=gen) * 0.05).half() for s in shapes]
    n_steps, cut = 12, 5
    draws = [[torch.randn(s, generator=gen) * 0.01 for s in shapes] for _ in range(n_steps)]
    bad_steps = {2, 7}

    def make(weights):
        params = [torch.nn.Parameter(w.clone().cuda()) for w in weights]
        opt = FusedAdamW([{"params": params[:2], "weight_decay": 0.01},
                          {"params": params[2:], "weight_decay": 0.0}], lr=1e-3)
        return params, opt, DynamicLossScaler(init_scale=2.**12, scale_window=2)

    def run(params, opt, sc, steps):
        out = []
        for t in steps:
            scale = sc.loss_scale()
            for p, g in zip(params, draws[t]):
                p.grad = (g * scale).half().cuda()
            if t in bad_steps:
                params[1].grad[4] = INF
            opt.step(grad_scale=sc)
            out.append(([p.detach().clone() for p in params],
                        [opt.state[id(p)]["master"].clone() for p in params],
                        sc.loss_scale(), sc.unskipped()))
        return out

    params, opt, sc = make(p0)
    full = run(params, opt, sc, range(n_steps))

    params, opt, sc = make(p0)
    run(params, opt, sc, range(cut))
    sd_opt, sd_sc = opt.state_dict(), sc.state_dict()
    params, opt, sc = make([p.detach().cpu() for p in params])
    opt.load_state_dict(sd_opt)
    sc.load_state_dict(sd_sc)
    resumed = run(params, opt, sc, range(cut, n_steps))

    for t, (a, b) in enumerate(zip(full[cut:], resumed), start=cut):
        assert a[2:] == b[2:], t
        assert all(torch.equal(x, y) for x, y in zip(a[0], b[0])), t
        assert all(torch.equal(x, y) for x, y in zip(a[1], b[1])), t
    assert len({s for _, _, s, _ in full}) >= 3
