"""GPU: whole training steps are bit-reproducible under torch.use_deterministic_algorithms(True).

Every comparison is torch.equal over the loss, the whole gradient arena, the weights, the optimizer's
masters, moments and device counters, and the loss scaler's table, after several steps from one saved
initial state.  Runs differ in the SM reserve (0, 6, 38: the SM-sized grids change), repeat at the same
reserve, and, eagerly, pad the batch with the dummy sequence of GraphedStep.  torch's flag also NaN-fills
every torch.empty (fill_uninitialized_memory), so a kernel that read scratch it never wrote would show.
Tests that reach cuBLAS run in a subprocess that sets CUBLAS_WORKSPACE_CONFIG before CUDA starts.
"""
import gc
import os
import subprocess
import sys

import pytest
import torch

from tests import util

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESERVES = (0, 6, 38)


@pytest.fixture(autouse=True)
def torch_flags():
    """Saves and restores torch's determinism flags, the fill of uninitialised memory and the SM reserve."""
    import torch.utils.deterministic as tud
    from uniter_b200 import _lib
    saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
             tud.fill_uninitialized_memory)
    yield
    torch.use_deterministic_algorithms(saved[0], warn_only=saved[1])
    tud.fill_uninitialized_memory = saved[2]
    _lib.load().ub200_set_sm_reserve(0)


def _set_reserve(n):
    from uniter_b200 import _lib
    _lib.load().ub200_set_sm_reserve(n)


def _round_up(v, m):
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------ models and batches
def _config(layers):
    from uniter_b200.model import UniterConfig
    c = util.BASE_L1
    return UniterConfig(c["vocab_size"], hidden_size=c["hidden_size"], num_hidden_layers=layers,
                        num_attention_heads=c["num_attention_heads"], intermediate_size=c["intermediate_size"],
                        max_position_embeddings=c["max_position_embeddings"], type_vocab_size=c["type_vocab_size"])


def _prepare(mod, dtype, p_drop):
    torch.manual_seed(0)
    mod = mod.to("cuda", dtype).train()
    for m in mod.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = p_drop
    init = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    return mod, init


def _c2_host(seed=1234, mrm=False):
    """The C2 batch (B = 64, text 12-28, regions 26-46) with fixed-size masked-token lists."""
    from uniter_b200.synth import pad_mlm_index, synth_batch, synth_mrm
    b = pad_mlm_index(synth_batch(64, 12, 28, 26, 46, seed, mlm_prob=0.15), 64)
    if mrm:
        b = synth_mrm(b, 0.15, 1601, seed=seed + 1, pad_multiple=64)
        b["targets"] = torch.randint(0, 2, (64,), generator=torch.Generator().manual_seed(seed + 2))
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    return {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens


def _device_batch(host, lens, pad=False):
    """Device copy with its packing bookkeeping; pad=True adds the dummy sequence GraphedStep uses."""
    from uniter_b200 import model as M
    b = {k: v.cuda() for k, v in host.items()}
    mask = b["attn_masks"]
    if pad:
        B, L = mask.shape
        T = sum(lens)
        T_pad = _round_up(T + 1, 128)
        buf, offs, _ = M._prefix_pack_host(lens, L, T_pad)
        M._meta_store(mask, M._meta_from_buffer(buf.cuda(), offs, B, L, T_pad, 128, None, True))
    else:
        M.register_lengths(mask, lens, prefix=True)
    return b


def _mlm_loss(mod):
    return lambda b: (mod(b).sum() * b["mlm_inv_n"]).squeeze()


def _task_loss(mod):
    def loss(b, task):
        out = mod(b, task)
        if task == "mlm":
            return (out.sum() * b["mlm_inv_n"]).squeeze()
        if task == "itm":
            return out[0].sum() / out[0].numel()
        v = b["mrm_valid"]
        l = out.float()
        if l.dim() == 2:
            l = l.sum(1) / (l.size(1) if task == "mrfr" else 1)
        return ((l * v).sum() * b["mrm_inv_n"]).squeeze()
    return loss


# ------------------------------------------------------------------------------ runs and snapshots
def _snapshot(losses, mod, opt, arena, scaler=None):
    out = {"loss": torch.stack([l.reshape(()) for l in losses]), "arena": arena.flat.clone()}
    for n, p in mod.named_parameters():
        out["weight " + n] = p.detach().clone()
    for i, st in enumerate(opt.state.values()):
        for k, v in sorted(st.items()):
            if torch.is_tensor(v):
                out["opt %d %s" % (i, k)] = v.clone()
    out["opt counters"] = opt._dev_state.clone()
    if scaler is not None:
        out["scaler"] = scaler.table.clone()
    torch.cuda.synchronize()
    return out


def _assert_identical(runs, names):
    ref = runs[0]
    assert torch.isfinite(ref["loss"]).all() and torch.isfinite(ref["arena"].float()).all()
    for r, name in zip(runs[1:], names[1:]):
        assert r.keys() == ref.keys()
        bad = [k for k in ref if not torch.equal(ref[k], r[k])]
        assert not bad, "%s differs from %s in %d tensors: %s (losses %s, %s)" % (
            name, names[0], len(bad), bad[:8], ref["loss"].tolist(), r["loss"].tolist())


def _eager_run(mod, init, loss_fn, batches, reserve=0, pad=False, scaler=None, **step_kw):
    """len(batches) eager steps (forward, backward, FusedAdamW with clipping) from `init`."""
    from uniter_b200 import model as M
    from uniter_b200.arena import GradArena
    from uniter_b200.optim import FusedAdamW
    _set_reserve(reserve)
    mod.load_state_dict(init)
    M._rng_offset[0] = 0                   # the same dropout masks in every run
    arena = GradArena.attach(mod)
    opt = FusedAdamW(mod.parameters(), lr=1e-4, weight_decay=0.01)
    losses = []
    for item in batches:
        (host, lens), tag = item if isinstance(item[0], tuple) else (item, None)
        b = _device_batch(host, lens, pad)
        arena.begin_step()
        loss = loss_fn(b) if tag is None else loss_fn(b, tag)
        (scaler.scale(loss) if scaler is not None else loss).backward()
        arena.finish_step()
        arena.end_step_mode()
        opt.step(max_grad_norm=1.0, **(dict(grad_scale=scaler) if scaler is not None else {}), **step_kw)
        losses.append(loss.detach().clone())
    out = _snapshot(losses, mod, opt, arena, scaler)
    _set_reserve(0)
    return out


def _graphed_run(mod, init, loss_fn, calls, reserve=0, scaler=None, **kw):
    """GraphedStep over `calls` [(host, lens, call kwargs)], FusedAdamW with clipping in the graph."""
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.optim import FusedAdamW
    _set_reserve(reserve)
    mod.load_state_dict(init)
    opt = FusedAdamW(mod.parameters(), lr=1e-4, weight_decay=0.01)
    step = GraphedStep(mod, loss_fn, optimizer=opt, optimizer_kwargs={"max_grad_norm": 1.0},
                       loss_scaler=scaler, **kw)
    losses = [step(host, lens, **ckw).clone() for host, lens, ckw in calls]
    out = _snapshot(losses, mod, opt, step.arena, scaler)
    out_captures = step.captures
    del step
    gc.collect()
    _set_reserve(0)
    return out, out_captures


# ------------------------------------------------------------------------------ eager C2 MLM step
def test_eager_c2_mlm_step_is_bit_reproducible_across_reserves_runs_and_padding():
    """UNITER-base (12 layers), bf16, dropout 0.1, FusedAdamW with clipping, three steps."""
    from uniter_b200 import _lib
    from uniter_b200.heads import UniterForMLM
    torch.manual_seed(0)
    mod, init = _prepare(UniterForMLM(_config(12), 2048), torch.bfloat16, 0.1)
    batches = [_c2_host(1234), _c2_host(1235), _c2_host(1236)]
    loss_fn = _mlm_loss(mod)

    torch.use_deterministic_algorithms(True)
    runs = [_eager_run(mod, init, loss_fn, batches, reserve=r) for r in RESERVES]
    runs.append(_eager_run(mod, init, loss_fn, batches, reserve=0))
    runs.append(_eager_run(mod, init, loss_fn, batches, reserve=0, pad=True))
    assert _lib.load().ub200_deterministic() == 0           # restored after every call
    _assert_identical(runs, ["reserve %d" % r for r in RESERVES] + ["repeat", "padded"])

    # without torch's flag the same check fails: the default mode's gradient bits follow the grid
    torch.use_deterministic_algorithms(False)
    default = [_eager_run(mod, init, loss_fn, batches[:1], reserve=r) for r in RESERVES]
    assert len({d["arena"].float().cpu().numpy().tobytes() for d in default}) >= 2
    # and the two modes compute the same step up to summation order
    assert torch.allclose(default[0]["loss"][0], runs[0]["loss"][0], rtol=1e-2)


# ------------------------------------------------------------------------------ every task and head
def test_every_pretraining_task_is_bit_reproducible():
    """mlm, mrfr, mrc, mrc-kl and itm in turn, on one UNITER-base layer at the C2 batch."""
    from uniter_b200.heads import UniterForPretraining
    torch.manual_seed(0)
    mod, init = _prepare(UniterForPretraining(_config(1), 2048, 1601), torch.bfloat16, 0.1)
    hb = _c2_host(1234, mrm=True)
    tasks = [(hb, t) for t in ("mlm", "mrfr", "mrc", "mrc-kl", "itm")]
    loss_fn = _task_loss(mod)
    torch.use_deterministic_algorithms(True)
    runs = [_eager_run(mod, init, loss_fn, tasks, reserve=r) for r in (0, 0, 38)]
    _assert_identical(runs, ["reserve 0", "repeat", "reserve 38"])


def _malformed_itm_batch(n=24, nbb=36, seed=5):
    """One image and n texts, gather_index built like data/itm.py:356-361: get_gather_index(...) gets the
    LAST text's length where the longest belongs, so image positions of longer texts repeat text rows."""
    from uniter_b200.synth import get_gather_index, synth_batch
    g = torch.Generator().manual_seed(seed)
    tl = torch.randint(12, 29, (n,), generator=g).tolist()
    tl[-1] = 13
    b = synth_batch(n, 0, 0, 0, 0, seed=seed, txt_lens=tl, num_bbs=[nbb] * n)
    b["img_feat"], b["img_pos_feat"] = b["img_feat"][:1].contiguous(), b["img_pos_feat"][:1].contiguous()
    L = b["attn_masks"].size(1)
    b["gather_index"] = get_gather_index(tl, [nbb] * n, n, tl[-1], L)
    assert not torch.equal(b["gather_index"], get_gather_index(tl, [nbb] * n, n, max(tl), L))
    return b


def test_itm_hard_negative_step_with_the_malformed_gather_index_is_bit_reproducible():
    from uniter_b200.heads import UniterForImageTextRetrievalHardNeg
    torch.manual_seed(0)
    # init_output() makes rank_output a view of row 1 of itm_output, as retrieval fine-tuning does: the
    # optimizer must update each shared element once (FusedAdamW gives it to rank_output)
    mod, init = _prepare(UniterForImageTextRetrievalHardNeg(_config(1), 2048, hard_size=7),
                         torch.bfloat16, 0.1)
    mod.init_output()
    init = {k: v.detach().clone() for k, v in mod.state_dict().items()}
    host = _malformed_itm_batch()
    lens = [a + c for a, c in zip(host["txt_lens"], host["num_bbs"])]

    def loss_fn(b):
        b = dict(b, txt_lens=host["txt_lens"], num_bbs=host["num_bbs"])
        return mod(b, sample_from="i").mean()
    tensors = {k: v for k, v in host.items() if torch.is_tensor(v)}
    torch.use_deterministic_algorithms(True)
    runs = [_eager_run(mod, init, loss_fn, [(tensors, lens)] * 2, reserve=r) for r in (0, 0, 38)]
    _assert_identical(runs, ["reserve 0", "repeat", "reserve 38"])
    # the ranking loss moved the shared row, itm_output's other row only decayed (its gradient is zero)
    row0 = init["itm_output.weight"][0].float()
    assert mod.rank_output.weight.data_ptr() == mod.itm_output.weight[1].data_ptr()
    assert not torch.equal(mod.rank_output.weight, init["rank_output.weight"].to(mod.rank_output.weight.dtype))
    assert torch.allclose(mod.itm_output.weight[0].float(), row0, rtol=1e-2, atol=1e-6)


def test_gather_rows_scatter_add_backward_is_deterministic_under_the_flag():
    """_GatherRows with an arbitrary index (the reference-layout embedding path) scatter-adds its
    gradient with torch's index_add_, which takes its deterministic form under torch's flag."""
    from uniter_b200.model import _GatherRows
    b = _malformed_itm_batch(n=64, nbb=46)
    B, L = b["attn_masks"].shape
    Lc = b["input_ids"].size(1) + 46
    flat = (b["gather_index"] + torch.arange(B).unsqueeze(1) * Lc).reshape(-1).to(torch.int32).cuda()
    g = torch.Generator(device="cuda").manual_seed(3)
    src = torch.randn(B * Lc, 768, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(flat.numel(), 768, device="cuda", generator=g)
    assert flat.unique().numel() < flat.numel()                     # rows gathered more than once

    def grad():
        s = src.clone().requires_grad_(True)
        (_GatherRows.apply(s, flat, B * Lc, None).float() * w).sum().backward()
        return s.grad.clone()
    def kernels():
        from torch.autograd import DeviceType
        from torch.profiler import ProfilerActivity, profile
        grad()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            grad()
            torch.cuda.synchronize()
        return {e.name for e in prof.events() if e.device_type == DeviceType.CUDA}
    torch.use_deterministic_algorithms(False)
    default_kernels = kernels()
    torch.use_deterministic_algorithms(True)
    det_kernels = kernels()
    # the flag selected another implementation of the scatter-add: kernels the default never launches
    assert det_kernels - default_kernels, (sorted(default_kernels), sorted(det_kernels))
    grads = [grad() for _ in range(3)]
    assert all(torch.equal(grads[0], x) for x in grads[1:])
    # a row gathered thousands of times, with terms from 1e-4 to 1e4: a bf16 sum whose bits follow the order
    hot = torch.cat([torch.zeros(4096, dtype=torch.int32, device="cuda"), flat])
    mag_w = torch.pow(10.0, torch.rand(hot.numel(), 768, device="cuda", generator=g) * 8 - 4)
    w_hot = mag_w * torch.where(torch.rand(hot.numel(), 768, device="cuda", generator=g) < 0.5, -1.0, 1.0)

    def grad_hot():
        s = src.clone().requires_grad_(True)
        (_GatherRows.apply(s, hot, B * Lc, None).float() * w_hot).sum().backward()
        return s.grad.clone()
    hots = [grad_hot() for _ in range(5)]
    assert all(torch.equal(hots[0], x) for x in hots[1:])
    w16 = w.to(torch.bfloat16).double()
    ref = torch.zeros(B * Lc, 768, dtype=torch.float64, device="cuda").index_add_(0, flat.long(), w16)
    mag = torch.zeros_like(ref).index_add_(0, flat.long(), w16.abs())
    assert ((grads[0].double() - ref).abs() <= 2 ** -7 * mag + 1e-6).all()


_VQA_CHILD = r"""
import torch
from tests import test_reproducible_step_gpu as t
from uniter_b200.heads import UniterForVisualQuestionAnswering
torch.manual_seed(0)
mod, init = t._prepare(UniterForVisualQuestionAnswering(t._config(1), 2048, 3129), torch.bfloat16, 0.1)
host, lens = t._c2_host(1234)
host = dict(host, targets=(torch.rand(64, 3129, generator=torch.Generator().manual_seed(4)) < 0.002)
            .to(torch.bfloat16).pin_memory())
loss_fn = lambda b: mod(b).float().sum() / 64
torch.use_deterministic_algorithms(True)
runs = [t._eager_run(mod, init, loss_fn, [(host, lens)] * 2, reserve=r) for r in (0, 0, 38)]
t._assert_identical(runs, ["reserve 0", "repeat", "reserve 38"])
print("vqa reproducible")
"""


def test_vqa_head_step_is_bit_reproducible_with_the_cublas_workspace_config():
    """The VQA MLP is torch (cuBLAS): under torch's flag it needs CUBLAS_WORKSPACE_CONFIG, set before
    CUDA starts, so this runs in a fresh interpreter."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _VQA_CHILD]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "vqa reproducible" in r.stdout, r.stdout[-3000:] + r.stderr[-6000:]


# ------------------------------------------------------------------------------ fp16 accumulation window
def test_fp16_accumulation_window_with_the_loss_scaler_is_bit_reproducible():
    """Three micro-batches per optimizer step (step_optimizer=False before the last), with one window
    whose middle micro-batch overflows: the scale trajectory, skips and weights repeat bit for bit."""
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.optim import DynamicLossScaler
    torch.manual_seed(0)
    mod, init = _prepare(UniterForMLM(_config(1), 2048), torch.float16, 0.1)
    hb0, lens = _c2_host(1234)
    loss_fn = lambda b: (mod(b).sum() * b["mlm_inv_n"] * b["boost"]).squeeze()    # noqa: E731
    calls = []
    for boosts in ([1.0, 1.0, 1.0], [1.0, 2.**30, 1.0], [1.0, 1.0, 1.0]):
        for j, bst in enumerate(boosts):
            hb = dict(hb0, boost=torch.tensor([bst], dtype=torch.float32).pin_memory())
            calls.append((hb, lens, dict(accumulate=j > 0, step_optimizer=j == 2)))
    torch.use_deterministic_algorithms(True)
    runs, scales = [], []
    for r in (0, 0, 38):
        sc = DynamicLossScaler(init_scale=2.**12, scale_window=2)
        snap, captures = _graphed_run(mod, init, loss_fn, calls, reserve=r, scaler=sc)
        assert captures == 3
        runs.append(snap)
        scales.append((sc.loss_scale(), sc.unskipped()))
    assert scales[0][0] <= 2.**11 and scales.count(scales[0]) == 3     # the overflowed window halved the scale
    _assert_identical(runs, ["reserve 0", "repeat", "reserve 38"])


# ------------------------------------------------------------------------------ GraphedStep
def test_graphed_replays_equal_eager_steps_and_follow_the_flag():
    from uniter_b200 import _lib
    from uniter_b200.heads import UniterForMLM
    torch.manual_seed(0)
    # dropout off: an eager step and a replay number their dropout streams differently
    mod, init = _prepare(UniterForMLM(_config(2), 2048), torch.bfloat16, 0.0)
    hbs = [_c2_host(1234 + i) for i in range(3)]
    loss_fn = _mlm_loss(mod)
    torch.use_deterministic_algorithms(True)
    eager = [_eager_run(mod, init, loss_fn, hbs, reserve=r) for r in (0, 6)]
    graphed = [_graphed_run(mod, init, loss_fn, [(h, l, {}) for h, l in hbs], reserve=r)[0] for r in (0, 38)]
    _assert_identical(eager + graphed, ["eager reserve 0", "eager reserve 6", "graphed reserve 0",
                                        "graphed reserve 38"])

    # flipping torch's flag captures a new graph; flipping it back replays the first one again
    from uniter_b200.graphed import GraphedStep
    mod.load_state_dict(init)
    step = GraphedStep(mod, loss_fn)
    hb, lens = hbs[0]
    step(hb, lens)
    step(hb, lens)
    assert step.captures == 1
    on = step.stage(hb, lens)
    torch.use_deterministic_algorithms(False)
    off = step.stage(hb, lens)
    step.replay(off)
    assert step.captures == 2 and off is not on and (on.mode, off.mode) == (1, None)
    assert on.launches > off.launches            # the fixed-order forms launch more kernels
    torch.use_deterministic_algorithms(True)
    assert step.stage(hb, lens) is on
    torch.cuda.synchronize()
    assert step.captures == 2 and _lib.load().ub200_deterministic() == 0


def _long_host():
    """A batch with one sequence longer than 128 tokens (attention backward without a fixed-order form)."""
    from uniter_b200.synth import pad_mlm_index, synth_batch
    b = pad_mlm_index(synth_batch(4, 0, 0, 0, 0, seed=9, txt_lens=[30, 12, 20, 16], num_bbs=[110, 26, 30, 40],
                                  mlm_prob=0.15), 64)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    assert max(lens) > 128
    return {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens


def test_long_batches_raise_under_the_flag_and_run_with_warn_only():
    from uniter_b200 import _lib
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForMLM
    torch.manual_seed(0)
    mod, init = _prepare(UniterForMLM(_config(1), 2048), torch.bfloat16, 0.1)
    hb, lens = _long_host()
    loss_fn = _mlm_loss(mod)
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match=r"max_seqlen 140 > 128"):
        _eager_run(mod, init, loss_fn, [(hb, lens)])
    step = GraphedStep(mod, loss_fn)
    with pytest.raises(RuntimeError, match=r"max_seqlen 256 > 128"):
        step(hb, lens)
    assert step.captures == 0 and _lib.load().ub200_deterministic() == 0

    torch.use_deterministic_algorithms(True, warn_only=True)
    with pytest.warns(UserWarning, match=r"max_seqlen 140 > 128"):
        snap = _eager_run(mod, init, loss_fn, [(hb, lens)])
    assert torch.isfinite(snap["loss"]).all() and torch.isfinite(snap["arena"].float()).all()
    with pytest.warns(UserWarning, match=r"max_seqlen 256 > 128"):
        loss = step(hb, lens)
    torch.cuda.synchronize()
    assert torch.isfinite(loss) and step.captures == 1
    assert next(iter(step.buckets.values())).mode == 1     # only the encoder node runs in the default mode
    assert _lib.load().ub200_deterministic() == 0


def test_without_the_flag_the_library_switch_stays_off(monkeypatch):
    from uniter_b200 import _lib
    from uniter_b200.heads import UniterForMLM
    lib = _lib.load()
    calls = []
    real = lib.ub200_set_deterministic
    monkeypatch.setattr(lib, "ub200_set_deterministic", lambda v: calls.append(v) or real(v))
    torch.manual_seed(0)
    mod, init = _prepare(UniterForMLM(_config(1), 2048), torch.bfloat16, 0.1)
    torch.use_deterministic_algorithms(False)
    hb = _c2_host(1234)
    _eager_run(mod, init, _mlm_loss(mod), [hb])
    _graphed_run(mod, init, _mlm_loss(mod), [(hb[0], hb[1], {})])
    assert lib.ub200_deterministic() == 0 and calls == []
