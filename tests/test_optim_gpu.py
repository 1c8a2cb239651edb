"""GPU: fused multi-tensor AdamW (ub200_grad_sumsq + ub200_adamw_step) against the reference
optimizer's own trajectory (tests/golden/adamw.npz, produced by the reference's optim/adamw.py +
clip_grad_norm_) and, for 16-bit models with fp32 master weights, against the CPU oracle."""
import numpy as np
import pytest
import torch

from oracle import encoder_oracle as orc
from tests import util

pytestmark = pytest.mark.gpu


def test_fused_adamw_reproduces_reference_trajectory_fp32():
    from uniter_b200.optim import FusedAdamW
    g = util.load_golden("adamw")
    n = int(g["n_params"])
    params = [torch.nn.Parameter(torch.from_numpy(g["p0_%d" % i]).cuda()) for i in range(n)]
    opt = FusedAdamW([{"params": [params[0], params[2]], "weight_decay": 0.01},
                      {"params": [params[1], params[3]], "weight_decay": 0.0}],
                     lr=3e-4, betas=(float(g["betas"][0]), float(g["betas"][1])))
    for t, lr in enumerate(g["lrs"]):
        for grp in opt.param_groups:                      # the loop of train_vqa.py:207-214
            grp["lr"] = float(lr)
        for i, p in enumerate(params):
            p.grad = torch.from_numpy(g["g%d_%d" % (t, i)]).cuda()
        opt.step(max_grad_norm=float(g["max_norm"]))
        total = opt.last_sumsq.sqrt().item()
        assert abs(total - float(g["norm%d" % t])) <= 1e-4 * float(g["norm%d" % t])
        for i, p in enumerate(params):
            np.testing.assert_allclose(p.detach().cpu().numpy(), g["p%d_%d" % (t + 1, i)],
                                       atol=2e-7, rtol=2e-6)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_fused_adamw_master_weights_16bit_model(dtype):
    """apex-O2 semantics in one kernel: 16-bit gradients carrying a loss scale, fp32 masters,
    model weights = round(master) after every step, global-norm clipping on the unscaled grads."""
    from uniter_b200.optim import FusedAdamW
    gen = torch.Generator().manual_seed(3)
    shapes = [(300, 64), (64,), (4097,), (2, 3, 8)]
    wd = [0.01, 0.0, 0.01, 0.0]
    p0 = [(torch.randn(s, generator=gen) * 0.05).to(dtype) for s in shapes]
    params = [torch.nn.Parameter(x.clone().cuda()) for x in p0]
    opt = FusedAdamW([{"params": [params[0], params[2]], "weight_decay": 0.01},
                      {"params": [params[1], params[3]], "weight_decay": 0.0}], lr=1e-3)
    scale, max_norm = 128.0, 1.0
    P = [x.float() for x in p0]
    M = [torch.zeros_like(x) for x in P]
    V = [torch.zeros_like(x) for x in P]
    for t in range(3):
        grads16 = [(torch.randn(s, generator=gen) * (0.3 if t == 1 else 0.01) * scale).to(dtype) for s in shapes]
        for p, gr in zip(params, grads16):
            p.grad = gr.cuda()
        opt.step(grad_scale=scale, max_grad_norm=max_norm)
        un = [gr.float() / scale for gr in grads16]
        un, total = orc.clip_grad_norm(un, max_norm)
        for i in range(len(P)):
            P[i], M[i], V[i] = orc.adamw_step(P[i], un[i], M[i], V[i], t + 1, 1e-3, weight_decay=wd[i])
            master = opt.state[id(params[i])]["master"].cpu()
            np.testing.assert_allclose(master.numpy(), P[i].numpy(), atol=1e-6, rtol=1e-5)
            assert torch.equal(params[i].detach().cpu(), master.to(dtype))     # exact 16-bit refresh
    sd = opt.state_dict()
    opt2 = FusedAdamW([{"params": [params[0], params[2]], "weight_decay": 0.01},
                       {"params": [params[1], params[3]], "weight_decay": 0.0}], lr=1e-3)
    opt2.load_state_dict(sd)
    assert opt2.state_dict()["state"][1]["step"] == 3          # params[2] = second tensor of group 0
    assert torch.equal(opt2.state[id(params[2])]["exp_avg"], opt.state[id(params[2])]["exp_avg"])


def test_fused_adamw_steps_the_model_from_its_gradient_arena():
    """End to end: backward fills the flat gradient arena, the optimizer reads the gradients in
    place (arena views) and the loss goes down."""
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.optim import build_optimizer
    from uniter_b200.synth import synth_batch
    import types
    torch.manual_seed(0)
    mod = UniterForMLM(util.tiny_config(), 64).to("cuda", torch.bfloat16).train()
    opts = types.SimpleNamespace(weight_decay=0.01, learning_rate=2e-3, betas=[0.9, 0.98], optim="adamw")
    opt = build_optimizer(mod, opts)
    batch = util.batch_to(synth_batch(8, 6, 14, 3, 9, seed=2, img_dim=64, vocab_size=2000, mlm_prob=0.3), "cuda")
    losses = []
    for it in range(8):
        opt.zero_grad()
        loss = mod(batch).mean()
        loss.backward()
        q = mod.uniter.encoder.layer[0].attention.self.query.weight
        assert q.grad.data_ptr() == mod.uniter._ensure_arena()[0].view(q).data_ptr()
        opt.step(max_grad_norm=2.0)
        losses.append(loss.item())
    assert all(l == l for l in losses)
    assert losses[-1] < losses[0] - 0.1, losses


def test_fused_adamw_skips_overflowed_steps_on_the_device():
    """fp16 + loss scaling: an inf / NaN gradient must not poison masters or moments (g * 0 = NaN);
    like apex's dynamic scaler the step is skipped — decided on the device, no host sync — the step
    count does not advance (bias correction of the next real step is that of step 1) and
    `found_inf` is raised for the caller to lower its loss scale."""
    from uniter_b200.optim import FusedAdamW
    gen = torch.Generator().manual_seed(5)
    shapes = [(130, 8), (33,)]
    p0 = [(torch.randn(s, generator=gen) * 0.05).half() for s in shapes]
    params = [torch.nn.Parameter(x.clone().cuda()) for x in p0]
    grads = [torch.nn.Parameter(torch.zeros_like(p)) for p in params]      # static gradient buffers
    for p, g in zip(params, grads):
        p.grad = g.data
    opt = FusedAdamW(params, lr=1e-3, weight_decay=0.01)
    for bad in (float("inf"), float("nan")):
        for p in params:
            p.grad.copy_((torch.randn(p.shape, generator=gen) * 0.01).half())
        params[0].grad[3, 2] = bad
        opt.step(grad_scale=64.0, max_grad_norm=1.0)
        assert int(opt.found_inf.item()) == 1
        for p, x in zip(params, p0):
            assert torch.equal(p.detach().cpu(), x)
            st = opt.state[id(p)]
            assert torch.equal(st["master"].cpu(), x.float())
            assert (st["exp_avg"] == 0).all() and (st["exp_avg_sq"] == 0).all()
    assert opt.skipped_steps() == 2 and opt._applied_steps() == 0
    gs = [(torch.randn(p.shape, generator=gen) * 0.01 * 64.0).half() for p in params]
    for p, g in zip(params, gs):
        p.grad.copy_(g)
    opt.step(grad_scale=64.0, max_grad_norm=-1.0)
    assert int(opt.found_inf.item()) == 0 and opt._applied_steps() == 1
    for i, (p, x) in enumerate(zip(params, p0)):
        want, _, _ = orc.adamw_step(x.float(), gs[i].float() / 64.0, torch.zeros(x.shape), torch.zeros(x.shape),
                                    1, 1e-3, weight_decay=0.01)
        np.testing.assert_allclose(opt.state[id(p)]["master"].cpu().numpy(), want.numpy(), atol=1e-6, rtol=1e-5)
