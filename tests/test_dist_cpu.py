"""CPU, world_size = 2, gloo: the data-parallel exchange step (SURVEY.md §8e).

The only collective on the path is the mean-allreduce of gradients once per optimizer step
(utils/distributed.py:16-43, Horovod average) plus the start-up parameter broadcast (:100-148).
Correctness criterion from the reference's own "emulation" equivalence (README.md:115): the
N-rank result equals the mean of the per-rank gradients == oracle.allreduce_mean.
"""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from uniter_b200.heads import UniterForMLM
        from uniter_b200.model import UniterConfig
        from uniter_b200 import distributed as ubd
        torch.manual_seed(100 + rank)                       # deliberately different init per rank
        cfg = UniterConfig(500, hidden_size=64, num_hidden_layers=2, num_attention_heads=1,
                           intermediate_size=128, max_position_embeddings=32)
        model = UniterForMLM(cfg, 16)
        ubd.broadcast_parameters(model, root=0)
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        # fake per-rank gradients: encoder-layer grads live in the arena (as after a real backward),
        # everything else gets ordinary .grad tensors (as autograd would assign them)
        from uniter_b200.arena import GradArena
        arena = GradArena.attach(model)
        g = torch.Generator().manual_seed(7 + rank)
        arena.flat.copy_(torch.randn(arena.flat.shape, generator=g))
        enc = model.uniter
        layer_ids = set(id(p) for p in enc.encoder.parameters())
        for p in model.parameters():
            if id(p) in layer_ids:
                p.grad = arena.view(p)
            else:
                p.grad = torch.randn(p.shape, generator=g)
        local = {n: p.grad.clone() for n, p in model.named_parameters()}
        ubd.GradientReducer(model).reduce()
        reduced = {n: p.grad.clone() for n, p in model.named_parameters()}
        out[rank] = (sd, local, reduced)
    finally:
        dist.destroy_process_group()


def test_broadcast_and_gradient_mean_two_ranks():
    from oracle import encoder_oracle as orc
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    sd0, loc0, red0 = out[0]
    sd1, loc1, red1 = out[1]
    # D2: every rank starts from rank 0's parameters
    for k in sd0:
        assert torch.equal(sd0[k], sd1[k]), k
    # D1: every rank ends with the mean of the per-rank gradients (oracle semantics)
    for n in loc0:
        want = orc.allreduce_mean([loc0[n], loc1[n]])[0]
        assert torch.allclose(red0[n], want, atol=1e-6), n
        assert torch.equal(red0[n], red1[n]), n
    # every gradient ended up inside ONE flat arena and was reduced there in place (no copy-in/out)
    assert "uniter.encoder.layer.0.attention.self.query.weight" in loc0


def test_chunk_shipping_covers_the_arena_exactly_once_and_survives_unreduced_warmups():
    """Host logic of the overlapped exchange (single process, no collective is issued: the reducer
    reports the ranges it would ship through its capture callback).  The slices shipped while the
    backward runs ([head | pooler] + top layer group, then the other groups) plus what reduce() ships
    afterwards (the front-end) must tile the arena exactly once.  GraphedStep warms a step up WITHOUT the
    reducer (a capture must not communicate): the per-step counters reduce() normally clears are then
    stale and nothing may be shipped early until reset_step_state() — the regression that silently
    removed all overlap."""
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.model import UniterConfig
    from uniter_b200 import distributed as ubd
    cfg = UniterConfig(500, hidden_size=64, num_hidden_layers=4, num_attention_heads=1,
                       intermediate_size=128, max_position_embeddings=32)
    model = UniterForMLM(cfg, 16)
    red = ubd.GradientReducer(model, overlap_chunks=2)
    enc = red.encoders[0]
    shipped = []
    red._split_cb = lambda ranges, final=False: shipped.append((list(ranges), final))

    def backward_hooks():
        for lo, hi in ((2, 4), (0, 2)):                    # top chunk first, as _EncoderStack.backward does
            red._on_chunk(enc, lo, hi)

    enc._fwd_since_reduce = 3                               # two warm-up forwards + the captured one, no reduce()
    backward_hooks()
    assert shipped == []                                    # stale counters: everything waits for reduce()
    red.reset_step_state()
    enc._fwd_since_reduce = 1                               # the captured step's forward
    backward_hooks()
    assert len(shipped) == 2 and not any(f for _, f in shipped)
    red.reduce()
    assert shipped[-1][1] is True                           # the remainder, reported as final
    ranges = sorted(r for rs, _ in shipped for r in rs)
    pos = 0
    for lo, hi in ranges:
        assert lo == pos and hi > lo, (ranges, pos)
        pos = hi
    assert pos == red.arena.numel
    assert all(lo % 8 == 0 and hi % 8 == 0 for lo, hi in ranges)   # 16-byte slices (ub200_peer_allreduce)
    assert enc._fwd_since_reduce == 0
