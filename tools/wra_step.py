"""Time word-region alignment (WRA, the optimal-transport term of ITM pre-training) on one GPU, two
comparisons in one run, alternating their variants:

  wra    WRA alone, forward + backward over packed 16-bit rows: the fused kernels (ub200_wra_*) against
         the fp32 torch composition of model/ot.py's math with bool masks (gather into the padded text /
         image tensors, normalize, bmm, 50 IPOT iterations of small batched ops, the diagonal sum,
         autograd), at C4's length draws and at the pre-training configs' maxima (62 x 100);
  step   one ITM pre-training step of UniterForPretraining (UNITER-base geometry, forward + backward +
         FusedAdamW with clipping), eager and GraphedStep replay, without and with WRA (itm_ot_lambda 0.1).

B defaults to 64.  The text and region counts are ASSUMPTIONS, not dataset statistics: each pair draws
its text length and region count uniformly from --txt-len and --num-bb (seeded; the defaults are the
ranges of bench.py's C4 configuration).  Times are medians over --rounds rounds of --iters calls each,
from CUDA events around work that ends in a synchronise.  One JSON line per comparison, with the card
name and power limit, goes to stdout and (appended) to --out.

    python tools/wra_step.py --out /tmp/wra_step.jsonl
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from re_step import card, compare  # noqa: E402


def batch(args, seed, txt_len, num_bb):
    from uniter_b200.batching import itm_ot_collate
    g = torch.Generator().manual_seed(seed)
    samples = []
    for i in range(args.batch):
        tl = int(torch.randint(txt_len[0], txt_len[1] + 1, (1,), generator=g))
        nbb = int(torch.randint(num_bb[0], num_bb[1] + 1, (1,), generator=g))
        samples.append((torch.randint(1000, 28000, (tl,), generator=g), torch.randn(nbb, 2048, generator=g),
                        torch.rand(nbb, 7, generator=g), torch.ones(tl + nbb, dtype=torch.long),
                        torch.tensor([i % 2])))
    b = itm_ot_collate(samples)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    return b, lens


def wra_variants(args, txt_len, num_bb):
    import torch.nn.functional as F
    from uniter_b200.heads import _WraDist
    b, lens = batch(args, 2, txt_len, num_bb)
    B, M, N = args.batch, b["input_ids"].size(1), b["img_feat"].size(1)
    cu = b["cu_seqlens"].cuda()
    tl = b["ot_txt_lens"].cuda()
    T = int(sum(lens))
    g = torch.Generator(device="cuda").manual_seed(3)
    rows = torch.randn(T, 768, device="cuda", generator=g).to(args.dtype).requires_grad_(True)
    # the padded text / image slot of every pair (index T = a zero row), built once
    ti = torch.full((B, M), T, dtype=torch.long)
    ii = torch.full((B, N), T, dtype=torch.long)
    c = b["cu_seqlens"].tolist()
    for k, (m, n) in enumerate(zip(b["txt_lens"], b["num_bbs"])):
        ti[k, :m] = torch.arange(c[k], c[k] + m)
        ii[k, :n] = torch.arange(c[k] + m, c[k] + m + n)
    ti, ii = ti.cuda(), ii.cuda()
    txt_pad, img_pad = ti == T, ii == T
    joint = txt_pad[:, :, None] | img_pad[:, None, :]
    jt = joint.transpose(1, 2)
    t_len = (M - txt_pad.sum(1)).float()
    i_len = (N - img_pad.sum(1)).float()
    xm, ym = (txt_pad.float() * 1e4)[:, None], (img_pad.float() * 1e4)[:, None]
    gd = torch.ones(B, device="cuda", dtype=args.dtype)

    def torch_composition():
        src = torch.cat([rows, rows.new_zeros(1, 768)])
        txt, img = src[ti].float(), src[ii].float()
        cost = 1 - F.normalize(txt, dim=-1, eps=1e-5) @ F.normalize(img, dim=-1, eps=1e-5).transpose(1, 2)
        cost = cost.masked_fill(joint, 0)
        with torch.no_grad():
            C = cost.detach()
            sigma = (torch.ones(B, M, device="cuda") / t_len[:, None]).masked_fill(txt_pad, 0)
            Tp = torch.ones(B, N, M, device="cuda").masked_fill(jt, 0)
            A = torch.exp(-C.transpose(1, 2) / 0.5).masked_fill(jt, 0)
            for _ in range(50):
                Q = A * Tp
                delta = 1 / (i_len[:, None, None] * Q.matmul(sigma.view(B, M, 1)).view(B, 1, N) + ym)
                sigma = 1 / (t_len[:, None, None] * delta.matmul(Q) + xm)
                Tp = delta.view(B, N, 1) * Q * sigma
            Tp = Tp.masked_fill(jt, 0)
        dist = torch.diagonal(cost.matmul(Tp), dim1=1, dim2=2).sum(-1).to(args.dtype)
        dist.backward(gd)

    def fused():
        _WraDist.apply(rows, cu, tl, B, M, N).backward(gd)

    return {"torch": torch_composition, "fused": fused}, {"txt_len": txt_len, "num_bb": num_bb, "T": T,
                                                          "max_m": M, "max_n": N}


def step_variants(args, with_wra):
    from uniter_b200.arena import GradArena
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForPretraining
    from uniter_b200.model import UniterConfig, register_lengths
    from uniter_b200.optim import FusedAdamW
    cfg = UniterConfig(28996, hidden_size=768, num_hidden_layers=args.layers, num_attention_heads=12,
                       intermediate_size=3072, max_position_embeddings=512)
    torch.manual_seed(0)
    mod = UniterForPretraining(cfg, 2048, 1601).to("cuda", args.dtype).train()
    b, lens = batch(args, 1, args.txt_len, args.num_bb)
    host = {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}

    def loss_fn(d):
        itm_loss, ot = mod(dict(d, ot_inputs={} if with_wra else None), "itm")
        loss = itm_loss.mean()
        if with_wra:
            pos, neg = ot
            loss = loss + 0.1 * (pos.float().sum() - neg.float().sum()) / (pos.numel() + neg.numel())
        return loss

    opt_e = FusedAdamW(mod.parameters(), lr=1e-6, weight_decay=0.01)
    arena = GradArena.attach(mod)
    dev = {k: v.cuda() for k, v in host.items()}

    def eager():
        register_lengths(dev["attn_masks"], lens, prefix=True)
        arena.begin_step()
        loss_fn(dev).backward()
        arena.finish_step()
        arena.end_step_mode()
        opt_e.step(max_grad_norm=2.0)

    opt_g = FusedAdamW(mod.parameters(), lr=1e-6, weight_decay=0.01)
    step = GraphedStep(mod, loss_fn, optimizer=opt_g, optimizer_kwargs={"max_grad_norm": 2.0})
    return {"eager": eager, "graphed": lambda: step(host, lens)}, {"T": sum(lens), "wra": with_wra}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--txt-len", type=int, nargs=2, default=[12, 28], metavar=("MIN", "MAX"),
                    help="text length range, [CLS] and [SEP] included (assumption)")
    ap.add_argument("--num-bb", type=int, nargs=2, default=[26, 46], metavar=("MIN", "MAX"),
                    help="regions per image (assumption)")
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=["step", "wra"], default=None)
    ap.add_argument("--out", default=None, help="JSONL file to append to")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wra_step.py measures on the GPU; no CUDA device here")
    args.dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    base = dict(card(), batch=args.batch, layers=args.layers, dtype=str(args.dtype).replace("torch.", ""),
                iters=args.iters, rounds=args.rounds)
    recs = []
    if args.only in (None, "wra"):
        for tl, nb in ((args.txt_len, args.num_bb), ([62, 62], [100, 100])):
            v, extra = wra_variants(args, tl, nb)
            recs.append(compare("wra_fwd_bwd", v, args, dict(base, **extra)))
    if args.only in (None, "step"):
        for with_wra in (False, True):
            v, extra = step_variants(args, with_wra)
            recs.append(compare("itm_train_step", v, args, dict(base, txt_len=args.txt_len, num_bb=args.num_bb,
                                                                **extra)))
    for r in recs:
        line = json.dumps(r)
        print(line)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
