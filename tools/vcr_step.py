"""Time VCR fine-tuning on one GPU, two comparisons in one run, alternating their variants:

  head   the head alone, forward + backward over the pooled [CLS] rows: vcr_output as the torch
         composition (nn.Linear -> nn.ReLU -> nn.LayerNorm -> nn.Linear, autograd) against the library
         (LibTransform(act="relu") with the fused ReLU + LayerNorm kernels at 2H, then LibLinear);
  step   one VCR training step of UniterForVisualCommonsenseReasoning (UNITER-base geometry after
         init_type_embedding / init_word_embedding(81); forward, backward, DynamicLossScaler and
         FusedAdamW with clipping at 2.0): eager against GraphedStep replay.

The batch is built to the token budget of config/train-vcr-base-4gpu.json (train_batch_size 4000): whole
questions of 4 choices are added while (longest sequence) x (number of sequences) stays within 4000.
The text and region counts are ASSUMPTIONS, not VCR statistics: each question draws one region count
uniformly from --num-bb (the config's min_bb / max_bb by default) and each choice its text length from
--txt-len (seeded).  Times are medians over --rounds alternated rounds of --iters steps each, from CUDA
events around work that ends in a synchronise.  One JSON line per comparison, with the card name and
power limit read in the same run, goes to stdout and (appended) to --out.

    python tools/vcr_step.py --out /tmp/vcr_step.jsonl
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

VOCAB, N_SPECIAL, H = 28996, 81, 768


def batch(args, seed):
    from uniter_b200.batching import vcr_collate
    g = torch.Generator().manual_seed(seed)
    questions, longest, n = [], 0, 0
    while True:
        nbb = int(torch.randint(args.num_bb[0], args.num_bb[1] + 1, (1,), generator=g))
        feat, pos = torch.randn(nbb, 2048, generator=g), torch.rand(nbb, 7, generator=g)
        choices = []
        for c in range(4):
            tl = int(torch.randint(args.txt_len[0], args.txt_len[1] + 1, (1,), generator=g))
            ids = torch.randint(1000, VOCAB + N_SPECIAL, (tl,), generator=g)
            types = torch.tensor([0] * (tl // 3) + [2] * (tl - tl // 3))
            choices.append((ids, types, feat, pos, torch.ones(tl + nbb, dtype=torch.long),
                            torch.tensor([1 if c == 0 else 0])))
        new_longest = max([longest] + [c[4].numel() for c in choices])
        if questions and new_longest * (n + 4) > args.tokens:
            break
        questions.append(tuple(choices))
        longest, n = new_longest, n + 4
    b = vcr_collate(questions)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    return {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens


def _model(args):
    from uniter_b200.heads import UniterForVisualCommonsenseReasoning
    from uniter_b200.model import UniterConfig
    cfg = UniterConfig(VOCAB, hidden_size=H, num_hidden_layers=args.layers, num_attention_heads=12,
                       intermediate_size=3072, max_position_embeddings=512)
    torch.manual_seed(0)
    mod = UniterForVisualCommonsenseReasoning(cfg, 2048)
    mod.init_type_embedding()
    mod.init_word_embedding(N_SPECIAL)
    return mod.to("cuda", args.dtype).train()


def step_variants(args):
    from uniter_b200.arena import GradArena
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.model import register_lengths
    from uniter_b200.optim import DynamicLossScaler, FusedAdamW
    mod = _model(args)
    host, lens = batch(args, 1)
    loss_fn = lambda b: mod(b)                      # noqa: E731
    opt_e = FusedAdamW(mod.parameters(), lr=1e-6, weight_decay=0.01)
    sc_e = DynamicLossScaler(init_scale=2.**12)
    arena = GradArena.attach(mod)
    dev = {k: v.cuda() for k, v in host.items()}

    def eager():
        register_lengths(dev["attn_masks"], lens, prefix=True)
        arena.begin_step()
        sc_e.scale(loss_fn(dev)).backward()
        arena.finish_step()
        arena.end_step_mode()
        opt_e.step(grad_scale=sc_e, max_grad_norm=2.0)

    opt_g = FusedAdamW(mod.parameters(), lr=1e-6, weight_decay=0.01)
    step = GraphedStep(mod, loss_fn, optimizer=opt_g, optimizer_kwargs={"max_grad_norm": 2.0},
                       loss_scaler=DynamicLossScaler(init_scale=2.**12))
    return {"eager": eager, "graphed": lambda: step(host, lens)}, {
        "sequences": len(lens), "T": sum(lens), "max_seqlen": max(lens)}


def head_variants(args):
    from uniter_b200.heads import LibTransform
    from uniter_b200.model import LibLinear
    host, lens = batch(args, 2)
    B = len(lens)
    g = torch.Generator(device="cuda").manual_seed(3)
    pooled = torch.randn(B, H, device="cuda", generator=g).to(args.dtype).requires_grad_(True)
    head = torch.nn.Sequential(torch.nn.Linear(H, 2 * H), torch.nn.ReLU(), torch.nn.LayerNorm(2 * H, eps=1e-12),
                               torch.nn.Linear(2 * H, 2)).to("cuda", args.dtype)
    targets = host["targets"].view(-1).cuda()
    F = torch.nn.functional

    def library():
        z = LibTransform.apply(pooled, head[0].weight, head[0].bias, head[2].weight, head[2].bias, "relu")
        s = LibLinear.apply(z, head[3].weight, head[3].bias, False, False)
        F.cross_entropy(s.float(), targets).backward()

    def torch_composition():
        F.cross_entropy(head(pooled).float(), targets).backward()

    return {"torch": torch_composition, "library": library}, {"sequences": B}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--tokens", type=int, default=4000, help="token budget (train_batch_size of the config)")
    ap.add_argument("--txt-len", type=int, nargs=2, default=[30, 90], metavar=("MIN", "MAX"),
                    help="text length of one choice, [CLS] / [SEP] included (assumption)")
    ap.add_argument("--num-bb", type=int, nargs=2, default=[10, 100], metavar=("MIN", "MAX"),
                    help="regions per image (assumption; the config's min_bb / max_bb)")
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=["step", "head"], default=None)
    ap.add_argument("--out", default=None, help="JSONL file to append to")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("vcr_step.py measures on the GPU; no CUDA device here")
    args.dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    base = dict(card(), tokens=args.tokens, txt_len=args.txt_len, num_bb=args.num_bb, layers=args.layers,
                dtype=str(args.dtype).replace("torch.", ""), iters=args.iters, rounds=args.rounds)
    recs = []
    if args.only in (None, "head"):
        v, extra = head_variants(args)
        recs.append(compare("vcr_head_fwd_bwd", v, args, dict(base, **extra)))
    if args.only in (None, "step"):
        v, extra = step_variants(args)
        recs.append(compare("vcr_train_step", v, args, dict(base, **extra)))
    for r in recs:
        line = json.dumps(r)
        print(line)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
