"""Time the referring-expression task on one GPU, two comparisons in one run, alternating their variants:

  step   one RE training step of UniterForReferringExpressionComprehension (UNITER-base geometry,
         cls loss, forward + backward + FusedAdamW with clipping): eager against GraphedStep replay;
  head   the head alone, forward + backward over the gathered region rows: the fused kernels
         (ub200_region_score_*) against the torch composition they replace (LibLinear with N = 1,
         scatter into the padded [B, max_num_bb] scores, masked_fill, F.cross_entropy, autograd).

B defaults to 128 (train_batch_size of config/train-refcoco-base-1gpu.json).  The text and region
counts are ASSUMPTIONS, not RefCOCO statistics: each sample draws its text length and region count
uniformly from --txt-len and --num-bb (seeded).  Times are medians over --rounds rounds of --iters
steps each, from CUDA events around work that ends in a synchronise.  One JSON line per comparison,
with the card name and power limit, goes to stdout and (appended) to --out.

    python tools/re_step.py --out /tmp/re_step.jsonl
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown", "max_sm_clock": "unknown"}


def batch(args, seed):
    from uniter_b200.batching import re_collate
    g = torch.Generator().manual_seed(seed)
    samples = []
    for _ in range(args.batch):
        tl = int(torch.randint(args.txt_len[0], args.txt_len[1] + 1, (1,), generator=g))
        nbb = int(torch.randint(args.num_bb[0], args.num_bb[1] + 1, (1,), generator=g))
        samples.append((torch.randint(1000, 28000, (tl,), generator=g), torch.randn(nbb, 2048, generator=g),
                        torch.rand(nbb, 7, generator=g), torch.ones(tl + nbb, dtype=torch.long),
                        torch.zeros(nbb, dtype=torch.uint8), torch.randint(0, nbb, (1,), generator=g)))
    b = re_collate(samples)
    lens = [a + c for a, c in zip(b["txt_lens"], b["num_bbs"])]
    return {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}, lens


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def compare(name, variants, args, extra):
    for fn in variants.values():          # warm-up: module loads, allocator, graph capture
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for k, fn in variants.items():
            times[k].append(timed(fn, args.iters))
    rec = dict(extra, what=name, unit="ms", **{k + "_ms": round(median(v), 4) for k, v in times.items()},
               **{k + "_all_ms": [round(x, 4) for x in v] for k, v in times.items()})
    a, b = list(times)
    rec["ratio_%s_over_%s" % (b, a)] = round(median(times[b]) / median(times[a]), 4)
    return rec


def step_variants(args):
    from uniter_b200.arena import GradArena
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForReferringExpressionComprehension
    from uniter_b200.model import UniterConfig, register_lengths
    from uniter_b200.optim import FusedAdamW
    cfg = UniterConfig(28996, hidden_size=768, num_hidden_layers=args.layers, num_attention_heads=12,
                       intermediate_size=3072, max_position_embeddings=512)
    torch.manual_seed(0)
    mod = UniterForReferringExpressionComprehension(cfg, 2048).to("cuda", args.dtype).train()
    host, lens = batch(args, 1)
    loss_fn = lambda b: mod(b).sum() / args.batch          # noqa: E731
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
    return {"eager": eager, "graphed": lambda: step(host, lens)}, {"T": sum(lens)}


def head_variants(args):
    import torch.nn.functional as F
    from uniter_b200 import _lib
    from uniter_b200.heads import _RegionScoreHead
    from uniter_b200.model import LibLinear
    host, _ = batch(args, 2)
    seg = host["re_seg"].cuda()
    om = host["obj_masks"].cuda()
    targets = host["targets"].view(-1).cuda()
    B, S = om.shape
    R = host["re_index"].numel()
    g = torch.Generator(device="cuda").manual_seed(3)
    rows = torch.randn(R, 768, device="cuda", generator=g).to(args.dtype).requires_grad_(True)
    lin = torch.nn.Linear(768, 1).to("cuda", args.dtype)
    # padded position of every row (b * S + k), R * 1 "no position" slots for the padding rows
    pos = torch.full((R,), B * S, dtype=torch.long)
    for b in range(B):
        st, n = int(host["re_seg"][0, b]), int(host["re_seg"][1, b])
        pos[st:st + n] = torch.arange(b * S, b * S + n)
    pos = pos.cuda()
    mask = om.bool()

    def fused():
        loss = _RegionScoreHead.apply(rows, lin.weight, lin.bias, seg, om, targets, None, _lib.RE_CLS, 0.0)
        loss.sum().backward()

    def torch_composition():
        s = LibLinear.apply(rows, lin.weight, lin.bias, False, False)          # [R, 1]
        flat = s.new_zeros(B * S + 1).index_copy(0, pos, s.view(-1))[:B * S]  # scatter; padding rows -> slot B*S
        scores = flat.view(B, S).masked_fill(mask, -1e4)
        F.cross_entropy(scores, targets, reduction="none").sum().backward()

    return {"torch": torch_composition, "fused": fused}, {"R": R, "max_num_bb": S}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--txt-len", type=int, nargs=2, default=[8, 24], metavar=("MIN", "MAX"),
                    help="text length range, [CLS] and [SEP] included (assumption)")
    ap.add_argument("--num-bb", type=int, nargs=2, default=[5, 20], metavar=("MIN", "MAX"),
                    help="regions per image (assumption)")
    ap.add_argument("--layers", type=int, default=12)
    ap.add_argument("--dtype", choices=["fp16", "bf16"], default="fp16")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=["step", "head"], default=None)
    ap.add_argument("--out", default=None, help="JSONL file to append to")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("re_step.py measures on the GPU; no CUDA device here")
    args.dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    base = dict(card(), batch=args.batch, txt_len=args.txt_len, num_bb=args.num_bb, layers=args.layers,
                dtype=str(args.dtype).replace("torch.", ""), iters=args.iters, rounds=args.rounds)
    recs = []
    if args.only in (None, "head"):
        v, extra = head_variants(args)
        recs.append(compare("re_head_fwd_bwd", v, args, dict(base, **extra)))
    if args.only in (None, "step"):
        v, extra = step_variants(args)
        recs.append(compare("re_train_step", v, args, dict(base, **extra)))
    for r in recs:
        line = json.dumps(r)
        print(line)
        if args.out:
            with open(args.out, "a") as fh:
                fh.write(line + "\n")


if __name__ == "__main__":
    main()
