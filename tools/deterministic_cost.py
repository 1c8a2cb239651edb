"""Cost of the deterministic mode (ub200_set_deterministic) on the C2 training step.

The step is the eager C2 step: UNITER-base (12 layers), B = 64 (T = 3451 tokens), MLM head, dropout 0.1,
forward + backward + FusedAdamW with clipping, bf16.  Runs with the mode off and on alternate
(`--runs` each, `--steps` timed steps after `--warmup`), timed with CUDA events around whole steps.
Prints one JSON record per run and a summary; `--out` also writes them as JSON lines.  The card's name
and power limit are read in the same process and recorded with the numbers.

    python tools/deterministic_cost.py --out profiles/h100_c2_deterministic_cost.jsonl
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_cost: needs a GPU")

    from uniter_b200 import _lib
    from uniter_b200.arena import GradArena
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.model import UniterConfig, register_lengths
    from uniter_b200.optim import FusedAdamW
    from uniter_b200.synth import pad_mlm_index, synth_batch
    lib = _lib.load()
    _lib.check(lib.ub200_device_check())

    torch.manual_seed(0)
    cfg = UniterConfig(28996, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                       intermediate_size=3072, max_position_embeddings=512)
    mod = UniterForMLM(cfg, 2048).to("cuda", torch.bfloat16).train()
    GradArena.attach(mod)
    opt = FusedAdamW(mod.parameters(), lr=1e-4, weight_decay=0.01)
    b = pad_mlm_index(synth_batch(64, 12, 28, 26, 46, 1234, mlm_prob=0.15), 64)
    lens = [x + y for x, y in zip(b["txt_lens"], b["num_bbs"])]
    batch = {k: v.cuda() for k, v in b.items() if torch.is_tensor(v)}
    register_lengths(batch["attn_masks"], lens, prefix=True)

    def step():
        opt.zero_grad()
        loss = (mod(batch).sum() * batch["mlm_inv_n"]).squeeze()
        loss.backward()
        opt.step(max_grad_norm=1.0)

    gpu = card()
    records = []
    for run in range(args.runs):
        for mode in (0, 1):
            lib.ub200_set_deterministic(mode)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            rec = dict(gpu=gpu, workload="C2 eager step: UNITER-base, B=64, T=%d, MLM, FusedAdamW + clipping, bf16"
                       % sum(lens), run=run, deterministic=mode, steps=args.steps,
                       ms_per_step=e0.elapsed_time(e1) / args.steps)
            records.append(rec)
            print(json.dumps(rec), flush=True)
    lib.ub200_set_deterministic(0)
    off = sorted(r["ms_per_step"] for r in records if not r["deterministic"])
    on = sorted(r["ms_per_step"] for r in records if r["deterministic"])
    summary = dict(gpu=gpu, summary=True, off_ms=off, on_ms=on,
                   cost_pct_median=100.0 * (on[len(on) // 2] / off[len(off) // 2] - 1.0))
    records.append(summary)
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            for r in records:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
