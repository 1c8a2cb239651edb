"""Cost of torch.use_deterministic_algorithms(True) on the graphed C2 training step.

The step is GraphedStep (UNITER-base, B = 64, MLM, FusedAdamW with clipping, bf16, dropout 0.1) replayed
from its CUDA graph; torch's flag off and on are alternated, one graph each (the flag is part of the
graph's key).  With the flag on torch also NaN-fills new allocations (its default), which is part of
what a user of the flag pays.  One JSON record per run, then a summary:

    python tools/reproducible_cost.py --out profiles/h100_c2_reproducible_graphed_cost.jsonl
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--modes", default="off,on",
                    help="torch flag settings to alternate; 'off' alone also runs against an earlier version of "
                         "the package (copy this script into its tree) to compare the default-mode step")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("reproducible_cost: needs a GPU")

    from uniter_b200 import _lib
    from uniter_b200.graphed import GraphedStep
    from uniter_b200.heads import UniterForMLM
    from uniter_b200.model import UniterConfig
    from uniter_b200.optim import FusedAdamW
    from uniter_b200.synth import pad_mlm_index, synth_batch
    lib = _lib.load()
    _lib.check(lib.ub200_device_check())

    torch.manual_seed(0)
    cfg = UniterConfig(28996, hidden_size=768, num_hidden_layers=12, num_attention_heads=12,
                       intermediate_size=3072, max_position_embeddings=512)
    mod = UniterForMLM(cfg, 2048).to("cuda", torch.bfloat16).train()
    opt = FusedAdamW(mod.parameters(), lr=1e-4, weight_decay=0.01)
    b = pad_mlm_index(synth_batch(64, 12, 28, 26, 46, 1234, mlm_prob=0.15), 64)
    lens = [x + y for x, y in zip(b["txt_lens"], b["num_bbs"])]
    host = {k: v.pin_memory() for k, v in b.items() if torch.is_tensor(v)}
    step = GraphedStep(mod, lambda bb: (mod(bb).sum() * bb["mlm_inv_n"]).squeeze(), optimizer=opt,
                       optimizer_kwargs={"max_grad_norm": 1.0})

    gpu = card()
    records = []
    for run in range(args.runs):
        for on in [m == "on" for m in args.modes.split(",")]:
            torch.use_deterministic_algorithms(on)
            bk = step.stage(host, lens)
            for _ in range(args.warmup):
                step.replay(bk)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step.replay(bk)
            e1.record()
            torch.cuda.synchronize()
            rec = dict(gpu=gpu, workload="C2 graphed step (replay): UNITER-base, B=64, T=%d, MLM, FusedAdamW + "
                       "clipping, bf16, dropout 0.1" % sum(lens), run=run, use_deterministic_algorithms=on,
                       launches=bk.launches, steps=args.steps, ms_per_step=e0.elapsed_time(e1) / args.steps)
            records.append(rec)
            print(json.dumps(rec), flush=True)
    torch.use_deterministic_algorithms(False)
    off = sorted(r["ms_per_step"] for r in records if not r["use_deterministic_algorithms"])
    on = sorted(r["ms_per_step"] for r in records if r["use_deterministic_algorithms"])
    summary = dict(gpu=gpu, summary=True, captures=step.captures, off_ms=off, on_ms=on)
    if off and on:
        summary["cost_pct_median"] = 100.0 * (on[len(on) // 2] / off[len(off) // 2] - 1.0)
    records.append(summary)
    print(json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            for r in records:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
