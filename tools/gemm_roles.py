#!/usr/bin/env python
"""Time each GEMM role of a UNITER-base encoder layer at the C2 shapes, with CUDA events.

    python tools/gemm_roles.py [--M 3456] [--dtype bf16] [--iters 200] [--reps 5]
                               [--roles qkv_fwd,...] [--tiles auto,192,256c2] [--root DIR] [--tag NAME]

Each role is ub200_gemm with the encoder's operand majors and epilogue (bias, GELU, dGELU + column
sum, dropout 0.1 + residual) at T = M tokens.  One JSON line per (role, tile): the median over --reps
replays of a CUDA graph of --iters back-to-back launches (after warm-up), the spread of those
replays, TFLOP/s, and the GPU name, power limit and maximum SM clock read in the same run.
--tiles: "auto" = pick_config's choice (what the encoder runs), "NNN" = N tile width NNN with single
CTAs, "NNNc2" = with 2-CTA clusters.  --root imports uniter_b200 from another checkout (e.g. the
parent commit) so that two builds can be timed alternately in one session.
"""
import argparse
import json
import os
import subprocess
import sys

H, I = 768, 3072
# role: (N, K, B_MN, epilogue keywords); A is [M, K] K-major
ROLES = {
    "qkv_fwd": (3 * H, H, False, "bias"),
    "attnout_fwd": (H, H, False, "bias_drop_res"),
    "ffn1_fwd": (I, H, False, "bias_gelu"),
    "ffn2_fwd": (H, I, False, "bias_drop_res"),
    "ffn2_dgrad": (I, H, True, "dgelu_colsum"),
    "ffn1_dgrad": (H, I, True, "res"),
    "attnout_dgrad": (H, H, True, "none"),
    "qkv_dgrad": (H, 3 * H, True, "res"),
}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in out.split(",")]
        return dict(gpu=name, power_limit=power, max_sm_clock=clk)
    except Exception as e:   # the timing itself does not depend on it
        return dict(gpu="unknown (%s)" % e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=3456)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--roles", default=",".join(ROLES))
    ap.add_argument("--tiles", default="auto")
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--tag", default="tree")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from uniter_b200 import _lib, ops

    assert torch.cuda.is_available(), "gemm_roles.py times on the GPU; there is no CPU fall-back"
    lib = _lib.load()
    _lib.check(lib.ub200_device_check())
    dt = torch.bfloat16 if args.dtype == "bf16" else torch.float16
    info = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(0)
    M = args.M
    lines = []
    for role in args.roles.split(","):
        N, K, b_mn, epi = ROLES[role]
        a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dt)
        b = (torch.randn(K, N, device="cuda", generator=g) if b_mn else
             torch.randn(N, K, device="cuda", generator=g)).mul(0.03).to(dt)
        out = torch.empty(M, N, device="cuda", dtype=dt)
        kw = dict(b_major=1 if b_mn else 0, out=out)
        if "bias" in epi:
            kw["bias"] = (torch.randn(N, device="cuda", generator=g) * 0.1).to(dt)
        if "res" in epi:
            kw["residual"] = torch.randn(M, N, device="cuda", generator=g).to(dt)
        if "drop" in epi:
            kw.update(dropout_p=0.1, rng_seed=7, rng_stream=3)
        if "gelu" in epi and "dgelu" not in epi:
            kw["gelu"] = True
        if "dgelu" in epi:
            kw.update(dgelu=True, aux=torch.randn(M, N, device="cuda", generator=g).to(dt),
                      colsum=torch.zeros(N, device="cuda"))
        for tile in args.tiles.split(","):
            mkw = dict(kw)
            if tile != "auto":
                mkw.update(tile_n=int(tile.split("c")[0]), cluster=2 if tile.endswith("c2") else 1)
            # the launches are replayed from one CUDA graph, as in the training step, so that the
            # host's per-call cost (tens of microseconds through ctypes) does not hide the kernel time
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(args.warmup):
                    ops.gemm(a, b, **mkw)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=s):
                    for _ in range(args.iters):
                        ops.gemm(a, b, **mkw)
            torch.cuda.current_stream().wait_stream(s)
            graph.replay()
            torch.cuda.synchronize()
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                graph.replay()
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / args.iters)
            del graph
            times.sort()
            us = times[len(times) // 2]
            rec = dict(tag=args.tag, role=role, tile=tile, M=M, N=N, K=K, dtype=args.dtype, us=round(us, 3),
                       spread_us=round(times[-1] - times[0], 3), tflops=round(2.0 * M * N * K / us * 1e-6, 1),
                       iters=args.iters, reps=args.reps, **info)
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "a") as fh:
            for r in lines:
                fh.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
