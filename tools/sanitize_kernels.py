"""One small launch of every libub200 kernel family at C1-like shapes, for compute-sanitizer:

    compute-sanitizer --tool memcheck  python tools/sanitize_kernels.py
    compute-sanitizer --tool racecheck python tools/sanitize_kernels.py

GEMM: every operand-major form, 1-SM / 2-SM / grouped / split-K kernels; attention
forward + backward at S = 1, 64, 129, 512 (pair packing, single block, multi block); LayerNorm
forward / backward; the embedding front-end, MLM head and optimizer kernels through one tiny
training step.  Prints 'sanitize ok' at the end (the sanitizer's own summary follows)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from uniter_b200 import ops  # noqa: E402

torch.manual_seed(0)
dev = "cuda"
dt = torch.bfloat16


def r(*s):
    return (torch.randn(*s, device=dev) * 0.1).to(dt)


# ---- GEMM forms
M, N, K = 112, 768, 768
a, w, bias, res = r(M, K), r(N, K), r(N), r(M, N)
ops.gemm(a, w, bias=bias)                                                  # K-major, bias
ops.gemm(a, w, bias=bias, residual=res, dropout_p=0.1, rng_seed=1, rng_stream=2)
ops.gemm(a, r(3072, K), bias=r(3072), gelu=True)
ops.gemm(a, w, b_major=1)                                                   # dgrad form
ops.gemm(r(M, N), r(M, K), a_major=1, b_major=1)                            # wgrad form
ops.gemm(r(300, K), w, bias=bias, tile_n=256, cluster=2)                    # 2-SM pair
ops.gemm(r(300, K), w, bias=bias, tile_n=128, cluster=2)
ops.gemm(a, w, tile_n=64, cluster=1)
ops.gemm(a, w, tile_n=192, cluster=1)
ops.gemm(r(M, 2000), r(2000, 128), b_major=1, k_splits=-1)                  # split-K, fp32 atomics
import ctypes as C  # noqa: E402
from uniter_b200 import _lib  # noqa: E402
lib = _lib.load()
T = 112
wg = (_lib.GemmArgs * 4)()
outs = []
for i, (m_, n_) in enumerate(((768, 3072), (3072, 768), (2304, 768), (768, 768))):
    A_, B_ = r(T, m_), r(T, n_)
    O_ = torch.empty(m_, n_, device=dev, dtype=dt)
    outs.append((A_, B_, O_))
    wg[i] = _lib.GemmArgs(a=A_.data_ptr(), b=B_.data_ptr(), lda=m_, ldb=n_, a_major=1, b_major=1, M=m_, N=n_,
                          K=T, dtype=_lib.BF16, epilogue=0, out=O_.data_ptr(), ldo=n_)
_lib.check(lib.ub200_gemm_grouped(wg, 4, _lib.current_stream()))

# ---- attention
for lens in ([1, 64, 33], [129, 70], [512]):
    cu = torch.tensor([0] + list(torch.tensor(lens).cumsum(0)), device=dev, dtype=torch.int32)
    Tt = sum(lens)
    qkv = r(Tt, 3 * 128)
    ctx, lse = ops.attn_fwd(qkv, cu, max(lens), 2, dropout_p=0.1, rng_seed=3, rng_stream=4)
    ops.attn_bwd(qkv, ctx, lse, r(Tt, 128), cu, max(lens), 2, dropout_p=0.1, rng_seed=3, rng_stream=4,
                 dbias=torch.zeros(3 * 128, device=dev))

# ---- LayerNorm
x, g, b = r(100, 768), r(N) + 1, r(N)
y = ops.layernorm_fwd(x, g, b)
ops.layernorm_bwd(r(100, 768), x, g, dropout_p=0.1, rng_seed=5, rng_stream=6)

# ---- one tiny training step: embedding front-end, encoder stack, MLM head, optimizer
from uniter_b200.heads import UniterForMLM  # noqa: E402
from uniter_b200.model import UniterConfig  # noqa: E402
from uniter_b200.optim import FusedAdamW  # noqa: E402
from uniter_b200.synth import synth_batch  # noqa: E402
cfg = UniterConfig(2000, hidden_size=128, num_hidden_layers=1, num_attention_heads=2, intermediate_size=512,
                   max_position_embeddings=64)
mod = UniterForMLM(cfg, 64).to(dev, dt).train()
batch = {k: (v.to(dev) if torch.is_tensor(v) else v)
         for k, v in synth_batch(3, 4, 9, 3, 7, seed=1, img_dim=64, vocab_size=2000, mlm_prob=0.3).items()}
opt = FusedAdamW(mod.parameters(), lr=1e-3)
mod(batch).mean().backward()
opt.step(max_grad_norm=1.0)
torch.cuda.synchronize()
print("sanitize ok")
