"""Output bits of the encoder's GEMM epilogues do not depend on the N tile width or the 2-CTA cluster,
at the multi-wave FFN shape M = 3456 (C2 tokens), N = 3072, K = 768.

The epilogue warpgroup drains a finished tile from shared memory while the consumers run the next
tile's mainloop; a 128-wide tile fits the hand-off ring whole, wider tiles make the consumers wait
for the first chunks to drain.  Each tile width (and the cluster) gives a different hand-off schedule
over many tiles per CTA, and all of them must give the same bits: the epilogue is the same fp32 code
on the same fp32 accumulators whatever the schedule."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M, N, K = 3456, 3072, 768
TILES = [(64, 1), (128, 1), (192, 1), (256, 1), (128, 2), (256, 2)]


def _operands(dtype, b_major, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(K, N, device="cuda", generator=g) if b_major else
         torch.randn(N, K, device="cuda", generator=g)).mul(0.03).to(dtype)
    return g, a, w


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bias_gelu_bits_do_not_depend_on_tile(dtype):
    from uniter_b200 import ops
    g, a, w = _operands(dtype, 0, 11)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).to(dtype)
    outs = [ops.gemm(a, w, bias=bias, gelu=True, tile_n=bn, cluster=c, k_splits=1) for bn, c in TILES]
    for f, pre in outs[1:]:
        assert torch.equal(f, outs[0][0])
        assert torch.equal(pre, outs[0][1])
    ref = a.float() @ w.float().t() + bias.float()
    assert (outs[0][1].float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_dgelu_colsum_bits_do_not_depend_on_tile(dtype):
    from uniter_b200 import ops
    g, a, w = _operands(dtype, 1, 12)
    aux = torch.randn(M, N, device="cuda", generator=g).to(dtype)
    outs, sums = [], []
    for bn, c in TILES:
        cs = torch.zeros(N, device="cuda")
        outs.append(ops.gemm(a, w, b_major=1, dgelu=True, aux=aux, colsum=cs, tile_n=bn, cluster=c, k_splits=1))
        sums.append(cs)
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    # the column sum (of the fp32 values, before rounding) meets in float atomics, whose order of
    # arrival varies from run to run
    for s in sums[1:]:
        torch.testing.assert_close(s, sums[0], rtol=1e-5, atol=1e-3)
    assert (sums[0] - outs[0].float().sum(0)).abs().max().item() < 0.5


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_bias_dropout_residual_bits_do_not_depend_on_tile(dtype):
    from uniter_b200 import ops
    g, a, w = _operands(dtype, 0, 13)
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).to(dtype)
    res = torch.randn(M, N, device="cuda", generator=g).to(dtype)
    outs = [ops.gemm(a, w, bias=bias, residual=res, dropout_p=0.1, rng_seed=7, rng_stream=3,
                     tile_n=bn, cluster=c, k_splits=1) for bn, c in TILES]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    dropped = (outs[0].float() == res.float()).float().mean().item()   # dropped elements keep the residual
    assert 0.08 < dropped < 0.12
