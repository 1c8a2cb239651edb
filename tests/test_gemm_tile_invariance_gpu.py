"""Output bits of the GEMM core do not depend on the N tile width or the 2-CTA cluster.

Every output element is one CTA's fp32 sum over K in k-block order; the tile width and the cluster
only change which CTA computes it.  So pick_config may change a shape's tile between token counts
(e.g. between a bucket's padded T and the eager T) without changing a single output bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H, I = 768, 3072


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("b_major", [0, 1])
def test_output_bits_do_not_depend_on_tile_width_or_cluster(dtype, b_major):
    from uniter_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(6)
    a = (torch.randn(1000, I, device="cuda", generator=g) * 0.5).to(dtype)
    w = (torch.randn(I, H, device="cuda", generator=g) if b_major else
         torch.randn(H, I, device="cuda", generator=g)).mul(0.03).to(dtype)
    res = torch.randn(1000, H, device="cuda", generator=g).to(dtype)
    outs = [ops.gemm(a, w, b_major=b_major, residual=res, tile_n=bn, cluster=c, k_splits=1)
            for bn, c in [(64, 1), (128, 1), (192, 1), (256, 1), (128, 2), (256, 2)]]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
