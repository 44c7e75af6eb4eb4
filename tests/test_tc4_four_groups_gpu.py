"""knn_tc4_kernel with four query tiles per CTA: every remainder of query tiles per CTA.

A CTA runs min(4, tiles left) filter warpgroups; the groups it does not need exit at once, and thread 0 of group 0
issues the TMA for all of them.  The rows below give the remainders 1, 2 and 3 of N / 128 mod 4 (and 0) at the
list lengths 20 and 32, on the set-only consumer (DynConv2d) and the full exact re-rank (the index lists).  Lists
must be bit-equal to the one-tile-per-CTA tensor-core kernel and to the fp32 kernel, features bit-equal to the
one-tile-per-CTA kernel.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cfg", [
    # B, C, c_out, N, k, d, conv
    (2, 64, 64, 768, 20, 1, "edge"),      # 6 query tiles: a CTA of four groups, then one of two
    (1, 32, 64, 256, 9, 1, "edge"),       # 2 query tiles: one CTA, two groups idle; list of 20
    (2, 64, 32, 1280, 16, 1, "edge"),     # 10 query tiles: 4 + 4 + 2
    (1, 64, 48, 1152, 20, 1, "mr"),       # 9 query tiles: 4 + 4 + 1, MRConv consumer (c_in = 64)
    (1, 40, 64, 384, 12, 1, "edge"),      # 3 query tiles: one group idle; C = 40 -> three zero-padded K=16 blocks
    (1, 64, 64, 1536, 10, 2, "edge"),     # 12 query tiles: 4 + 4 + 4, dilation (exact re-rank path)
])
def test_four_groups_equal_tile_per_cta_and_fp32_paths(cfg):
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B, C, co, N, k, d, conv = cfg
    g = torch.Generator().manual_seed(N * 3 + C)
    x = torch.randn(B, C, N, 1, generator=g).cuda()
    x[0, :, 130] = x[0, :, 3]                                 # exact duplicates in two query tiles: ties
    x[-1, :, N - 1] = x[-1, :, 3]
    torch.manual_seed(3)
    mod = D.DynConv2d(C, co, k, d, conv, "relu", "batch", True).cuda().eval()
    graph = D.DenseDilatedKnnGraph(k, d)
    out = {}
    try:
        for path in ("ffma", "tc1", "tc"):
            _native.set_knn_path(path)
            with torch.no_grad():
                out[path] = (graph(x), mod(x))
    finally:
        _native.set_knn_path("auto")
    assert torch.equal(out["tc"][0], out["ffma"][0])
    assert torch.equal(out["tc"][0], out["tc1"][0])
    assert torch.equal(out["tc"][1], out["tc1"][1])
    torch.testing.assert_close(out["tc"][1], out["ffma"][1], rtol=1e-5, atol=1e-6)
