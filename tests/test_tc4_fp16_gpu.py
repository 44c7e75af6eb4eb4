"""knn_tc4_kernel's single fp16 pre-filter product at the edges of the fp16 range.

Clouds scaled by 2^16 (|x_c| beyond the fp16 range: the clamp and the range guard send every query to the exact
completion kernel), by 2^-20 (fp16 subnormals) and a cloud with one far outlier (large max |x_j|, hence a wide eps).
Neighbour lists must equal the fp32 kernel's bit for bit, features stay within the four-tile tests' tolerance of
it and equal the one-tile-per-CTA kernel's (bf16 split) bit for bit: the completion kernel and the fused consumer
reduce the same neighbour set by max / min, which commute with the rounded p + q and the activation, so who
answered a query does not change its bits.  At the headline shape at most 1e-4 of the set-only queries may be left
uncertified."""
import pytest
import torch


def _clouds():
    g = torch.Generator().manual_seed(4242)
    base = torch.randn(2, 64, 1024, 1, generator=g)
    outlier = base.clone()
    outlier[0, :, 7] *= 60.0
    outlier[1, :, 1000] += 500.0
    return {"scaled_2p16": base * 65536.0, "scaled_2m20": base * 2.0 ** -20, "outlier": outlier}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["scaled_2p16", "scaled_2m20", "outlier"])
def test_fp16_prefilter_range_edges_equal_fp32_path(name):
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    x = _clouds()[name].cuda()
    torch.manual_seed(3)
    mod = D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch", True).cuda().eval()
    graph = D.DenseDilatedKnnGraph(20, 1)
    out = {}
    try:
        for path in ("ffma", "tc1", "tc"):
            _native.set_knn_path(path)
            with torch.no_grad():
                out[path] = (graph(x), mod(x))
    finally:
        _native.set_knn_path("auto")
    assert torch.isfinite(out["tc"][1]).all()
    assert torch.equal(out["tc"][0], out["ffma"][0])
    torch.testing.assert_close(out["tc"][1], out["ffma"][1], rtol=1e-5, atol=1e-6)
    assert torch.equal(out["tc"][1], out["tc1"][1])


@pytest.mark.gpu
def test_fp16_prefilter_range_guard_sends_every_query_to_the_completion_kernel():
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    x = _clouds()["scaled_2p16"].cuda()
    torch.manual_seed(3)
    mod = D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch", True).cuda().eval()
    _native.tc_certification(True)
    try:
        _native.tc_certification_read()
        with torch.no_grad():
            mod(x)
        failed, queries = _native.tc_certification_read()
    finally:
        _native.tc_certification(False)
    assert queries == 2 * 1024 and failed == queries, (failed, queries)


@pytest.mark.gpu
def test_fp16_prefilter_certifies_the_headline_shape():
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(77)
    torch.manual_seed(0)
    mod = D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch", True).cuda().eval()
    _native.tc_certification(True)
    try:
        _native.tc_certification_read()
        with torch.no_grad():
            for _ in range(2):
                mod(torch.randn(16, 64, 4096, 1, generator=g).cuda())
        failed, queries = _native.tc_certification_read()
    finally:
        _native.tc_certification(False)
    assert queries == 2 * 16 * 4096, queries
    assert failed <= 1e-4 * queries, (failed, queries)
