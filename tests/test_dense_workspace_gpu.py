"""The dense workspace queries size every route exactly: each C entry point runs in a workspace of exactly the
queried size, followed by a sentinel-filled guard that must come back untouched.  Also the fused EdgeConv with
train-mode BatchNorm at 33 <= K <= 48 on one 128-point cloud, where the tensor-core route's completion kernel
writes statistic rows past the (N/128)*B rows of its query tiles."""
import pytest
import torch

from oracle import dense as od

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
SENTINEL, GUARD = 0xA5, 1 << 16


@pytest.fixture
def guarded(monkeypatch):
    """Every workspace _native allocates is exactly the queried size, followed by GUARD sentinel bytes."""
    from deep_gcns_torch_b200 import _native
    bufs = []

    def workspace(nbytes, dev):
        buf = torch.full((int(nbytes) + GUARD,), SENTINEL, dtype=torch.uint8, device=dev)
        bufs.append((buf, int(nbytes)))
        return buf[:int(nbytes)]

    monkeypatch.setattr(_native, "_workspace", workspace)
    yield bufs
    torch.cuda.synchronize()
    assert bufs
    for buf, n in bufs:
        assert bool((buf[n:] == SENTINEL).all()), "a kernel wrote past the queried workspace"
    _native.set_knn_path("auto")


def _params(C, co, train, g):
    from deep_gcns_torch_b200 import _native
    w = (torch.randn(co, 2 * C, generator=g) / (2 * C) ** 0.5).cuda()
    b = (torch.randn(co, generator=g) * 0.1).cuda()
    bn = dict(bn_weight=torch.randn(co, generator=g).cuda(), bn_bias=(torch.randn(co, generator=g) * 0.2).cuda())
    if not train:
        bn.update(bn_mean=torch.zeros(co).cuda(), bn_var=torch.ones(co).cuda())
    return _native.ConvParams(w, b, "relu", None, _native.NORM_BATCH_TRAIN if train else _native.NORM_BATCH_EVAL, **bn)


def _x(B, C, N, g):
    return torch.randn(B, C, N, 1, generator=g).cuda()


def _knn(path, B, C, N, k):
    def run(_native, g):
        _native.set_knn_path(path)
        _native.knn_graph(_x(B, C, N, g), k, want_nbr=True)
    return run


def _dyn(conv, path, train, B, C, co, N, k):
    def run(_native, g):
        _native.set_knn_path(path)
        _native.dyn_conv_forward(conv, _x(B, C, N, g), _params(C, co, train, g), k, want_nbr=True)
    return run


def _static(conv, use_nbr, backward):
    def run(_native, g):
        B, C, co, N, k = 2, 40, 64, 300, 9
        x = _x(B, C, N, g)
        nbr = torch.randint(0, N, (B, N, k), generator=g, dtype=torch.int32).cuda()
        centre = torch.randint(0, N, (B, N, k), generator=g).cuda()
        graph = dict(nbr=nbr) if use_nbr else dict(edge_index=torch.stack([nbr.long(), centre]))
        prm = _params(C, co, True, g)
        out = _native.graph_conv_forward(conv, x, prm, **graph)
        if backward:
            _native.graph_conv_backward(conv, x, prm, torch.randn(out.shape, generator=g).cuda(), **graph)
    return run


ROUTES = {
    "small_fp32": _knn("auto", 2, 96, 1000, 16),
    "tc4": _knn("auto", 2, 64, 1024, 16),
    "tc1": _knn("tc1", 2, 64, 1024, 16),
    "tc1_train": _dyn("edge", "auto", True, 2, 64, 64, 1024, 16),
    "slab_tc_rows": _knn("auto", 2, 64, 4096, 64),
    "slab_ffma_rows": _knn("ffma", 2, 64, 4096, 64),
    "static_edge_index": _static("edge", False, False),
    "static_nbr": _static("edge", True, False),
    "mr_node": _dyn("mr", "auto", True, 2, 64, 64, 1024, 16),
    "mr_static": _static("mr", True, False),
    "edge_backward": _static("edge", True, True),
    "mr_backward": _static("mr", False, True),
}


@pytest.mark.parametrize("route", sorted(ROUTES))
def test_route_fits_queried_workspace(guarded, route):
    from deep_gcns_torch_b200 import _native
    ROUTES[route](_native, torch.Generator().manual_seed(len(route)))


@pytest.mark.parametrize("K", [33, 40, 48])
@pytest.mark.parametrize("co", [64, 128])
def test_train_edgeconv_single_tile_large_k(guarded, co, K):
    from deep_gcns_torch_b200 import _native
    g = torch.Generator().manual_seed(co + K)
    C, N = 64, 128
    x = _x(1, C, N, g)
    prm = _params(C, co, True, g)
    y, nbr = _native.dyn_conv_forward("edge", x, prm, K, want_nbr=True)
    _native.set_knn_path("ffma")
    _, nbr_ffma = _native.dyn_conv_forward("edge", x, _params(C, co, True, g), K, want_nbr=True)
    assert torch.equal(nbr, nbr_ffma)

    # fp64 oracle on the graph the kernel selected
    centre = torch.arange(N, device=nbr.device).view(1, N, 1).expand_as(nbr)
    ei = torch.stack([nbr.long(), centre]).cpu()
    p = {"weight": prm.weight.double().cpu().view(co, 2 * C, 1, 1), "bias": prm.bias.double().cpu(),
         "norm": {"weight": prm.bn_weight.double().cpu(), "bias": prm.bn_bias.double().cpu(),
                  "running_mean": None, "running_var": None}}
    xd = x.double().cpu()
    ref_y = od.graph_conv(xd, ei, p, "edge", "relu", "batch", training=True)
    torch.testing.assert_close(y.double().cpu(), ref_y, rtol=RTOL, atol=ATOL)
    x_i, x_j = od.batched_index_select(xd, ei[1]), od.batched_index_select(xd, ei[0])
    feat = torch.cat([x_i, x_j - x_i], 1)
    a = torch.relu(torch.nn.functional.conv2d(feat, p["weight"], p["bias"]))
    torch.testing.assert_close(prm.batch_mean.double().cpu(), a.mean((0, 2, 3)), rtol=RTOL, atol=1e-5)
    torch.testing.assert_close(prm.batch_var.double().cpu(), a.var((0, 2, 3), unbiased=False), rtol=RTOL, atol=1e-5)
