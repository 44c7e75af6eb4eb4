"""Exact ties and kinks on the GPU: zero-padded clouds, repeated points, zero biases, gamma = 0, parallel edges.

On the exact fixtures of exact_util every tie and every z == 0 is real, so nothing is adjudicated and nothing masked:
- every kNN route (profiler kernel names checked) returns the (distance, index)-lexicographic lists bit for bit, on
  clouds padded by one point, 25 % and 60 %, an all-zero cloud and a cloud of triplets, self-excluded or not;
- the dense EdgeConv / MRConv forward and every gradient match fp64 autograd of oracle.dense on that graph, with
  torch's subgradients: relu'(0) = 0, leaky_relu'(0) = 0.2, prelu'(0) = slope, and a tie of the EdgeConv max
  (gamma = 0 ties every edge) routed to the first edge;
- the sparse GENConv max routes a tie to the first edge in edge order (torch_scatter's CPU scatter_max, restated
  here: oracle.sparse's scatter_reduce('amax') splits ties evenly), and power / power_sum pass the gradient at the
  clamp bound 10 and none above it."""
import copy

import pytest
import torch
import torch.nn.functional as F

import backward_util as bu
import exact_util as eu
from oracle import dense as od
from oracle import sparse as osp

pytestmark = pytest.mark.gpu

KINDS = ["pad1", "pad25", "pad60", "zeros", "dup3"]


def _kernel_names(fn):
    return bu.kernel_names(fn)


def _on_path(path, fn):
    from deep_gcns_torch_b200 import _native
    _native.set_knn_path(path)
    try:
        return _kernel_names(fn)
    finally:
        _native.set_knn_path("auto")


def _assert_lists(got, want, what):
    got = got.long()
    bad = (got != want).any(-1)
    if bool(bad.any()):
        b, i = (int(v) for v in bad.nonzero()[0])
        raise AssertionError("%s: %d lists differ, first cloud %s query %d: got %s, want %s" % (
            what, int(bad.sum()), KINDS[b], i, got[b, i].tolist(), want[b, i].tolist()))


# name: C, N, k, dilation, knn path, kernel that must run
KNN_CASES = {
    "small-ragged": (3, 300, 16, 1, "auto", "knn_small_kernel"),
    "small-ffma": (16, 256, 20, 1, "ffma", "knn_small_kernel"),
    "tc-K40": (16, 256, 20, 2, "auto", "knn_tc_kernel"),
    "tc1-K20": (64, 512, 20, 1, "tc1", "knn_tc_kernel"),
    "tc4-K9": (16, 512, 9, 1, "auto", "knn_tc4_kernel"),
    "tc4-K20": (64, 512, 20, 1, "auto", "knn_tc4_kernel"),
    "slab-K100": (32, 512, 100, 1, "auto", "select_rows_fast_kernel"),
    "slab-K540": (64, 4096, 20, 27, "auto", "select_rows_fast_kernel"),
}


@pytest.mark.parametrize("exclude_self", [False, True], ids=["self", "no-self"])
@pytest.mark.parametrize("name", list(KNN_CASES))
def test_knn_lists_lexicographic(name, exclude_self):
    """DenseDilatedKnnGraph (self included) / DilatedKnnGraph (self excluded by index, with copies of the query at
    distance 0): the dilated lists equal the lexicographic order."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    C, N, k, d, path, kernel = KNN_CASES[name]
    x = eu.batch(KINDS, C, N, seed=N + C).cuda()
    graph = (D.DilatedKnnGraph if exclude_self else D.DenseDilatedKnnGraph)(k, d)
    ei, names = _on_path(path, lambda: graph(x))
    assert any(kernel in n for n in names), (kernel, sorted(names))
    if path == "tc1" or name == "tc-K40":
        assert not any("knn_tc4_kernel" in n for n in names)
    want = eu.lex_knn(x, k * d, exclude_self)[..., ::d]
    _assert_lists(ei[0], want, name)
    assert torch.equal(ei[1], torch.arange(N, device=x.device).view(1, N, 1).expand_as(ei[1]))


@pytest.mark.parametrize("k,C,conv", [(9, 16, "edge"), (20, 64, "edge"), (9, 64, "mr"), (20, 64, "mr")])
def test_tc4_set_consumer(k, C, conv):
    """knn_tc4_kernel's membership-only consumer (DynConv2d in inference, no list written): the K-th place of a
    padded cloud is an exact tie of hundreds of points, and the set must hold the lowest indices - the output
    equals fp64 on the lexicographic graph."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    x = eu.batch(KINDS, C, 512, seed=k).cuda()
    torch.manual_seed(0)
    mod = eu.set_params(D.DynConv2d(C, 32, k, 1, conv, "relu", "batch", True), "on", seed=k)
    p = od.params_from_module(mod.gconv.nn, dtype=torch.float64)
    mod = mod.cuda().eval()
    with torch.no_grad():
        y, names = _kernel_names(lambda: mod(x))
    assert any("knn_tc4_kernel" in n for n in names), sorted(names)
    ei = eu.edge_index_of(eu.lex_knn(x, k)).cpu()
    bu.assert_grads_close("output", y, od.graph_conv(x.cpu().double(), ei, p, conv, "relu", "batch", False))


ACTS = {"relu": ("relu", None), "leakyrelu": ("leakyrelu", None), "prelu": ("prelu", 0.25),
        "prelu-neg": ("prelu", -0.25)}
DENSE_KINDS = ["pad25", "dup3"]


def _module_grads(mod, x, wgt, ei=None):
    """Forward (static on `ei`, else dynamic) and backward of a copy of `mod`; returns (output, the graph the
    forward used, {x, weight, bias, slope, bn_w, bn_b: gradient})."""
    mod = copy.deepcopy(mod)
    xc = x.clone().requires_grad_(True)
    y = mod(xc, ei) if ei is not None else mod(xc)
    used = ei if ei is not None else eu.edge_index_of(y.grad_fn.nbr)
    (y * wgt).sum().backward()
    nn_ = mod.gconv.nn
    got = {"x": xc.grad, "weight": nn_[0].weight.grad, "bias": nn_[0].bias.grad if nn_[0].bias is not None else None}
    for m in nn_:
        if isinstance(m, torch.nn.PReLU):
            got["slope"] = m.weight.grad
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            got["bn_w"], got["bn_b"] = m.weight.grad, m.bias.grad
    return y, used, got


def _compare(tag, y, got, ref_y, ref_g, mod=None, wgt=None):
    """With `mod` and `wgt` (train mode): the dead channel's bias gradient is exactly 0 - its batch variance is 0 and
    the sum over the edges of s (g_e - dbeta/n) cancels - and an fp32 sum of terms of total size s * sum|g| leaves
    a rounding residue; it is held to 2^-20 of that size (a wrongly routed gradient is of size s * |g|)."""
    bu.assert_grads_close(tag + " output", y, ref_y)
    for name, want in ref_g.items():
        assert got[name] is not None, name
        g = got[name].detach().cpu().double()
        if name == "bias" and mod is not None:
            s = abs(float(mod.gconv.nn[2].weight.detach()[eu.DEAD])) / 1e-5 ** 0.5
            tol = 2.0 ** -20 * s * float(wgt[:, eu.DEAD].abs().sum())
            assert abs(float(g[eu.DEAD])) <= tol, (tag, float(g[eu.DEAD]), tol)
            live = torch.arange(g.numel()) != eu.DEAD
            g, want = g[live], want[live]
        bu.assert_grads_close("%s %s" % (tag, name), g, want)


@pytest.mark.parametrize("bias", ["on", "zero", "none"])
@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_dense_grads_exact(conv, act, train, bias):
    """Static and dynamic graph, BatchNorm scales {-1.5, -0.5, 0, 0.5, 1.25} and a dead channel: every gradient
    against fp64 autograd with no tie mask.  Padding points of a zero-bias layer sit on the kink (z == 0 on all
    their edges and channels)."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    a, slope = ACTS[act]
    B, C, co, N, k = len(DENSE_KINDS), 16, 24, 256, 9
    g = torch.Generator().manual_seed(5)
    x = eu.batch(DENSE_KINDS, C, N, seed=3).cuda()
    wgt = torch.randn(B, co, N, 1, generator=g)
    torch.manual_seed(0)
    mod = eu.set_params(D.DynConv2d(C, co, k, 1, conv, a, "batch", bias != "none"), bias, slope, seed=co)
    ei = eu.edge_index_of(eu.lex_knn(x, k))
    ref_y, ref_g = bu.oracle_grads(x, ei, mod.gconv.nn, conv, a, "batch", train, wgt)
    if bias != "on":
        z = bu._pre_activation(x, ei.cpu(), od.params_from_module(mod.gconv.nn, torch.float64), conv)
        assert bool((z == 0).any())
    mod = mod.cuda().train(train)
    for static in (True, False):
        y, used, got = _module_grads(mod, x, wgt.cuda(), ei if static else None)
        assert torch.equal(used, ei), "the kernel's graph is not the lexicographic one"
        _compare("%s %s" % (conv, "static" if static else "dynamic"), y, got, ref_y, ref_g,
                 *((mod, wgt) if train else ()))


@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_sync_batchnorm_one_rank(conv, monkeypatch):
    """DynConv2d with nn.SyncBatchNorm in training on one rank (the all-reduce is the identity): the synced
    statistics and backward take the same tie and kink rules."""
    import torch.distributed as dist
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    monkeypatch.setattr(dist, "all_reduce", lambda *a, **kw: None)
    monkeypatch.setattr(_native, "sync_group", lambda bn: object() if isinstance(bn, torch.nn.SyncBatchNorm) and
                        bn.training else None)
    B, C, co, N, k = len(DENSE_KINDS), 16, 24, 256, 9
    x = eu.batch(DENSE_KINDS, C, N, seed=4).cuda()
    wgt = torch.randn(B, co, N, 1, generator=torch.Generator().manual_seed(6))
    torch.manual_seed(0)
    mod = eu.set_params(D.DynConv2d(C, co, k, 1, conv, "leakyrelu", "batch", True), "zero", seed=1)
    ei = eu.edge_index_of(eu.lex_knn(x, k))
    ref_y, ref_g = bu.oracle_grads(x, ei, mod.gconv.nn, conv, "leakyrelu", "batch", True, wgt)
    mod = torch.nn.SyncBatchNorm.convert_sync_batchnorm(mod).cuda().train()
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in mod.modules())
    for static in (True, False):
        (y, used, got), names = _kernel_names(lambda: _module_grads(mod, x, wgt.cuda(), ei if static else None))
        assert any("bn_merge_kernel" in n for n in names), sorted(names)
        assert torch.equal(used, ei)
        _compare("sync %s %s" % (conv, "static" if static else "dynamic"), y, got, ref_y, ref_g, mod, wgt)


# ---- sparse GENConv ---------------------------------------------------------------------------------------------
def _sparse_graph(x, g):
    """x (N, C) integer features; edges in a fixed order: random edges, then a copy of the first 150 of them
    (parallel edges), then rows whose messages are all equal: from one all-negative source, from two sources with
    equal features, and from zero rows."""
    N = x.shape[0]
    src = torch.randint(0, N, (600,), generator=g)
    dst = torch.randint(0, N - 8, (600,), generator=g)
    src, dst = torch.cat((src, src[:150])), torch.cat((dst, dst[:150]))
    x[N - 1] = -torch.randint(1, 5, (x.shape[1],), generator=g).float()
    x[N - 2] = x[N - 3] = x[5]
    x[N - 4] = x[N - 5] = 0
    extra = [(N - 1, N - 8)] * 3 + [(N - 2, N - 7), (N - 3, N - 7), (N - 2, N - 7), (N - 4, N - 6), (N - 5, N - 6)]
    src = torch.cat((src, torch.tensor([s for s, _ in extra])))
    dst = torch.cat((dst, torch.tensor([t for _, t in extra])))
    return torch.stack((src, dst))


def _messages64(x64, x32, src):
    """The fp32 messages relu(x_j) + 1e-7 as the kernel rounds them, promoted to fp64 and differentiable in x:
    relu(x_j) is exact in both precisions, the rounded eps is added as a constant."""
    x_j = x32.index_select(0, src)
    off = ((F.relu(x_j) + 1e-7) - F.relu(x_j)).double()
    return F.relu(x64.index_select(0, src)) + off


def _scatter_max_first(msg, dst, N):
    """torch_scatter's scatter_max on the CPU: per (row, channel) the first edge in edge order that holds the
    maximum takes the value and the whole gradient; an empty row is 0."""
    E, C = msg.shape
    with torch.no_grad():
        top = osp._seg_max(msg, dst, N)
        eid = torch.arange(E).view(E, 1).expand(E, C)
        cand = torch.where(msg == top.index_select(0, dst), eid, torch.full_like(eid, E))
        first = torch.full((N, C), E, dtype=torch.int64).scatter_reduce(0, dst.view(E, 1).expand(E, C), cand, "amin")
    return torch.cat((msg, msg.new_zeros(1, C))).gather(0, first)


def _genconv_grads(mod, x, ei, wgt):
    mod = mod.cuda().train()
    xc = x.cuda().requires_grad_(True)
    h = mod.propagate(ei.cuda(), x=xc, msg_scale=None, residual=True)
    (h * wgt.cuda()).sum().backward()
    return h, xc.grad


def test_genconv_max_ties_route_to_first_edge():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(12)
    N, C = 96, 40
    x = torch.randint(-4, 5, (N, C), generator=g).float()
    ei = _sparse_graph(x, g)
    wgt = torch.randn(N, C, generator=g)
    x64 = x.double().requires_grad_(True)
    h_ref = x64 + _scatter_max_first(_messages64(x64, x, ei[0]), ei[1], N)
    (h_ref * wgt.double()).sum().backward()
    torch.manual_seed(1)
    h, gx = _genconv_grads(S.GENConv(C, C, aggr="max", mlp_layers=1, norm="layer"), x, ei, wgt)
    bu.assert_grads_close("max output", h, h_ref)
    bu.assert_grads_close("max x", gx, x64.grad)
    # the shim's even split of ties is a different subgradient: the fixture has ties that tell them apart
    x2 = x.double().requires_grad_(True)
    (osp.aggregate(_messages64(x2, x, ei[0]), ei[1], N, "max") * wgt.double()).sum().backward()
    assert not torch.allclose(x2.grad, x64.grad - wgt.double())


@pytest.mark.parametrize("aggr,p", [("power", 1.5), ("power_sum", 2.5)])
def test_genconv_power_clamp_bounds(aggr, p):
    """Messages up to 12: some exactly 10 (the clamp bound, where torch passes the gradient), some above (none),
    and rows whose mean of u^p is above the clamp; learnable p (and y)."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(13)
    N, C = 96, 40
    x = torch.randint(-4, 13, (N, C), generator=g).float()
    x[::7] = 10.0
    ei = _sparse_graph(x, g)
    x[N - 4] = x[N - 5] = 10.0                       # a row whose messages are all exactly 10
    wgt = torch.randn(N, C, generator=g)
    torch.manual_seed(1)
    kw = dict(y=-0.2, learn_y=True) if aggr == "power_sum" else {}
    mod = S.GENConv(C, C, aggr=aggr, p=p, learn_p=True, mlp_layers=1, norm="layer", **kw)
    ref = copy.deepcopy(mod).double()
    x64 = x.double().requires_grad_(True)
    msg = _messages64(x64, x, ei[0])
    assert bool((msg == 10).any()) and bool((msg > 10).any())
    h_ref = x64 + osp.aggregate(msg, ei[1], N, aggr, p=ref.p, y=getattr(ref, "y", 0.0))
    (h_ref * wgt.double()).sum().backward()
    h, gx = _genconv_grads(mod, x, ei, wgt)
    bu.assert_grads_close(aggr + " output", h, h_ref)
    bu.assert_grads_close(aggr + " x", gx, x64.grad)
    bu.assert_grads_close(aggr + " p", mod.p.grad, ref.p.grad, floor=1.0)
    if aggr == "power_sum":
        bu.assert_grads_close(aggr + " y", mod.y.grad, ref.y.grad, floor=1.0)
