"""The sparse GENConv path at the ogbn-proteins and ogbn-products shapes against fp64: the loops that only a
production-size graph runs more than once.

proteins (132,534 nodes, ~80 M edges, C = 64; ogb_graph_util.proteins_graph): a fifth of the rows are hub rows
(degree >= HUB_MIN_DEGREE), so
- MODE 1 (one CTA per (hub row, segment), a grid of 4 x SMs CTAs) takes more items than its grid: CTAs loop to a
  second and later item;
- MODE 2 (one warp per hub row, 32 CTAs x 8 warps) has more than 256 rows: warps merge a second and later row;
- planted rows sit at the MODE 0 / hub boundary (1023, 1024 edges) and at segment boundaries (4095 .. 4097,
  8192, 8193), and one row of 10^6 edges is merged by one MODE 2 warp over 245 segments and walked by one warp in
  the backward;
and every aggregate instantiation that has the hub kernels runs on it: fp32, bf16, fp16, PRE and PRE + KEEP.

products (2,449,029 nodes, 61,859,140 uniform edges, C = 128): MODE 0 at full size, the backward at full size, and
the drop-in module's Linear (dgcn_linear_residual) over ~145 tiles per CTA.

fp64 references are taken on a compact subgraph (ogb_graph_util.compact_subgraph): a sample of destination rows,
their in-edges found on edge_index with torch.isin (not through the kernel's CSR) and those edges' sources.  Each
test prints its wall time and peak device memory.
"""
import copy
import time
import types

import pytest
import torch

import backward_util as bu
import ogb_graph_util as ogb
from oracle import sparse as osp
from test_sparse_backward_gpu import CFGS, _oracle_h

pytestmark = pytest.mark.gpu

MAX_PEAK = 12 * 2**30                 # the GPUs are shared: no test may hold more device memory than this
RTOL, ATOL = 2e-3, 2e-4               # fp32 against fp64 on rows of up to 10^6 edges (as test_power_law_graph_hub_rows)
HUB_RTOL, HUB_ATOL = 1e-4, 1e-5       # hub kernels against one warp per row, both fp32 ...
# ... on rows below this degree.  One warp sums a row's edges in one fp32 chain per lane: on the 10^6-edge row that
# chain drifts by up to 2.3e-4 of the aggregate from fp64 (softmax; 5.5e-5 for add / mean), while the hub kernels'
# 8 x 245 shorter chains stay within 2e-6 (H100, all nine aggregators).  With a hub list, as csr_build always
# makes one when a row reaches HUB_MIN_DEGREE, the forward never walks such a row on one warp; the
# one-warp call is held to fp64 on the sampled rows, the 10^6-edge row included, instead.
ONE_WARP_TIGHT_DEGREE = 10**5
PRE_RTOL, PRE_ATOL = 1e-5, 1e-6       # fused pre-activation against the rows materialised by torch
MODE1_CTAS_PER_SM, MODE2_WARPS = 4, 32 * 8   # sparse_aggr.cuh, launch_aggr: the hub kernels' grids


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _cfg_id(cfg):
    return cfg["aggr"] + ("_lt" if cfg.get("learn_t") else "") + ("_lp" if cfg.get("learn_p") else "")


@pytest.fixture(autouse=True)
def _time_and_peak(request):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("\n%s: %.2f s, peak %.2f GiB" % (request.node.name, time.perf_counter() - t0, peak / 2**30))
    assert peak <= MAX_PEAK, "%s held %.2f GiB of device memory" % (request.node.name, peak / 2**30)


def _graph(name, make, C, seed):
    """Everything the tests of one shape share: edge_index, the kernel's CSR (with its hub list), fp32 features,
    the sampled rows and their compact subgraph.  make() -> (edge_index, N, sampled rows, extra attributes)."""
    from deep_gcns_torch_b200 import _native
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    ei, N, rows, extra = make()
    csr = _native.csr_build(ei, N)
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, C, generator=g, device="cuda")
    rows = torch.unique(rows)
    nodes, ei_c, rows_c = ogb.compact_subgraph(ei, rows)
    deg = (csr[0][1:] - csr[0][:-1]).long()
    torch.cuda.synchronize()
    print("\n%s graph: N=%d E=%d, %d sampled rows, subgraph of %d nodes and %d edges: %.2f s, peak %.2f GiB" % (
        name, N, ei.shape[1], rows.numel(), nodes.numel(), ei_c.shape[1], time.perf_counter() - t0,
        torch.cuda.max_memory_allocated() / 2**30))
    return types.SimpleNamespace(name=name, ei=ei, N=N, C=C, csr=csr, deg=deg, x=x, rows=rows, nodes=nodes, ei_c=ei_c,
                                 rows_c=rows_c, **extra)


def _teardown():
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import clear_csr_cache
    clear_csr_cache()
    torch.cuda.empty_cache()


def _proteins():
    """The proteins-shaped graph and its sample: the planted and empty rows, rows 0 and N - 1, 128 ordinary hub
    rows and 128 rows below HUB_MIN_DEGREE, spread over the row range."""
    from deep_gcns_torch_b200 import _native
    ei, planted, empty = ogb.proteins_graph(seed=0)
    N = ogb.PROTEINS_N
    deg = torch.bincount(ei[1], minlength=N)
    special = torch.zeros(N, dtype=torch.bool, device="cuda")
    special[list(planted) + empty] = True
    hub = ((deg >= _native.HUB_MIN_DEGREE) & ~special).nonzero().squeeze(1)
    low = ((deg > 0) & (deg < _native.HUB_MIN_DEGREE) & ~special).nonzero().squeeze(1)
    pick = lambda v, k: v[torch.linspace(0, v.numel() - 1, k, device="cuda").long()]
    rows = torch.cat((torch.tensor(list(planted) + empty + [0, N - 1], device="cuda"), pick(hub, 128), pick(low, 128)))
    return ei, N, rows, dict(planted=planted, empty=empty)


def _products():
    """The products-shaped graph (ogb_graph_util.products_edges, also test_csr_build_is_stable_and_complete's) and
    every 9973rd row plus row N - 1."""
    N, _E = ogb.PRODUCTS
    rows = torch.cat((torch.arange(0, N, 9973, device="cuda"), torch.tensor([N - 1], device="cuda")))
    return ogb.products_edges(), N, rows, {}


@pytest.fixture(scope="module", params=["proteins", "products"])
def graph(request):
    """One shape's graph at a time (a test picks its shape by indirect parametrization; the tests are grouped by
    shape, and the proteins graph is released before the products graph is built)."""
    make, C, seed = {"proteins": (_proteins, 64, 1), "products": (_products, 128, 2)}[request.param]
    built = _graph(request.param, make, C, seed)
    yield built
    built.__dict__.clear()                # pytest still holds `built`: drop its tensors before emptying the cache
    _teardown()


PROTEINS = pytest.mark.parametrize("graph", ["proteins"], indirect=True)
PRODUCTS = pytest.mark.parametrize("graph", ["products"], indirect=True)


def _hub_table(csr):
    """(items (n_items, 2), rows (n_rows, 3)) of the CSR's hub work list, on the host."""
    items, hrows, counts, n_items = csr[3]
    counts = counts.cpu()
    assert int(counts[0]) == n_items
    return items[:2 * n_items].view(-1, 2).long().cpu(), hrows[:3 * int(counts[1])].view(-1, 3).long().cpu()


def _describe_row(graph, r, hubs):
    """Which kernel produced row r and in which round of its grid-stride loop (for a failure message)."""
    from deep_gcns_torch_b200 import _native
    d = int(graph.deg[r])
    if not hubs or graph.csr[3] is None or d < _native.HUB_MIN_DEGREE:
        return "row %d (degree %d, MODE 0)" % (r, d)
    _items, table = _hub_table(graph.csr)
    i = int((table[:, 0] == r).nonzero()[0, 0])
    first, nseg = int(table[i, 1]), int(table[i, 2])
    grid1 = MODE1_CTAS_PER_SM * _sms()
    return ("row %d (degree %d, %d segments, MODE 1 + 2: items %d..%d = MODE 1 rounds %d..%d of %d CTAs, hub row %d = "
            "MODE 2 round %d of %d warps)" % (r, d, nseg, first, first + nseg - 1, first // grid1,
                                              (first + nseg - 1) // grid1, grid1, i, i // MODE2_WARPS, MODE2_WARPS))


def _assert_rows(what, got, want, graph, rows=None, rtol=0.0, atol=0.0, hubs=True):
    """got, want: (R, C) values of destination rows `rows` (all rows when None); rtol = atol = 0: bit for bit.  A
    failure names the worst rows, their degree, segments and the kernel (and its loop round) that produced them."""
    if rtol == 0.0 and atol == 0.0:
        bad = (got != want).any(1)
    else:
        bad = ~torch.isclose(got, want, rtol=rtol, atol=atol).all(1)
    if not bool(bad.any()):
        return
    err = ((got - want).abs() / (atol + rtol * want.abs())).nan_to_num(float("inf")).amax(1)
    worst = [int(i) for i in torch.topk(torch.where(bad, err, torch.zeros_like(err)), min(5, int(bad.sum()))).indices]
    idx = rows if rows is not None else torch.arange(got.shape[0], device=got.device)
    lines = ["%s: max |got - want| = %.3g (got %.6g, want %.6g)" % (
        _describe_row(graph, int(idx[i]), hubs), float((got[i] - want[i]).abs().max()),
        float(got[i][(got[i] - want[i]).abs().argmax()]), float(want[i][(got[i] - want[i]).abs().argmax()]))
        for i in worst]
    raise AssertionError("%s on %s: %d of %d rows out of tolerance (rtol %g, atol %g)\n  %s" % (
        what, graph.name, int(bad.sum()), got.shape[0], rtol, atol, "\n  ".join(lines)))


def _scalars(cfg, msg_norm):
    return cfg.get("t", 1.0), cfg.get("p", 1.0), cfg.get("y", 0.0), (0.7 if msg_norm else None)


def _fp64_rows(graph, cfg, msg_norm, z=None):
    """osp.genconv_pre_mlp in fp64 on the sampled rows (z: the rows as the kernel reads them, default x)."""
    t, p, y, scale = _scalars(cfg, msg_norm)
    z = graph.x if z is None else z
    h = osp.genconv_pre_mlp(z[graph.nodes].double(), graph.ei_c, None, cfg["aggr"], t, p, y, scale, 1e-7)
    return h[graph.rows_c]


def _half_rows_bit_identical(graph, prm, what):
    """bf16 / fp16 rows read as they are give the bits of the fp32 call on the upcast rows (dgcn_genconv_aggregate's
    contract), hub kernels included."""
    from deep_gcns_torch_b200 import _native
    for dtype in (torch.bfloat16, torch.float16):
        xh = graph.x.to(dtype)
        got = _native.genconv_aggregate(xh, xh, graph.csr, prm)
        xf = xh.float()
        del xh
        want = _native.genconv_aggregate(xf, xf, graph.csr, prm)
        del xf
        _assert_rows("%s %s rows" % (what, dtype), got, want, graph)
        del got, want


@PROTEINS
def test_proteins_hub_work_list(graph):
    """The CSR's hub work list against a host recomputation from rowptr: every row of degree >= HUB_MIN_DEGREE once,
    with items (row, 0 .. nseg - 1) from its first item on, nseg = ceil(degree / HUB_SEG_EDGES), no other row.  The
    graph is large enough for both hub kernels to loop: more items than MODE 1's 4 x SMs CTAs, more hub rows than
    MODE 2's 256 warps, and sampled rows in the second and later rounds of both."""
    from deep_gcns_torch_b200 import _native
    g = graph
    rowptr = g.csr[0].long().cpu()
    deg = rowptr[1:] - rowptr[:-1]
    assert torch.equal(deg, torch.bincount(g.ei[1], minlength=g.N).cpu())
    for r, d in g.planted.items():
        assert int(deg[r]) == d, (r, d)
    assert all(int(deg[r]) == 0 for r in g.empty)
    items, table = _hub_table(g.csr)
    hub = (deg >= _native.HUB_MIN_DEGREE).nonzero().squeeze(1)
    grid1 = MODE1_CTAS_PER_SM * _sms()
    assert items.shape[0] > grid1 and table.shape[0] > MODE2_WARPS, (items.shape[0], table.shape[0])
    order = table[:, 0].argsort()
    t = table[order]
    assert torch.equal(t[:, 0], hub)                              # every hub row exactly once, nothing else
    nseg = (deg[hub] + _native.HUB_SEG_EDGES - 1) // _native.HUB_SEG_EDGES
    assert torch.equal(t[:, 2], nseg)
    assert int(nseg.sum()) == items.shape[0]
    seg = torch.arange(items.shape[0]) - torch.repeat_interleave(nseg.cumsum(0) - nseg, nseg)
    pos = torch.repeat_interleave(t[:, 1], nseg) + seg
    assert torch.equal(pos.sort().values, torch.arange(items.shape[0]))   # the rows' item ranges tile the list
    assert torch.equal(items[pos], torch.stack((torch.repeat_interleave(t[:, 0], nseg), seg), 1))
    assert int(nseg[(hub == 70001).nonzero()[0, 0]]) == 245
    # the sample reaches past the first round of both grid-stride loops
    sampled = torch.isin(table[:, 0], g.rows.cpu())
    assert int(sampled.sum()) >= 100
    where = sampled.nonzero().squeeze(1)
    assert bool((where >= MODE2_WARPS).any())
    assert bool((table[where, 1] + table[where, 2] > grid1).any())


def _aggregate_checks(graph, cfg, msg_norm, pre_variants):
    from deep_gcns_torch_b200 import _native
    t, p, y, scale = _scalars(cfg, msg_norm)
    prm, _keep = _native.genconv_params(cfg["aggr"], t, p, y, 1e-7, scale, add_residual=True)
    what = "%s msg_norm=%s" % (cfg["aggr"], msg_norm)
    out = _native.genconv_aggregate(graph.x, graph.x, graph.csr, prm)
    ref = _fp64_rows(graph, cfg, msg_norm).float()
    _assert_rows(what + " fp32 vs fp64", out[graph.rows], ref, graph, graph.rows, RTOL, ATOL)
    if graph.csr[3] is not None:              # the same call without the hub list: one warp per row
        one = _native.genconv_aggregate(graph.x, graph.x, graph.csr[:3], prm)
        _assert_rows(what + " one warp per row vs fp64", one[graph.rows], ref, graph, graph.rows, RTOL, ATOL, hubs=False)
        short = (graph.deg < ONE_WARP_TIGHT_DEGREE).nonzero().squeeze(1)
        _assert_rows(what + " hub kernels vs one warp per row", out[short], one[short], graph, short, HUB_RTOL, HUB_ATOL)
        del one
    del out
    _half_rows_bit_identical(graph, prm, what)
    if not pre_variants:
        return
    gen = torch.Generator(device="cuda").manual_seed(3)
    s = torch.rand(graph.C, generator=gen, device="cuda") + 0.5
    sh = torch.randn(graph.C, generator=gen, device="cuda") * 0.1
    z = torch.relu(graph.x * s + sh)
    got = _native.genconv_aggregate(graph.x, graph.x, graph.csr, prm, pre=(s, sh, True))
    _assert_rows(what + " PRE vs materialised rows", got, _native.genconv_aggregate(z, z, graph.csr, prm), graph,
                 None, PRE_RTOL, PRE_ATOL)
    drop = 0.2
    mask = torch.rand(graph.x.shape, generator=gen, device="cuda") >= drop
    keep = (_native.keep_bits(mask.float()), 1.0 / (1.0 - drop))
    got = _native.genconv_aggregate(graph.x, graph.x, graph.csr, prm, pre=(s, sh, True), keep=keep)
    zk = torch.where(mask, z * keep[1], torch.zeros_like(z))
    _assert_rows(what + " PRE+KEEP vs materialised rows", got, _native.genconv_aggregate(zk, zk, graph.csr, prm),
                 graph, None, PRE_RTOL, PRE_ATOL)
    _assert_rows(what + " PRE+KEEP fp32 vs fp64", got[graph.rows], _fp64_rows(graph, cfg, msg_norm, zk).float(), graph,
                 graph.rows, RTOL, ATOL)


def _backward_vs_fp64(graph, cfg):
    """GENConv.propagate(residual=True) under autograd with the upstream gradient non-zero only on the sampled rows
    D: every gradient then depends only on the edges into D, and fp64 autograd of the oracle on the compact subgraph
    (D and those edges' sources) gives all of them.  grad x of every node outside the subgraph must be exactly 0."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    N, C = graph.N, graph.C
    gen = torch.Generator(device="cuda").manual_seed(4)
    wgt = torch.zeros(N, C, device="cuda")
    wgt[graph.rows] = torch.randn(graph.rows.numel(), C, generator=gen, device="cuda")
    torch.manual_seed(1)
    mod = S.GENConv(C, C, mlp_layers=1, norm="layer", **cfg)
    if mod.msg_norm is not None:
        mod.msg_norm.msg_scale.data.fill_(0.7)
    ref = copy.deepcopy(mod).double().cuda()
    mod = mod.cuda().train()
    xk = graph.x.detach().requires_grad_(True)
    scale = mod.msg_norm.msg_scale if mod.msg_norm is not None else None
    h = mod.propagate(graph.ei, x=xk, msg_scale=scale, residual=True)
    h_rows = h.detach()[graph.rows]
    h.backward(wgt)
    del h
    xr = graph.x[graph.nodes].double().requires_grad_(True)
    hr = _oracle_h(ref, xr, graph.ei_c, graph.nodes.numel())
    (hr * wgt[graph.nodes].double()).sum().backward()
    tag = "%s %s" % (graph.name, _cfg_id(cfg))
    _assert_rows(tag + " forward", h_rows, hr.detach()[graph.rows_c].float(), graph, graph.rows, 1e-3, 1e-4)
    gx = xk.grad
    bu.assert_grads_close(tag + "/x", gx[graph.nodes], xr.grad)
    gx[graph.nodes] = 0
    outside = gx.abs().amax(1)
    assert not bool(outside.any()), "%s: grad x is non-zero at %d nodes outside the subgraph, e.g. node %d" % (
        tag, int((outside != 0).sum()), int(outside.argmax()))
    for name in ("t", "p", "y"):
        pr = getattr(ref, name, None)
        if torch.is_tensor(pr) and pr.requires_grad:
            bu.assert_grads_close("%s/%s" % (tag, name), getattr(mod, name).grad, pr.grad, floor=1.0)
    if ref.msg_norm is not None and ref.msg_norm.msg_scale.requires_grad:
        bu.assert_grads_close(tag + "/msg_scale", mod.msg_norm.msg_scale.grad, ref.msg_norm.msg_scale.grad, floor=1.0)


@PROTEINS
@pytest.mark.parametrize("msg_norm", [False, True], ids=["plain", "msgnorm"])
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_proteins_aggregate_hub_loops(graph, cfg, msg_norm):
    """Forward at the ogbn-proteins shape, where MODE 1 CTAs and MODE 2 warps loop over several work items: fp32
    against fp64 on the sampled rows (planted boundary rows, the 10^6-edge row, 128 ordinary hub rows, 128 short
    rows, empty rows, rows 0 and N - 1); the call without hubs (one warp per row) against fp64 on the same rows and
    against the hub kernels on every row below ONE_WARP_TIGHT_DEGREE; bf16 / fp16 rows bit for bit against fp32 on
    the upcast rows; PRE and PRE + KEEP against the plain call on the materialised rows."""
    _aggregate_checks(graph, cfg, msg_norm, pre_variants=True)


@PROTEINS
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_proteins_backward_vs_fp64(graph, cfg):
    """Backward at the ogbn-proteins shape: one warp per row walks every row, the 10^6-edge row included."""
    _backward_vs_fp64(graph, cfg)


@PRODUCTS
@pytest.mark.parametrize("msg_norm", [False, True], ids=["plain", "msgnorm"])
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_products_aggregate_full_size(graph, cfg, msg_norm):
    """Forward at the ogbn-products shape (MODE 0 over 2.4 M rows): fp32 against fp64 on every 9973rd row and row
    N - 1; bf16 / fp16 rows bit for bit against fp32 on the upcast rows."""
    _aggregate_checks(graph, cfg, msg_norm, pre_variants=False)


@PRODUCTS
@pytest.mark.parametrize("cfg", CFGS, ids=_cfg_id)
def test_products_backward_vs_fp64(graph, cfg):
    """Backward at the ogbn-products shape (2.4 M rows, gradients scattered over all of them)."""
    _backward_vs_fp64(graph, cfg)


@PRODUCTS
def test_products_genconv_module_row_linear(graph):
    """GENConv(128, 128, mlp_layers=1) at inference ends in dgcn_linear_residual (torch_vertex.py GENConv.forward):
    at the products shape its persistent CTAs take ~145 tiles each.  Against the fp64 oracle of the whole layer on
    the sampled rows."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = graph
    torch.manual_seed(5)
    conv = S.GENConv(g.C, g.C, mlp_layers=1).cuda().eval()
    assert -(-g.N // 128) > 2 * _sms()
    with torch.no_grad():
        y, names = bu.kernel_names(lambda: conv(g.x, g.ei))
    assert any("rowlinear_tc_kernel" in n for n in names), sorted(names)
    ref = osp.genconv_forward(conv, g.x[g.nodes], g.ei_c, dtype=torch.float64)[g.rows_c]
    _assert_rows("GENConv module", y[g.rows], ref.float(), g, g.rows, 1e-3, 1e-4)
