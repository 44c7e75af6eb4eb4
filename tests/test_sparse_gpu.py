"""GPU parity of the sparse path (CSR build, fused GENConv aggregate) against the
golden vectors of the unmodified reference and against oracle/ on seeded graphs."""
import pytest
import torch

import golden_util as gu
import ogb_graph_util as ogb
from oracle import sparse as osp

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def _genconv_from_golden(c):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    m = dict(c.meta)
    in_dim, emb_dim = m.pop("in_dim"), m.pop("emb_dim")
    m.pop("N")
    mod = S.GENConv(in_dim, emb_dim, **m)
    res = mod.load_state_dict(c.sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return mod.cuda().eval()


@pytest.mark.parametrize("name", gu.names("sparse_"))
def test_golden_genconv(name):
    c = gu.load(name)
    mod = _genconv_from_golden(c)
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    ea = c.ins["edge_attr"].cuda() if "edge_attr" in c.ins else None
    with torch.no_grad():
        y = mod(x, ei, ea)
        m = mod.propagate(ei, x=x, edge_attr=mod.edge_encoder(ea) if ea is not None else None)
    torch.testing.assert_close(m.cpu(), c.outs["m"], rtol=RTOL, atol=ATOL)
    torch.testing.assert_close(y.cpu(), c.outs["y"], rtol=RTOL, atol=ATOL)
    if name.endswith("_sum"):
        torch.testing.assert_close(mod.sigmoid_y.cpu(), torch.sigmoid(c.sd["y"]))


def _first_diff(got, want):
    i = int((got != want).nonzero()[0, 0])
    return "first difference at %d: got %d, want %d" % (i, int(got[i]), int(want[i]))


def test_csr_build_is_stable_and_complete():
    """dgcn_csr_build against a stable sort of the destinations on the device.  Besides small and empty graphs:
    - the ogbn-products shape (N = 2,449,029, E = 61,859,140): the radix histogram has 256 * ceil(E / RS_CHUNK)
      > 2^20 entries and rowptr N + 1 > 2^20, so scan_totals_kernel scans several 1024-block strips and carries
      between them (8 strips for the histogram, 3 for rowptr);
    - N = 2^24 + 5: destinations need 25 bits, so the sort makes 4 passes, N - 1 included."""
    from deep_gcns_torch_b200 import _native
    g = torch.Generator(device="cuda").manual_seed(0)
    for (n, e) in [(1, 5), (10, 0), (300, 3050), (70000, 200000), (5, 4099), ogb.PRODUCTS, (2**24 + 5, 4_000_000)]:
        if (n, e) == ogb.PRODUCTS:
            ei = ogb.products_edges()
            assert 256 * ogb.ceil_div(e, ogb.RS_CHUNK) > 2**20 and n + 1 > 2**20
        else:
            ei = torch.randint(0, n, (2, e), generator=g, device="cuda")
        if n > 2**24:
            ei[1, ::4001] = n - 1
            assert ogb.radix_passes(n) == 4 and int(ei[1].max()) == n - 1
        rowptr, src, eid = _native.csr_build(ei, n)[:3]
        order = torch.sort(ei[1], stable=True).indices
        what = "csr_build N=%d E=%d, " % (n, e)
        assert torch.equal(eid[:e].long(), order), what + "eid " + _first_diff(eid[:e].long(), order)
        want_src = ei[0][order]
        assert torch.equal(src[:e].long(), want_src), what + "src " + _first_diff(src[:e].long(), want_src)
        want_ptr = torch.cat((torch.zeros(1, dtype=torch.long, device="cuda"), torch.bincount(ei[1], minlength=n).cumsum(0)))
        assert torch.equal(rowptr.long(), want_ptr), what + "rowptr " + _first_diff(rowptr.long(), want_ptr)
        del ei, rowptr, src, eid, order, want_src, want_ptr
        torch.cuda.empty_cache()


AGGRS = ["softmax", "softmax_sg", "softmax_sum", "power", "power_sum", "add", "mean", "max"]


@pytest.mark.parametrize("C", [7, 32, 64, 128, 200, 256, 512])
@pytest.mark.parametrize("aggr", AGGRS)
def test_sweep_vs_oracle(C, aggr):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(C)
    N, E = 500, 6000
    dst = torch.randint(0, N - 30, (E,), generator=g)
    dst[:1500] = 3                                               # hub row, plus 30 empty rows
    ei = torch.stack((torch.randint(0, N, (E,), generator=g), dst))
    x = torch.randn(N, C, generator=g)
    torch.manual_seed(2)
    mod = S.GENConv(C, C, aggr=aggr, t=0.4, learn_t=True, p=2.5, learn_p=True, y=0.3, learn_y=True,
                    msg_norm=(C % 2 == 0), mlp_layers=1, norm="layer").eval()
    ref = osp.genconv_forward(mod, x, ei)
    ref64 = osp.genconv_forward(mod, x, ei, dtype=torch.float64).float()
    torch.testing.assert_close(ref, ref64, rtol=RTOL, atol=ATOL)
    mod = mod.cuda()
    with torch.no_grad():
        y = mod(x.cuda(), ei.cuda())
    torch.testing.assert_close(y.cpu(), ref, rtol=RTOL, atol=ATOL)


def test_aggregate_on_explicit_messages_and_empty_graph():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(5)
    msg = torch.rand(400, 24, generator=g) + 0.1
    index = torch.randint(0, 50, (400,), generator=g)
    for aggr in ("softmax", "power", "mean", "max"):
        mp = S.GenMessagePassing(aggr=aggr, t=0.8, p=2.0).cuda()
        got = mp.aggregate(msg.cuda(), index.cuda(), dim_size=60)
        ref = osp.aggregate(msg, index, 60, aggr, 0.8, 2.0)
        torch.testing.assert_close(got.cpu(), ref, rtol=RTOL, atol=ATOL)
    conv = S.GENConv(8, 8, aggr="softmax", mlp_layers=1, norm="layer").cuda().eval()
    x = torch.randn(20, 8).cuda()
    with torch.no_grad():
        y = conv(x, torch.zeros((2, 0), dtype=torch.long, device="cuda"))
        torch.testing.assert_close(y, conv.mlp(x))                # no edges: m = 0, h = x
    with pytest.raises(NotImplementedError):
        S.GENConv(8, 8, aggr="median").cuda()(x, torch.zeros((2, 4), dtype=torch.long, device="cuda"))


def test_arxiv_shape_properties():
    """c3-shaped graph (169,343 nodes, ~2.5 M edges, C=128): properties that need no
    full-size oracle, plus an oracle check restricted to a row sample."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(0)
    N, C = 169343, 128
    s, d = torch.randint(0, N, (1166243,), generator=g), torch.randint(0, N, (1166243,), generator=g)
    ei = osp.to_undirected_with_self_loops(s, d, N)
    x = torch.randn(N, C, generator=g)
    xc, eic = x.cuda(), ei.cuda()
    mp = S.GenMessagePassing(aggr="softmax_sg", t=0.1).cuda()
    mp.eps = 1e-7
    m1 = mp.propagate(eic, x=xc)
    perm = torch.randperm(ei.shape[1], generator=g)
    m2 = mp.propagate(ei[:, perm].cuda(), x=xc)                   # edge order must not matter
    torch.testing.assert_close(m1, m2, rtol=1e-4, atol=1e-5)
    assert torch.equal(m1, mp.propagate(eic, x=xc))               # run-to-run identical
    msg_max = S.GenMessagePassing(aggr="max").cuda()
    msg_mean = S.GenMessagePassing(aggr="mean").cuda()
    for q in (msg_max, msg_mean):
        q.eps = 1e-7
    mx, mn = msg_max.propagate(eic, x=xc), msg_mean.propagate(eic, x=xc)
    assert bool((m1 <= mx + 1e-5).all()) and bool((m1 >= mn - 1e-4).all())   # softmax(t>0) in [mean, max]
    add = S.GenMessagePassing(aggr="add").cuda()
    add.eps = 1e-7
    A = torch.sparse_coo_tensor(torch.stack((eic[1], eic[0])), torch.ones(ei.shape[1], device="cuda"), (N, N))
    torch.testing.assert_close(add.propagate(eic, x=xc), torch.sparse.mm(A, torch.relu(xc) + 1e-7),
                               rtol=1e-4, atol=1e-4)
    rows = torch.arange(0, N, 1009)                               # oracle on a row sample
    keep = torch.isin(ei[1], rows)
    sub = ei[:, keep]
    ref = osp.aggregate(osp.message(x, sub), sub[1], N, "softmax", 0.1)[rows]
    torch.testing.assert_close(m1.cpu()[rows], ref, rtol=RTOL, atol=ATOL)


def test_power_law_graph_hub_rows():
    """dst ~ Zipf: a few destinations collect tens of thousands of edges (SURVEY.md 8d load-balance
    stress).  Long rows take the CTA-per-row kernel; results must not depend on which kernel ran."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(0)
    N, E, C = 20000, 400000, 128
    u = torch.rand(E, generator=g).clamp_min(1e-9)
    dst = (u.pow(-1.0 / 0.5) - 1).clamp(max=N - 1).long()          # heavy tail: node 0..few are hubs
    ei = torch.stack((torch.randint(0, N, (E,), generator=g), dst))
    deg = torch.bincount(dst, minlength=N)
    assert int(deg.max()) > 20000 and int((deg >= _native.HUB_MIN_DEGREE).sum()) >= 3
    x = torch.randn(N, C, generator=g)
    for aggr in ("softmax", "softmax_sum", "power", "mean", "max"):
        torch.manual_seed(0)
        conv = S.GENConv(C, C, aggr=aggr, t=0.2, p=1.5, y=0.3, msg_norm=True, mlp_layers=1, norm="layer").eval()
        ref = osp.genconv_forward(conv, x, ei, dtype=torch.float64).float()
        conv = conv.cuda()
        with torch.no_grad():
            y = conv(x.cuda(), ei.cuda())
        torch.testing.assert_close(y.cpu(), ref, rtol=2e-3, atol=2e-4)
        csr = _native.csr_build(ei.cuda(), N)
        prm, keep = _native.genconv_params(aggr, 0.2, 1.5, 0.3, 1e-7, None, add_residual=False)
        with_hubs = _native.genconv_aggregate(x.cuda(), x.cuda(), csr, prm)
        no_hubs = _native.genconv_aggregate(x.cuda(), x.cuda(), csr[:3], prm)
        torch.testing.assert_close(with_hubs, no_hubs, rtol=1e-4, atol=1e-5)


def test_sparse_graph_builders_match_golden_and_oracle():
    """gcn_lib.sparse.torch_edge (knn='matrix'): flattened, globally numbered kNN graphs from the dense
    selection kernels - bit-exact against the reference's vectors up to fp32 near-ties (adjudicated
    in fp64), regular and stochastic dilation under the reference's RNG consumption."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from oracle import dense as od
    c = gu.load("spgraph_knn_matrix")
    x, batch = c.ins["x"], c.ins["batch"].long()
    n, B = c.meta["n"], c.meta["B"]
    xc, bc = x.cuda(), batch.cuda()

    def check(got, ref, k, xs, nb):
        assert got.shape == ref.shape and got.dtype == torch.int64
        assert torch.equal(got[1].cpu(), ref[1])
        npts = xs.shape[0] // nb
        xb = xs.reshape(nb, npts, -1).transpose(1, 2).unsqueeze(-1)
        off = torch.arange(0, nb * npts, npts).view(nb, 1, 1)
        n_bad, n_unexplained = od.knn_mismatch_report(xb, got[0].cpu().view(nb, npts, k) - off,
                                                      ref[0].view(nb, npts, k) - off)
        assert n_unexplained == 0 and n_bad <= 1e-3 * got[0].numel()

    check(S.knn_graph_matrix(xc, 9, bc), c.outs["knn_k9"].long(), 9, x, B)
    nn_idx, centre = S.knn_matrix(xc, 9, bc)
    assert nn_idx.shape == (1, B * n * 9) and torch.equal(centre[0].cpu(), c.outs["knn_k9"][1].long())
    # dilation happens inside the selection kernel: must equal striding the full list
    full = S.knn_graph_matrix(xc, 10, bc)
    got = S.DilatedKnnGraph(5, 2)(xc, bc)
    assert torch.equal(got, full[:, ::2])
    assert (got.cpu() == c.outs["dilated_k5_d2"].long()).float().mean() > 0.999
    single = S.DilatedKnnGraph(6, 3)(xc[:n], torch.zeros(n, dtype=torch.long, device="cuda"))
    assert (single.cpu() == c.outs["single_cloud_k6_d3"].long()).float().mean() > 0.999
    # stochastic dilation: same CPU generator draws, same random columns as the reference
    sto = S.DilatedKnnGraph(5, 3, True, 1.0).train()
    torch.manual_seed(11)
    got = sto(xc, bc)
    assert (got.cpu() == c.outs["stochastic_k5_d3_seed11"].long()).float().mean() > 0.999
    with pytest.raises(NotImplementedError):
        S.DilatedKnnGraph(5, 1, knn="cluster")


def test_partitioned_layer_emulated_on_one_gpu():
    """The node-partitioned layer without NCCL: two partitions live on the one GPU, the halo all-to-all is
    emulated by row copies, everything else is the product path - persistent [local | halo] buffers,
    interior / boundary row lists (split launches), hub rows, fused pre-activation.  Must equal the
    full-graph kernel bit for bit (same per-row edge order) and the oracle within tolerance."""
    from deep_gcns_torch_b200 import _native, partition as P
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(3)
    N, E, C, world = 5003, 90000, 128, 2
    ei = torch.randint(0, N, (2, E), generator=g)
    ei[1, :3000] = 11                                              # a hub row (>= 1024 edges) in partition 0
    low = ei[1] < 400                                              # rows 0..399 only hear from partition 0: interior rows
    ei[0, low] = ei[0, low] % (N // 2)
    x = torch.randn(N, C, generator=g).cuda()
    eic = ei.cuda()
    s = (torch.rand(C, generator=g) + 0.5).cuda()
    t = (torch.randn(C, generator=g) * 0.1).cuda()
    parts = [P.GraphPartition(eic, N, r, world) for r in range(world)]
    for aggr in ("softmax_sg", "power_sum", "mean"):
        conv = S.GENConv(C, C, aggr=aggr, t=0.3, p=1.5, y=0.2, msg_norm=True, mlp_layers=1).cuda().eval()
        tt, pp, yy = conv._scalars()
        prm, _k = _native.genconv_params(conv._check_aggr(), tt, pp, yy, conv.eps, conv.msg_norm.msg_scale, True)
        for pre in (None, (s, t, True)):
            z = x if pre is None else torch.relu(x * s + t)
            full = _native.genconv_aggregate(x, x, _native.csr_build(eic, N), prm, pre=pre)
            if pre is not None:      # fused pre-activation == aggregate of the materialised relu(s * x + t)
                torch.testing.assert_close(full, _native.genconv_aggregate(z, z, _native.csr_build(eic, N), prm),
                                           rtol=1e-5, atol=1e-6)
            ref = osp.genconv_pre_mlp(z.cpu(), ei, None, aggr, 0.3, 1.5, 0.2, float(conv.msg_norm.msg_scale), 1e-7)
            for part in parts:
                part.send_rows = torch.empty(0, dtype=torch.int32, device="cuda")     # no NCCL in this test
                xbuf, _send = part.buffers(C)
                xbuf[:part.n_local].copy_(x[part.lo:part.hi])
                xbuf[part.n_local:].copy_(x[part.halo_nodes])                          # the emulated exchange
                out = torch.full((part.n_local, C), float("nan"), device="cuda")
                _native.genconv_aggregate(xbuf, xbuf[:part.n_local], part.csr(), prm, out=out, pre=pre,
                                          rows=part.interior_rows, skip_hubs=True)
                _native.genconv_aggregate(xbuf, xbuf[:part.n_local], part.csr(), prm, out=out, pre=pre,
                                          rows=part.boundary_rows, skip_hubs=False)
                assert part.interior_rows.numel() + part.boundary_rows.numel() == part.n_local
                # same kernel, same per-row edge order: identical bits (the fused pre-activation is evaluated by the
                # same code on both sides: `full` above also goes through pre=)
                assert torch.equal(out, full[part.lo:part.hi]), (aggr, pre is not None, part.rank)
            torch.testing.assert_close(full.cpu(), ref, rtol=RTOL, atol=ATOL)
    assert parts[0].interior_rows.numel() > 0 and parts[0].boundary_rows.numel() > 0


@pytest.mark.parametrize("N,K,M", [
    (1000, 128, 128), (129, 64, 32), (5000, 256, 64), (3000, 64, 256), (128 * 150 + 7, 128, 64), (1, 64, 96),
    (20000, 256, 96),                     # at K = 256 the widest M whose W and A planes fit one SM's shared memory
    (5000, 128, 160), (5000, 64, 224),    # odd numbers of 32-column output blocks
    (132534, 64, 64),                     # ogbn-proteins' hidden width: ~8 tiles per CTA
    (169343, 128, 128),                   # ogbn-arxiv: ~10 tiles per CTA
    (2449029, 128, 128),                  # ogbn-products: ~145 tiles per CTA
])
def test_row_linear_with_bias_and_skip(N, K, M):
    """dgcn_linear_residual (wgmma, two-plane bf16 split of both operands) against an fp64 Linear: the split
    leaves <= ~2^-16 * sum|a||w| of error, far inside the 1e-3 parity tolerance; bias / skip optional; rows beyond
    the last full 128-row tile; out aliasing res.  The OGB row counts run the persistent tile loop for 3 and more
    tiles per CTA, where the a_full / a_free mbarrier phases wrap around.  The fp64 reference is taken in row chunks."""
    from deep_gcns_torch_b200 import _native
    g = torch.Generator(device="cuda").manual_seed(N + K + M)
    a = torch.randn(N, K, generator=g, device="cuda") * 3
    w = torch.randn(M, K, generator=g, device="cuda") / K ** 0.5
    b = torch.randn(M, generator=g, device="cuda")
    h = torch.randn(N, M, generator=g, device="cuda")
    if N >= 100000:
        assert -(-N // 128) > 2 * torch.cuda.get_device_properties(0).multi_processor_count   # a third tile per CTA
    w64 = w.double()

    def check(out, bias, res, chunk=1 << 17):
        for lo in range(0, N, chunk):
            a64 = a[lo:lo + chunk].double()
            ref = a64 @ w64.t()
            mag = a64.abs() @ w64.abs().t()                            # sum_k |a||w| per output
            if bias is not None:
                ref = ref + bias.double()
            if res is not None:
                ref = ref + res[lo:lo + chunk].double()
            got = out[lo:lo + chunk]
            err = (got.double() - ref).abs()
            assert bool((err <= 4e-5 * mag + 1e-6 * ref.abs() + 1e-6).all()), (lo, float((err / (mag + 1e-9)).max()))
            torch.testing.assert_close(got, ref.float(), rtol=1e-3, atol=1e-4)

    for bias, res in ((b, h), (None, h), (b, None), (None, None)):
        check(_native.linear_residual(a, w, bias, res), bias, res)
    b_odd = torch.cat((torch.zeros(1, device="cuda"), b))[1:]            # bias at an odd float offset (4-byte aligned)
    check(_native.linear_residual(a, w, b_odd, h), b, h)
    buf = h.clone()
    _native.linear_residual(a, w, b, buf, out=buf)                     # in place on the skip tensor
    check(buf, b, h)
    assert not _native.linear_residual_supported(100, 128) and not _native.linear_residual_supported(128, 300)
    assert not _native.linear_residual_supported(256, 256)            # operands would not fit one SM's shared memory


def test_sparse_layout_mrconv_and_dyn_block_match_reference():
    """gcn_lib/sparse/torch_vertex.py:91-103 (MRConv, all aggregators, isolated nodes) and :300-312 (ResDynBlock
    over equally sized clouds) against the unmodified reference (golden spconv_mr), forward and backward."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    c = gu.load("spconv_mr")
    m = c.meta
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    for aggr in ("max", "add", "mean", "min"):
        conv = S.MRConv(m["C"], m["out"], "relu", "batch", True, aggr)
        conv.load_state_dict({k[len(aggr) + 1:]: v for k, v in c.sd.items() if k.startswith(aggr + ".")}, strict=True)
        conv = conv.cuda().eval()
        with torch.no_grad():
            y = conv(x, ei)
        torch.testing.assert_close(y.cpu(), c.outs["y_" + aggr], rtol=RTOL, atol=ATOL, msg=lambda s_, a=aggr: a + ": " + s_)
    blk = S.ResDynBlock(m["C"], m["k"], m["dilation"], "mr", "relu", "batch", True, res_scale=m["res_scale"])
    blk.load_state_dict({k[6:]: v for k, v in c.sd.items() if k.startswith("block.")}, strict=True)
    blk = blk.cuda().eval()
    xb, batch = c.ins["xb"].cuda(), c.ins["batch"].long().cuda()
    with torch.no_grad():
        yb, b2 = blk(xb, batch)
        eib = blk.body.dilated_knn_graph(xb, batch)
    assert b2 is batch
    same = (eib.cpu().view(2, -1, m["k"])[0].sort(-1).values ==
            c.outs["edge_index_block"].long().view(2, -1, m["k"])[0].sort(-1).values).all(-1)
    assert same.float().mean() > 0.99
    torch.testing.assert_close(yb.cpu()[same], c.outs["y_block"][same], rtol=RTOL, atol=ATOL)
    # gradients flow through the raw max aggregation (arg-max routing) like torch_scatter's scatter_max
    conv = S.MRConv(m["C"], m["out"], "relu", None, True, "max").cuda()
    xg = x.clone().requires_grad_(True)
    conv(xg, ei).sum().backward()
    xr = x.detach().cpu().double().requires_grad_(True)
    src, dst = ei.cpu()
    msg = xr[src] - xr[dst]
    agg = torch.zeros(m["N"], m["C"], dtype=torch.double).scatter_reduce(0, dst.view(-1, 1).expand(-1, m["C"]), msg, "amax",
                                                                         include_self=False)
    lin = conv.nn[0]
    torch.relu(torch.cat([xr, agg], 1) @ lin.weight.detach().cpu().double().t() + lin.bias.detach().cpu().double()).sum().backward()
    torch.testing.assert_close(xg.grad.cpu().double(), xr.grad, rtol=1e-3, atol=1e-4)
    with pytest.raises(NotImplementedError):
        S.GraphConv(8, 8, "gat")
