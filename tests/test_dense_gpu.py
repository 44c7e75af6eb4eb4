"""GPU parity of the dense path (kNN graph, EdgeConv2d, MRConv2d, DynConv2d) against
the golden vectors of the unmodified reference and against oracle/ on seeded inputs.
Tolerance (BASELINE.json north_star): 1e-3 relative fp32 for features; kNN indices
exact except fp32 near-ties that the fp64 restatement adjudicates."""
import pytest
import torch

import golden_util as gu
from oracle import dense as od

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def _mod_from_golden(c, train=None):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    m = c.meta
    mod = D.DynConv2d(m["in_channels"], m["out_channels"], m["k"], m["dilation"], m["conv"], m["act"], m["norm"],
                      m["bias"])
    missing = mod.load_state_dict(c.sd, strict=True)
    assert not missing.missing_keys and not missing.unexpected_keys
    mod = mod.cuda()
    mod.train(m["training"] if train is None else train)
    return mod


def _adjudicate(x, mine, ref, max_frac=2e-3):
    n_bad, n_unexplained = od.knn_mismatch_report(x.cpu(), mine.cpu().long(), ref.cpu().long())
    assert n_unexplained == 0, "kNN index mismatch that is not an fp32 near-tie"
    assert n_bad <= max_frac * mine.numel()
    return n_bad


DYN = [n for n in gu.names("dense_") if "static" not in n and "grid" not in n]


@pytest.mark.parametrize("name", DYN)
def test_golden_dynconv(name):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    c = gu.load(name)
    m, x = c.meta, c.ins["x"].cuda()
    mod = _mod_from_golden(c)
    # 1. graph: dilated list and the full sorted K list
    with torch.no_grad():
        ei = mod.dilated_knn_graph(x)
        full = D.dense_knn_matrix(x, m["k"] * m["dilation"])
    assert ei.dtype == torch.int64 and tuple(ei.shape) == (2,) + tuple(c.outs["nn_idx"].shape)
    assert torch.equal(ei[1].cpu(), c.outs["center_idx"].long())
    _adjudicate(x, full[0], c.outs["nn_idx_full"])
    _adjudicate(x, ei[0], c.outs["nn_idx"])
    # 2. convolution on the reference's own graph
    gold_ei = torch.stack((c.outs["nn_idx"].long(), c.outs["center_idx"].long()), 0).cuda()
    sd_before = {k: v.clone() for k, v in mod.state_dict().items()}
    with torch.no_grad():
        y_static = D.GraphConv2d.forward(mod, x, gold_ei)
    torch.testing.assert_close(y_static.cpu(), c.outs["y"], rtol=RTOL, atol=ATOL)
    if m["training"]:
        bn = mod.gconv.nn[2]
        torch.testing.assert_close(bn.running_mean.cpu(), c.outs["running_mean"], rtol=RTOL, atol=1e-5)
        torch.testing.assert_close(bn.running_var.cpu(), c.outs["running_var"], rtol=RTOL, atol=1e-5)
        assert int(bn.num_batches_tracked) == int(c.outs["num_batches_tracked"])
        mod.load_state_dict(sd_before)
    # 3. fused dynamic path; rows whose neighbour set differs by an adjudicated near-tie are skipped
    with torch.no_grad():
        y_dyn = mod(x)
    same = (ei[0].cpu().sort(-1).values == c.outs["nn_idx"].long().sort(-1).values).all(-1)   # (B,N)
    assert same.float().mean() > 0.995
    if m["training"]:
        if bool(same.all()):
            torch.testing.assert_close(y_dyn.cpu(), c.outs["y"], rtol=RTOL, atol=ATOL)
    else:
        mask = same.unsqueeze(1).unsqueeze(-1).expand_as(c.outs["y"])
        torch.testing.assert_close(y_dyn.cpu()[mask], c.outs["y"][mask], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_golden_static_arbitrary_centres(conv):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    c = gu.load("dense_static_%s_arbitrary_centres" % conv)
    mod = D.GraphConv2d(10, 14, conv, "relu", "batch", True)
    mod.load_state_dict(c.sd, strict=True)
    mod = mod.cuda().eval()
    with torch.no_grad():
        y = mod(c.ins["x"].cuda(), c.ins["edge_index"].long().cuda())
    torch.testing.assert_close(y.cpu(), c.outs["y"], rtol=RTOL, atol=ATOL)


def test_grid_ties_bit_exact():
    """Exact-arithmetic cloud: every evaluation order gives identical fp32 distances, so
    the kernel must reproduce the (distance, index)-lexicographic order bit for bit."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    c = gu.load("dense_knn_grid_ties")
    x, dist = c.ins["x"], c.outs["dist"]
    N = dist.shape[-1]
    key = dist.double() * (64 * N) + torch.arange(N).double()     # distances are multiples of 1/64: exact
    expect = key.argsort(-1)
    for K in (1, 7, 32, 33, 64, 65, 100, 128):
        got = D.dense_knn_matrix(x.cuda(), K)[0].cpu()
        assert torch.equal(got, expect[..., :K]), K
        # and it agrees with the reference's list up to permutations inside exact ties
        gold = c.outs["nn_idx_full"].long()[..., :K]
        assert torch.equal(dist.gather(2, got), dist.gather(2, gold))


SWEEP = [
    # B, C, N, k, d, conv, act, norm, bias
    (1, 5, 77, 3, 2, "edge", "relu", "batch", True),
    (3, 20, 130, 7, 1, "mr", "leakyrelu", "batch", False),
    (2, 3, 1000, 9, 3, "edge", "prelu", None, True),
    (2, 33, 257, 16, 4, "edge", "relu", "batch", True),      # K = 64, vector loads off (N % 4 != 0)
    (2, 64, 512, 20, 5, "edge", "relu", "batch", True),      # K = 100 -> slab path
    (1, 16, 700, 20, 27, "mr", "relu", "batch", True),       # K = 540 -> slab path
    (2, 70, 384, 12, 1, "mr", "leakyrelu", None, True),
    (2, 96, 300, 8, 2, "edge", "relu", "batch", True),       # C_out 40 below
]


@pytest.mark.parametrize("cfg", SWEEP)
def test_sweep_vs_oracle(cfg):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B, C, N, k, d, conv, act, norm, bias = cfg
    g = torch.Generator().manual_seed(hash(cfg) % 1000)
    torch.manual_seed(1)
    co = 40 if C == 96 else 24
    mod = D.DynConv2d(C, co, k, d, conv, act, norm, bias)
    for m in mod.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data = torch.randn(co, generator=g) * 0.7 + 0.3
            m.bias.data = torch.randn(co, generator=g) * 0.2
            m.running_mean.data = torch.randn(co, generator=g) * 0.3
            m.running_var.data = torch.rand(co, generator=g) + 0.4
    x = torch.randn(B, C, N, 1, generator=g)
    p = od.params_from_module(mod.gconv.nn)
    ref_full = od.knn_matrix(x, k * d)
    ref_ei = ref_full[:, :, :, ::d]
    ref_y = od.graph_conv(x, ref_ei, p, conv, act, norm)
    mod = mod.cuda().eval()
    xc = x.cuda()
    with torch.no_grad():
        full = D.dense_knn_matrix(xc, k * d)
        ei = mod.dilated_knn_graph(xc)
        y_static = mod(xc, ref_ei.cuda())
        y_dyn = mod(xc)
    _adjudicate(x, full[0], ref_full[0])
    assert torch.equal(ei, full[:, :, :, ::d])
    torch.testing.assert_close(y_static.cpu(), ref_y, rtol=RTOL, atol=ATOL)
    same = (ei[0].cpu().sort(-1).values == ref_ei[0].sort(-1).values).all(-1)
    assert same.float().mean() > 0.99
    mask = same.unsqueeze(1).unsqueeze(-1).expand_as(ref_y)
    torch.testing.assert_close(y_dyn.cpu()[mask], ref_y[mask], rtol=RTOL, atol=ATOL)


def test_noncontiguous_slice_and_exclude_self():
    """inputs[:, 0:3] is what the model stacks feed the head graph builder
    (examples/sem_seg_dense/architecture.py:49); DilatedKnnGraph excludes self."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(3)
    inputs = torch.rand(2, 9, 640, 1, generator=g)
    pos = inputs[:, 0:3]
    ref = od.knn_matrix(pos.contiguous(), 20)
    got = D.DenseDilatedKnnGraph(20, 1)(inputs.cuda()[:, 0:3])
    _adjudicate(pos.contiguous(), got[0], ref[0])
    ref_x = od.knn_exclude_self(pos.contiguous(), 12)[:, :, :, ::3]
    got_x = D.DilatedKnnGraph(4, 3)(inputs.cuda()[:, 0:3])
    assert tuple(got_x.shape) == (2, 2, 640, 4)
    _adjudicate(pos.contiguous(), got_x[0], ref_x[0])
    assert not (got_x[0] == got_x[1]).any()


def test_stochastic_dilation_consumes_rng_like_reference():
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 8, 200, 1, generator=g)
    graph = D.DenseDilatedKnnGraph(5, 4, stochastic=True, epsilon=1.0).train()
    torch.manual_seed(9)
    got = graph(x.cuda())
    torch.manual_seed(9)
    ref = od.dilated_knn_graph(x, 5, 4, stochastic=True, epsilon=1.0, training=True)
    after_ref = torch.rand(1)
    torch.manual_seed(9)
    graph(x.cuda())
    assert torch.equal(torch.rand(1), after_ref)          # same number of host draws
    _adjudicate(x, got[0], ref[0])
    graph.eval()                                           # eval: regular dilation, still one draw
    torch.manual_seed(9)
    got_eval = graph(x.cuda())
    assert torch.equal(got_eval.cpu()[0], od.knn_matrix(x, 20)[0][:, :, ::4])


def test_errors_mirror_reference():
    from deep_gcns_torch_b200.gcn_lib import dense as D
    with pytest.raises(NotImplementedError):
        D.GraphConv2d(4, 4, conv="gat")
    with pytest.raises(RuntimeError):
        D.dense_knn_matrix(torch.randn(1, 4, 8, 1).cuda(), 9)      # k > N, torch.topk raises too
    with pytest.raises(RuntimeError):
        D.dense_knn_matrix(torch.randn(1, 4, 8, 1), 3)             # CPU tensor: no fallback


def test_headline_shape_properties():
    """BASELINE shape B=16 N=4096 k=20 C=64: size-independent properties + an oracle
    cross-check on two of the clouds (the oracle needs ~0.2 s per cloud)."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(0)
    torch.manual_seed(0)
    x = torch.randn(16, 64, 4096, 1, generator=g)
    mod = D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch", True).cuda().eval()
    xc = x.cuda()
    with torch.no_grad():
        ei = mod.dilated_knn_graph(xc)
        y1 = mod(xc)
        y2 = mod(xc)
        y_static = mod(xc, ei)
    assert torch.equal(y1, y2)                                   # deterministic / re-entrant
    assert torch.equal(y1, y_static)                             # fused == graph-then-conv
    nn_idx = ei[0]
    assert torch.equal(nn_idx[..., 0], torch.arange(4096, device="cuda").expand(16, -1))   # self first
    assert int(nn_idx.min()) >= 0 and int(nn_idx.max()) < 4096
    srt = nn_idx.sort(-1).values
    assert bool((srt[..., 1:] != srt[..., :-1]).all())           # no duplicate neighbours
    xt = xc.squeeze(-1).transpose(1, 2).double()                 # sortedness in fp64 on a row sample
    rows = torch.arange(0, 4096, 97, device="cuda")
    d = (xt[:, rows].unsqueeze(2) - xt.gather(1, nn_idx[:, rows].reshape(16, -1, 1).expand(-1, -1, 64))
         .view(16, rows.numel(), 20, 64)).pow(2).sum(-1)
    assert bool((d[..., 1:] - d[..., :-1] > -1e-3).all())
    # every one of the 16 clouds against the oracle (indices adjudicated, features on all rows whose
    # neighbour SET agrees; the number of masked rows is bounded by the counted near-ties)
    p = od.params_from_module(mod.gconv.nn)
    p = {k: (v.cpu() if torch.is_tensor(v) else {kk: vv.cpu() for kk, vv in v.items()}) for k, v in p.items()}
    y_cpu, nn_cpu = y1.cpu(), nn_idx.cpu()
    for b0 in range(0, 16, 4):
        sub = x[b0:b0 + 4]
        ref = od.knn_matrix(sub, 20)
        n_bad = _adjudicate(sub, nn_cpu[b0:b0 + 4], ref[0], max_frac=5e-4)
        ref_y = od.graph_conv(sub, ref, p, "edge", "relu", "batch")
        same = (nn_cpu[b0:b0 + 4].sort(-1).values == ref[0].sort(-1).values).all(-1)
        assert int((~same).sum()) <= n_bad                       # a row is masked only where a near-tie was counted
        mask = same.unsqueeze(1).unsqueeze(-1).expand_as(ref_y)
        torch.testing.assert_close(y_cpu[b0:b0 + 4][mask], ref_y[mask], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("k,d,conv", [(20, 5, "edge"), (20, 27, "edge"), (20, 8, "mr")])
def test_large_k_at_full_cloud_size_vs_oracle(k, d, conv):
    """K = k*d > 48 at N = 4096 (the 25 dilated layers of ResGCN-28, config 2): the large-K selection at the
    size where its slab tiling, sampled bound / retry and exact-fallback list are actually exercised; one cloud
    through the oracle (full sorted K list, dilated list, fused convolution)."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(k * d)
    torch.manual_seed(2)
    x = torch.randn(2, 64, 4096, 1, generator=g)
    mod = D.DynConv2d(64, 64, k, d, conv, "relu", "batch", True)
    p = od.params_from_module(mod.gconv.nn)
    mod = mod.cuda().eval()
    xc = x.cuda()
    with torch.no_grad():
        full = D.dense_knn_matrix(xc, k * d)
        ei = mod.dilated_knn_graph(xc)
        y = mod(xc)
    assert torch.equal(ei, full[:, :, :, ::d])
    ref_full = od.knn_matrix(x[:1], k * d)
    _adjudicate(x[:1], full[0][:1], ref_full[0], max_frac=1e-3)
    ref_ei = ref_full[:, :, :, ::d]
    ref_y = od.graph_conv(x[:1], ref_ei, p, conv, "relu", "batch")
    same = (ei[0][:1].cpu().sort(-1).values == ref_ei[0].sort(-1).values).all(-1)
    assert same.float().mean() > 0.99
    mask = same.unsqueeze(1).unsqueeze(-1).expand_as(ref_y)
    torch.testing.assert_close(y[:1].cpu()[mask], ref_y[mask], rtol=RTOL, atol=ATOL)
    # second cloud: size-independent properties (self first, no duplicates, ascending fp64 distances on a sample)
    nn2 = full[0][1]
    assert torch.equal(nn2[:, 0], torch.arange(4096, device="cuda"))
    srt = nn2.sort(-1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all())
    xt = xc[1].squeeze(-1).t().double()
    rows = torch.arange(0, 4096, 173, device="cuda")
    dd = (xt[rows].unsqueeze(1) - xt[nn2[rows]]).pow(2).sum(-1)
    assert bool((dd[:, 1:] - dd[:, :-1] > -1e-3).all())


@pytest.mark.parametrize("shape", [(2, 64, 1024, 20, 1), (2, 3, 512, 20, 1), (1, 32, 256, 9, 3), (3, 9, 384, 9, 2),
                                   (2, 48, 640, 4, 1), (1, 64, 128, 7, 4), (1, 17, 2048, 12, 1),
                                   (1, 16, 8192, 10, 1),      # N > 4096: unpacked (key, index) list entries
                                   (1, 8, 4224, 20, 2)])      # unpacked entries, K = 40 (list length 56)
def test_tensor_core_prefilter_equals_exact_fp32_path(shape):
    """The tensor-core pre-filter is certified + re-ranked in exact fp32, so its neighbour lists
    must be IDENTICAL (not just adjudicated-equal) to those of the pure fp32 FMA kernel."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B, C, N, k, d = shape
    g = torch.Generator().manual_seed(N + C)
    x = torch.randn(B, C, N, 1, generator=g).cuda()
    x[0, :, 5] = x[0, :, 9]                                   # exact duplicates: forces ties
    x[0, :, 17] = x[0, :, 9]
    graph = D.DenseDilatedKnnGraph(k, d)
    try:
        _native.set_knn_path("ffma")
        ref = graph(x)
        _native.set_knn_path("tc")
        got = graph(x)
        assert torch.equal(got, ref)
        torch.manual_seed(0)
        mod = D.DynConv2d(C, 24, k, d, "edge", "relu", "batch", True).cuda()
        for train in (False, True):
            mod.train(train)
            _native.set_knn_path("ffma")
            with torch.no_grad():
                y_ref = mod(x)
            _native.set_knn_path("tc")
            with torch.no_grad():
                y = mod(x)
            torch.testing.assert_close(y, y_ref, rtol=1e-5, atol=1e-6)
    finally:
        _native.set_knn_path("auto")


@pytest.mark.parametrize("path", ["tc", "tc1"])
def test_tensor_core_prefilter_certifies_random_clouds(path):
    """The exact completion kernel makes every answer right whatever the pre-filter certifies, so parity alone
    cannot see a pre-filter that certifies nothing: on random clouds at most 1e-3 of the queries may be left to
    it - set-only consumer (EdgeConv, eval), index output, and K = 40 (list of 56)."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(77)
    x = torch.randn(4, 64, 4096, 1, generator=g).cuda()
    torch.manual_seed(0)
    conv = D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch", True).cuda().eval()
    _native.set_knn_path(path)
    _native.tc_certification(True)
    try:
        _native.tc_certification_read()
        with torch.no_grad():
            conv(x)
            D.DenseDilatedKnnGraph(20, 1)(x)
            D.DenseDilatedKnnGraph(20, 2)(x)
        failed, queries = _native.tc_certification_read()
    finally:
        _native.tc_certification(False)
        _native.set_knn_path("auto")
    assert queries == 3 * 4 * 4096, queries
    assert failed <= 1e-3 * queries, (failed, queries)


@pytest.mark.parametrize("cfg", [
    # C, c_out, N, k, d, conv, act
    (32, 32, 256, 9, 1, "edge", "relu"),
    (64, 64, 512, 20, 2, "edge", "leakyrelu"),
    (16, 128, 384, 16, 1, "edge", "prelu"),
    (64, 24, 256, 12, 1, "mr", "relu"),
    (32, 40, 384, 20, 1, "mr", "relu"),
])
def test_wide_consumer_matches_generic_and_oracle(cfg):
    """Channel counts 32 / 64 / 128 take the float4 half-warp-per-query consumer of the tensor-core
    kernel (cta_epilogue_wide): same numbers as the generic consumer of the fp32 kernel and as the
    oracle, with negative BatchNorm scales (min branch), a negative PReLU slope (non-monotone
    activation) and train-mode batch statistics."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    C, co, N, k, d, conv, act = cfg
    g = torch.Generator().manual_seed(C * 1000 + co)
    torch.manual_seed(3)
    mod = D.DynConv2d(C, co, k, d, conv, act, "batch", True)
    for m in mod.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data = torch.randn(co, generator=g)              # about half negative
            m.bias.data = torch.randn(co, generator=g) * 0.2
            m.running_mean.data = torch.randn(co, generator=g) * 0.3
            m.running_var.data = torch.rand(co, generator=g) + 0.4
        if isinstance(m, torch.nn.PReLU):
            m.weight.data.fill_(-0.3)
    x = torch.randn(2, C, N, 1, generator=g)
    p = od.params_from_module(mod.gconv.nn)
    ref_ei = od.knn_matrix(x, k * d)[:, :, :, ::d]
    ref_y = od.graph_conv(x, ref_ei, p, conv, act, "batch")
    mod = mod.cuda()
    xc = x.cuda()
    try:
        for train in (False, True):
            mod.train(train)
            _native.set_knn_path("ffma")
            with torch.no_grad():
                y_ref = mod(xc)
            _native.set_knn_path("tc")
            with torch.no_grad():
                y = mod(xc)
            torch.testing.assert_close(y, y_ref, rtol=2e-5, atol=2e-6)
            if not train:
                ei = mod.dilated_knn_graph(xc)
                same = (ei[0].cpu().sort(-1).values == ref_ei[0].sort(-1).values).all(-1)
                assert same.float().mean() > 0.99
                mask = same.unsqueeze(1).unsqueeze(-1).expand_as(ref_y)
                torch.testing.assert_close(y.cpu()[mask], ref_y[mask], rtol=RTOL, atol=ATOL)
    finally:
        _native.set_knn_path("auto")


def test_tensor_core_prefilter_clustered_cloud_falls_back_exactly():
    """Many near-identical points defeat the certification margin: those queries must be
    completed by the exact kernel and still match the fp32 path bit for bit."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(7)
    centres = torch.randn(1, 16, 8, generator=g)
    x = centres[:, :, torch.randint(0, 8, (512,), generator=g)] + 1e-6 * torch.randn(1, 16, 512, generator=g)
    x = x.unsqueeze(-1).cuda()
    graph = D.DenseDilatedKnnGraph(20, 1)
    try:
        _native.set_knn_path("ffma")
        ref = graph(x)
        _native.set_knn_path("tc")
        got = graph(x)
    finally:
        _native.set_knn_path("auto")
    assert torch.equal(got, ref)


@pytest.mark.parametrize("cfg", [
    # C, N, k, d, conv, norm        (selection path)
    (64, 512, 20, 1, "edge", "batch"),      # tensor-core path, wide consumer
    (64, 512, 20, 4, "edge", "batch"),      # K = 80: slab path
    (24, 100, 5, 2, "edge", None),          # fp32 small path, generic consumer
    (32, 256, 9, 1, "mr", "batch"),         # MRConv: skip connection in the node kernel
    (64, 384, 16, 3, "mr", "batch"),
])
def test_block_epilogues_fused_into_the_consumer(cfg):
    """SURVEY.md 8f rank 1, dense: ResDynBlock2d's `+ x * res_scale` and the write into a channel slice of a wider
    buffer (DenseDynBlock2d's cat, a model's fusion buffer) happen in the consumer's store in inference.  Must give
    the bits of the unfused module sequence (conv, then x * scale, then the add)."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    C, N, k, d, conv, norm = cfg
    g = torch.Generator().manual_seed(C + N)
    torch.manual_seed(4)
    x = torch.randn(3, C, N, 1, generator=g).cuda()
    blk = D.ResDynBlock2d(C, k, d, conv, "relu", norm, True, res_scale=0.7).cuda().eval()
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data = torch.randn(C, generator=g).cuda()
            m.running_mean.data = (torch.randn(C, generator=g) * 0.3).cuda()
            m.running_var.data = (torch.rand(C, generator=g) + 0.4).cuda()
    with torch.enable_grad():                       # autograd on: the reference's module sequence, nothing fused
        ref = (blk.body(x) + x * blk.res_scale).detach()
    with torch.no_grad():
        got = blk(x)
        wide = torch.full((3, 3 * C, N, 1), float("nan"), device="cuda")
        wide[:, :C] = x
        ret = blk(wide[:, :C], out=wide[:, 2 * C:])            # strided input slice, strided output slice
    assert torch.equal(got, ref)
    assert ret.data_ptr() == wide[:, 2 * C:].data_ptr() and torch.equal(wide[:, 2 * C:], ref)
    assert torch.isnan(wide[:, C:2 * C]).all()                  # nothing outside the slice was touched
    dense_blk = D.DenseDynBlock2d(C, 32, k, d, conv, "relu", norm, True).cuda().eval()
    with torch.enable_grad():
        ref_cat = torch.cat((x, dense_blk.body(x)), 1).detach()
    with torch.no_grad():
        assert torch.equal(dense_blk(x), ref_cat)
    blk.train()                                     # train-mode BatchNorm: falls back to the module sequence
    if norm == "batch":
        with torch.no_grad():
            y_train = blk(x)
        assert y_train.shape == ref.shape and torch.isfinite(y_train).all()


@pytest.mark.parametrize("cfg", [
    # B, C, c_out, N, k, d, conv          (multi-tile kernel: C % 8 == 0, K <= 20, c_out in {32, 64, 128})
    (2, 64, 64, 4096, 20, 1, "edge"),     # the headline layer shape: 16 CTAs x 2 warpgroups per cloud
    (3, 64, 64, 1024, 10, 2, "edge"),     # dilation inside the kernel's rank selection (K = 20)
    (2, 32, 128, 640, 9, 1, "edge"),      # list of 16; 5 query tiles: the second CTA runs one warpgroup
    (1, 16, 32, 384, 16, 1, "edge"),      # 3 query tiles: one CTA with an idle warpgroup
    (2, 8, 64, 128, 20, 1, "edge"),       # a single query tile, two candidate half-tiles
    (2, 64, 24, 512, 12, 1, "mr"),        # MRConv consumer (c_in = 64)
    (1, 40, 64, 2048, 4, 1, "edge"),      # C = 40 -> three K=16 blocks of channels, zero padded
])
def test_four_tile_kernel_equals_tile_per_cta_and_fp32_paths(cfg):
    """knn_tc4_kernel (two query tiles per CTA, TMA producer warp + two filter warpgroups, sorting-network flush)
    must return the neighbour lists of knn_tc_kernel and of the pure fp32 kernel bit for bit, and the features
    of knn_tc_kernel bit for bit (same consumer code on the same lists)."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B, C, co, N, k, d, conv = cfg
    g = torch.Generator().manual_seed(N * 7 + C)
    x = torch.randn(B, C, N, 1, generator=g).cuda()
    x[0, :, 5] = x[0, :, 9]                                   # exact duplicates: forces ties
    x[0, :, 17] = x[0, :, 9]
    torch.manual_seed(1)
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


def test_four_tile_kernel_self_exclusion_clusters_and_block_fusion():
    """Same kernel: DilatedKnnGraph's self exclusion (applied in the exact re-rank), a clustered cloud whose
    queries cannot be certified (exact completion kernel), and the fused block epilogue (skip connection +
    channel-slice store) on top of it."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(11)
    x = torch.randn(2, 64, 512, 1, generator=g).cuda()
    centres = torch.randn(1, 16, 8, generator=g)
    xc = (centres[:, :, torch.randint(0, 8, (512,), generator=g)] + 1e-6 * torch.randn(1, 16, 512, generator=g))
    xc = xc.unsqueeze(-1).cuda()
    torch.manual_seed(2)
    blk = D.ResDynBlock2d(64, 20, 1, "edge", "relu", "batch", True, res_scale=0.7).cuda().eval()
    conv_c = D.DynConv2d(16, 32, 20, 1, "edge", "relu", "batch", True).cuda().eval()   # set-only membership path on
    got = {}                                                                            # the clustered cloud
    try:
        for path in ("ffma", "tc1", "tc"):
            _native.set_knn_path(path)
            with torch.no_grad():
                got[path] = (_native.knn_graph(x, 20, 1, exclude_self=True)[0], D.DenseDilatedKnnGraph(20, 1)(xc), blk(x),
                             conv_c(xc))
    finally:
        _native.set_knn_path("auto")
    for i in range(2):
        assert torch.equal(got["tc"][i], got["ffma"][i])
        assert torch.equal(got["tc"][i], got["tc1"][i])
    assert torch.equal(got["tc"][2], got["tc1"][2])
    assert torch.equal(got["tc"][3], got["tc1"][3])
    torch.testing.assert_close(got["tc"][3], got["ffma"][3], rtol=1e-5, atol=1e-6)
    assert not bool((got["tc"][0][0] == got["tc"][0][1]).any())          # no query lists itself
