"""The sparse GIN / GraphSAGE layers on the GPU (dgcn_gin_sage_aggregate and its backward, through GraphConv / DynConv
/ the blocks): the reference's outputs (goldens of tests/golden/gen_golden_gin_sage.py), bit-exact aggregates and
gradients on exact-arithmetic graphs, fp64 autograd on random graphs with hub rows, SyncBatchNorm in the MLP, the
shared CSR cache, and an arxiv-shaped graph."""
import copy

import pytest
import torch
import torch.nn.functional as F

import backward_util as bu
import gin_sage_util as gsu
import golden_util as gu
from deep_gcns_torch_b200 import _native
from deep_gcns_torch_b200.gcn_lib import sparse as S
from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import clear_csr_cache, csr_of

pytestmark = pytest.mark.gpu
RTOL, ATOL_FRAC = 1e-3, 1e-4
CONVS = ("gin", "sage", "rsage")


def close(got, ref, what, floor=0.0):
    bu.assert_grads_close(what, got, ref, atol_frac=ATOL_FRAC, rtol=RTOL, floor=floor)


def _sd(c, prefix):
    return {k[len(prefix) + 1:]: v for k, v in c.sd.items() if k.startswith(prefix + ".")}


# ---- the reference's outputs -------------------------------------------------------------------------------------
def test_graphconv_matches_reference():
    c = gu.load("spconv_gin_sage")
    m = c.meta
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    for name in m["cases"]:
        conv, act, norm = name.split("_")
        mod = S.GraphConv(m["C"], m["out"], conv, act, None if norm == "none" else "batch", True).cuda()
        mod.load_state_dict(_sd(c, name), strict=True)
        with torch.no_grad():
            if norm == "train":
                mod.train()
                y = mod(x, ei)
                mod(x, ei)
                bn = next(b for b in mod.modules() if isinstance(b, torch.nn.BatchNorm1d))
                close(bn.running_mean, c.outs["running_mean_" + name], name + " running_mean")
                close(bn.running_var, c.outs["running_var_" + name], name + " running_var")
            else:
                y = mod.eval()(x, ei)
        close(y, c.outs["y_" + name], name)


def test_blocks_and_dynconv_match_reference():
    c = gu.load("spconv_gin_sage_blocks")
    m = c.meta
    x, ei, batch = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda(), c.ins["batch"].long().cuda()
    C, k = m["C"], m["k"]
    for conv in m["convs"]:
        mods = {"res": S.ResGraphBlock(C, conv, "relu", "batch", True, res_scale=0.5),
                "dense": S.DenseGraphBlock(C, 4, conv, "leakyrelu", "batch", True),
                "dyn": S.DynConv(C, C, k, 1, conv, "relu", "batch", True)}
        for name, mod in mods.items():
            mod.cuda().eval().load_state_dict(_sd(c, "%s_%s" % (conv, name)), strict=True)
        with torch.no_grad():
            close(mods["res"](x, ei)[0], c.outs["y_%s_res" % conv], conv + " ResGraphBlock")
            close(mods["dense"](x, ei)[0], c.outs["y_%s_dense" % conv], conv + " DenseGraphBlock")
            graph = mods["dyn"].dilated_knn_graph(x, batch)
            ref_graph = c.outs["graph_dyn"].long()
            key = lambda g: sorted(zip(g[1].tolist(), g[0].tolist()))
            assert key(graph.cpu()) == key(ref_graph), "kNN graph differs from the reference's"
            close(mods["dyn"](x, batch), c.outs["y_%s_dyn" % conv], conv + " DynConv")


@pytest.mark.parametrize("conv", CONVS)
def test_ppi_deepgcn_matches_reference(conv):
    c = gu.load("spconv_ppi_" + conv)
    model = gsu.ppi_deepgcn(S, c.meta).cuda().eval()
    model.load_state_dict(c.sd, strict=True)
    with torch.no_grad():
        y = model(c.ins["x"].cuda(), c.ins["edge_index"].long().cuda())
    close(y, c.outs["y"], "PPI DeepGCN " + conv)


# ---- exact arithmetic ----------------------------------------------------------------------------------------------
def _ref_aggr(conv, x, ei, eps=0.0):
    return gsu.gin_aggr(x, ei, eps) if conv == "gin" else gsu.sage_aggr(x, ei, conv == "rsage")


@pytest.mark.parametrize("hub", [0, 1024])
@pytest.mark.parametrize("C", [3, 64, 130])
@pytest.mark.parametrize("conv", CONVS)
def test_exact_aggregate_and_gradient_bit_equal(conv, C, hub):
    """Integer features, c_i in {1, 2, 4, 8} (the hub row 1024), eps = 0.25: the aggregate, its gradient (upstream in
    quarters) and - below the hub row and C = 130, where the layer's partial sums could outgrow fp32's mantissa - the
    whole layer without norm (weights in eighths) equal fp64 bit for bit."""
    g = torch.Generator().manual_seed(C + hub)
    N = 203
    ei = gsu.exact_graph(N, g, hub).cuda()
    x = gsu.exact_features(N, C, g).cuda().requires_grad_(True)
    gout = (torch.randint(-4, 5, (N, C), generator=g).float() / 4).cuda()
    eps = torch.tensor([0.25], device="cuda")
    csr = csr_of(ei, N)
    assert (csr[3] is not None) == bool(hub)
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import _GinSageFn
    agg = _GinSageFn.apply(conv, csr, x, eps if conv == "gin" else None)
    x64 = x.detach().double().requires_grad_(True)
    ref = _ref_aggr(conv, x64, ei, 0.25)
    assert torch.equal(agg, ref.float()), (agg - ref.float()).abs().max()
    agg.backward(gout)
    ref.backward(gout.double())
    assert torch.equal(x.grad, x64.grad.float()), (x.grad - x64.grad.float()).abs().max()
    # the hub path against the one-warp path: the same bits on exact data
    if hub:
        assert torch.equal(_native.gin_sage_aggregate(conv, x, csr[:3], eps), agg)
    if hub or C > 64:
        return
    # the whole layer (norm None: no normalisation either)
    mod = S.GraphConv(C, 8, conv, "relu", None, True).cuda()
    with torch.no_grad():
        for p in mod.parameters():
            p.copy_(torch.randint(-8, 9, p.shape, generator=g).float() / 8)
        if conv == "gin":
            mod.gconv.eps.fill_(0.25)
    y = mod(x.detach(), ei)
    lay = mod.gconv
    with torch.no_grad():
        a = _ref_aggr(conv, x.detach().double(), ei, 0.25)
        nn64 = copy.deepcopy(lay.nn).double()
        if conv == "gin":
            y64 = nn64(a)
        else:
            y64 = nn64(torch.cat((x.detach().double(), a @ lay.weight.double()), 1)) + lay.bias.double()
    assert torch.equal(y, y64.float())


# ---- random graphs against fp64 autograd ------------------------------------------------------------------------------
def random_graph(N, E, g, hubs=(1100, 5000)):
    """E random edges over N nodes with self loops (every 9th edge) and duplicates (every 7th repeats its predecessor),
    plus rows 1 and 2 with `hubs` extra in-edges (self loops among them)."""
    src, dst = torch.randint(0, N, (E,), generator=g), torch.randint(0, N, (E,), generator=g)
    k = torch.arange(E)
    src = torch.where(k % 9 == 0, dst, src)
    src[1:] = torch.where(k[1:] % 7 == 0, src[:-1], src[1:])
    dst[1:] = torch.where(k[1:] % 7 == 0, dst[:-1], dst[1:])
    parts = [torch.stack((src, dst))]
    for row, n in zip((1, 2), hubs):
        s = torch.randint(0, N, (n,), generator=g)
        s[::50] = row
        parts.append(torch.stack((s, torch.full((n,), row))))
    ei = torch.cat(parts, 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)]


def reference_forward(mod, x64, ei, conv):
    """fp64 forward of GraphConv(conv) with leaves: the module's parameters copied to fp64."""
    lay = copy.deepcopy(mod.gconv).double()
    if conv == "gin":
        return lay.nn(_ref_aggr(conv, x64, ei, float(lay.eps))), lay
    out = lay.nn(torch.cat((x64, _ref_aggr(conv, x64, ei) @ lay.weight), 1))
    if lay.bias is not None:
        out = out + lay.bias
    return (F.normalize(out, p=2, dim=-1) if lay.normalize else out), lay


@pytest.mark.parametrize("train", [False, True])
@pytest.mark.parametrize("C", [1, 3, 33, 64, 128])
@pytest.mark.parametrize("conv", CONVS)
def test_random_graph_forward_and_gradients_against_fp64(conv, C, train):
    g = torch.Generator().manual_seed(7 * C + train)
    N = 1001                                            # N % 4 != 0
    ei = random_graph(N, 6 * N, g).cuda()
    mod = S.GraphConv(C, 24, conv, None, "batch", True).cuda()   # smooth: no activation kink to straddle
    with torch.no_grad():
        for b in mod.modules():
            if isinstance(b, torch.nn.BatchNorm1d):
                b.weight.uniform_(0.5, 1.5)
                b.bias.uniform_(-0.5, 0.5)
                b.running_mean.uniform_(-0.3, 0.3)
                b.running_var.uniform_(0.5, 1.5)
        if conv == "gin":
            mod.gconv.eps.fill_(0.125)
    mod.train(train)
    x = torch.randn(N, C, generator=g).cuda().requires_grad_(True)
    gout = torch.randn(N, 24, generator=g).cuda()
    y = mod(x, ei)
    y.backward(gout)
    x64 = x.detach().double().requires_grad_(True)
    y64, lay = reference_forward(mod, x64, ei, conv)
    y64.backward(gout.double())
    close(y, y64, "%s y" % conv)
    close(x.grad, x64.grad, "%s grad x" % conv)
    mine = dict(mod.gconv.named_parameters())
    ref_grads = dict(lay.named_parameters())
    scale = lambda key: float(ref_grads[key].grad.abs().max())
    for name, p in ref_grads.items():
        # train mode: the batch mean cancels the Linear's bias, whose gradient is 0 up to rounding - measured against
        # the scale of the weight's gradient instead of its own.  GIN with C = 1 feeds Linear(1, C_out): the batch
        # variance cancels each output channel's weight too, so both are measured against BatchNorm gamma's gradient.
        floor = 0.0
        if train and name.startswith("nn.0."):
            floor = scale("nn.1.weight") if (conv == "gin" and C == 1) else \
                (scale("nn.0.weight") if name == "nn.0.bias" else 0.0)
        close(mine[name].grad, p.grad, "%s grad %s" % (conv, name), floor)
    assert set(mine) >= {"nn.0.weight", "nn.0.bias", "nn.1.weight", "nn.1.bias"}


@pytest.mark.parametrize("C", [3, 64])
@pytest.mark.parametrize("conv", CONVS)
def test_hub_rows_with_and_without_the_hub_list(conv, C):
    """Rows of 1100 and 5000 edges: the segmented hub path and the one-warp path agree with fp64 and each other."""
    g = torch.Generator().manual_seed(C)
    N = 3001
    ei = random_graph(N, 4 * N, g).cuda()
    x = torch.randn(N, C, generator=g).cuda()
    eps = torch.tensor([0.5], device="cuda")
    csr = csr_of(ei, N)
    assert csr[3] is not None
    ref = _ref_aggr(conv, x.double(), ei, 0.5)
    with_hubs = _native.gin_sage_aggregate(conv, x, csr, eps)
    one_warp = _native.gin_sage_aggregate(conv, x, csr[:3], eps)
    close(with_hubs, ref, conv + " hub list")
    close(one_warp, ref, conv + " one warp per row")
    close(with_hubs, one_warp.double(), conv + " hub list vs one warp")


# ---- SyncBatchNorm, modules and the graph cache ------------------------------------------------------------------
@pytest.mark.parametrize("conv", CONVS)
def test_sync_batchnorm_without_process_group_gives_the_same_bits(conv):
    g = torch.Generator().manual_seed(3)
    N, C = 777, 16
    ei = random_graph(N, 5 * N, g, hubs=(1100, 30)).cuda()
    torch.manual_seed(0)
    plain = S.GraphConv(C, 32, conv, "relu", "batch", True).cuda().train()
    synced = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    assert any(isinstance(b, torch.nn.SyncBatchNorm) for b in synced.modules())
    x = torch.randn(N, C, generator=g).cuda()
    gout = torch.randn(N, 32, generator=g).cuda()
    outs = []
    for mod in (plain, synced):
        xi = x.clone().requires_grad_(True)
        y = mod(xi, ei)
        y.backward(gout)
        outs.append((y, xi.grad, {n: p.grad for n, p in mod.named_parameters()}))
    assert torch.equal(outs[0][0], outs[1][0])
    for n in outs[0][2]:
        assert torch.equal(outs[0][2][n], outs[1][2][n]), n
    close(outs[1][1], outs[0][1].double(), "grad x")     # atomics: the order of the additions varies


def test_dynconv_and_resdynblock_share_one_csr_build():
    g = torch.Generator().manual_seed(11)
    B, n, C = 4, 256, 32
    x = torch.rand(B * n, C, generator=g).cuda().requires_grad_(True)
    batch = torch.arange(B).repeat_interleave(n).cuda()
    dyn = S.DynConv(C, C, 9, 1, "sage", "relu", "batch", True).cuda()
    res = S.ResDynBlock(C, 9, 1, "rsage", "relu", "batch", True).cuda()
    ei = S.DilatedKnnGraph(9, 1)(x.detach(), batch)
    clear_csr_cache()
    _, first = bu.kernel_names(lambda: (clear_csr_cache(), dyn(x, batch, ei))[1])
    assert any("csr_init_kernel" in k for k in first), sorted(first)
    assert any("genconv_aggregate_kernel" in k for k in first), sorted(first)
    (y, _), second = bu.kernel_names(lambda: res(x, batch, ei))
    assert not any("csr_" in k for k in second), sorted(second)
    assert any("genconv_aggregate_kernel" in k for k in second), sorted(second)
    # and both are the layers they claim to be: kNN graph + RSAGEConv + x
    with torch.no_grad():
        ref, _ = reference_forward(res.body, x.detach().double(), ei, "rsage")
        close(y, ref + x.detach().double(), "ResDynBlock(rsage)")
    y.sum().backward()
    assert torch.isfinite(x.grad).all()


def test_sage_with_size_skips_the_self_loop_rewrite():
    g = torch.Generator().manual_seed(4)
    N, C = 300, 8
    ei = random_graph(N, 4 * N, g, hubs=(20, 30)).cuda()
    x = torch.randn(N, C, generator=g).cuda()
    for relative in (False, True):
        lay = S.RSAGEConv(C, 8, "relu", None, True, relative).cuda()
        y = lay(x, ei, size=(N, N))
        x64 = x.double()
        src, dst = ei[0], ei[1]
        msg = x64[src] - (x64[dst] if relative else 0)
        s = torch.zeros_like(x64).index_add_(0, dst, msg)
        cnt = torch.bincount(dst, minlength=N).clamp(min=1).double().unsqueeze(1)
        l64 = copy.deepcopy(lay).double()
        ref = l64.nn(torch.cat((x64, (s / cnt) @ l64.weight), 1)) + l64.bias
        close(y, ref, "size given, relative=%s" % relative)


def test_dtype_and_edge_cases():
    ei = torch.tensor([[0, 1], [1, 0]]).cuda()
    for conv in CONVS:
        mod = S.GraphConv(4, 4, conv).cuda()
        with pytest.raises(RuntimeError, match="fp32"):
            mod(torch.randn(2, 4, device="cuda", dtype=torch.float64), ei)
        y = mod.eval()(torch.randn(5, 4, device="cuda"), torch.zeros((2, 0), dtype=torch.long, device="cuda"))
        assert y.shape == (5, 4) and torch.isfinite(y).all()


# ---- scale ---------------------------------------------------------------------------------------------------------------
def test_arxiv_shaped_graph_against_fp64_on_a_row_sample():
    """N = 169,343, ~2.5 M edges with power-law-ish in-degrees (hub rows included), C = 128: the aggregate of each
    rule and its gradient against fp64 on 4096 sampled rows."""
    g = torch.Generator().manual_seed(2)
    N, E, C = 169343, 2484941, 128
    dev = "cuda"
    dst = (torch.rand(E, generator=g) ** 3 * N).long()          # skewed: low ids collect thousands of edges
    src = torch.randint(0, N, (E,), generator=g)
    src[::97] = dst[::97]                                      # self loops
    ei = torch.stack((src, dst)).to(dev)
    x = torch.randn(N, C, generator=g).to(dev)
    gout = torch.randn(N, C, generator=g).to(dev)
    rows = torch.randperm(N, generator=g)[:4096].to(dev)
    rows = torch.cat((rows, torch.arange(8, device=dev)))       # the hubs
    csr = csr_of(ei, N)
    assert csr[3] is not None
    eps = torch.tensor([0.25], device=dev)
    x64 = x.double()
    for conv in CONVS:
        out = _native.gin_sage_aggregate(conv, x, csr, eps)
        ref = _ref_aggr(conv, x64, ei, 0.25)
        close(out[rows], ref[rows], conv + " forward")
        gx = _native.gin_sage_aggregate_backward(conv, gout, csr, eps)
        xr = x64.clone().requires_grad_(True)
        _ref_aggr(conv, xr, ei, 0.25).backward(gout.double())
        close(gx[rows], xr.grad[rows], conv + " grad x")
        del ref, xr
