"""The sparse GIN / GraphSAGE layers without a GPU: constructor and state_dict layout against the reference's
(goldens of tests/golden/gen_golden_gin_sage.py), 'gat' / 'gcn' still refused, CPU tensors refused (no fallback),
and the premises of the exact fixtures of tests/test_gin_sage_gpu.py and tests/test_gin_sage_scale_gpu.py."""
import numpy as np
import pytest
import torch

import gin_sage_util as gsu
import golden_util as gu
from deep_gcns_torch_b200.gcn_lib import sparse as S


def _layout(mod):
    return [[k, list(v.shape)] for k, v in mod.state_dict().items()]


def test_graphconv_state_dict_matches_reference():
    c = gu.load("spconv_gin_sage")
    m = c.meta
    for name in m["cases"]:
        conv, act, norm = name.split("_")
        mod = S.GraphConv(m["C"], m["out"], conv, act, None if norm == "none" else "batch", True)
        assert _layout(mod) == m["state_dict"][name], name
        mod.load_state_dict({k[len(name) + 1:]: v for k, v in c.sd.items() if k.startswith(name + ".")}, strict=True)


def test_layer_classes_and_defaults():
    gin = S.GraphConv(5, 7, "gin").gconv
    assert isinstance(gin, S.GinConv) and gin.eps.shape == (1,) and float(gin.eps) == 0.0
    assert [k for k, _ in gin.state_dict().items()] == ["eps", "nn.0.weight", "nn.0.bias"]
    sage, rsage = S.GraphConv(5, 7, "sage").gconv, S.GraphConv(5, 7, "rsage", norm="batch", bias=False).gconv
    assert isinstance(sage, S.RSAGEConv) and not sage.relative and not sage.normalize
    assert isinstance(rsage, S.SAGEConv) and rsage.relative and rsage.normalize and rsage.bias is None
    assert sage.weight.shape == (5, 7) and sage.nn[0].weight.shape == (7, 12)
    bound = 1 / 5 ** 0.5
    assert float(sage.weight.abs().max()) <= bound and float(sage.bias.abs().max()) <= bound
    for cls in (S.DynConv, S.PlainDynBlock, S.ResDynBlock):
        assert isinstance((cls(6, kernel_size=3, conv="gin") if cls is not S.DynConv else cls(6, 6, 3, conv="gin")),
                          torch.nn.Module)
    assert isinstance(S.DenseDynBlock(6, 4, 3, conv="rsage").body.gconv, S.RSAGEConv)
    assert isinstance(S.DenseGraphBlock(6, 4, "sage").body.gconv, S.RSAGEConv)
    assert isinstance(S.ResGraphBlock(6, "gin").body.gconv, S.GinConv)


@pytest.mark.parametrize("conv", ["gin", "sage", "rsage"])
def test_ppi_model_state_dict_matches_reference(conv):
    c = gu.load("spconv_ppi_" + conv)
    model = gsu.ppi_deepgcn(S, c.meta)
    assert _layout(model) == c.meta["state_dict"]
    model.load_state_dict(c.sd, strict=True)


@pytest.mark.parametrize("conv", ["gat", "gcn", "GAT", "other"])
def test_unsupported_convs_still_raise(conv):
    with pytest.raises(NotImplementedError):
        S.GraphConv(8, 8, conv)
    with pytest.raises(NotImplementedError):
        S.DynConv(8, 8, 3, conv=conv)


@pytest.mark.parametrize("conv", ["gin", "sage", "rsage"])
def test_cpu_tensors_raise(conv):
    mod = S.GraphConv(4, 4, conv)
    with pytest.raises(RuntimeError, match="CUDA"):
        mod(torch.randn(5, 4), torch.zeros((2, 3), dtype=torch.long))


@pytest.mark.parametrize("hub", [0, 1024])
def test_exact_fixture_premises(hub):
    """Every row's c_i is 1, 2, 4 or 8 (the hub row 1024); the graph has an empty row, rows with one and with several
    self loops, and duplicate edges; the fp32 aggregates on the CPU equal the fp64 ones."""
    g = torch.Generator().manual_seed(5)
    N = 61
    ei = gsu.exact_graph(N, g, hub)
    src, dst = ei
    other = torch.zeros(N, dtype=torch.long).index_add_(0, dst[src != dst], torch.ones_like(dst[src != dst]))
    loops = torch.zeros(N, dtype=torch.long).index_add_(0, dst[src == dst], torch.ones_like(dst[src == dst]))
    allowed = {1, 2, 4, 8} | ({hub} if hub else set())
    assert set((other + 1).tolist()) <= allowed and {1, 2, 4, 8} <= set((other + 1).tolist())
    indeg = torch.bincount(dst, minlength=N)
    assert (indeg == 0).any() and (loops == 1).any() and (loops >= 2).any()
    pairs = ei.t().tolist()
    assert len(set(map(tuple, pairs))) < len(pairs)             # duplicate edges
    x = gsu.exact_features(N, 5, g)
    assert x.abs().max() <= 4 and torch.equal(x, x.round())
    for relative in (False, True):
        assert torch.equal(gsu.sage_aggr(x, ei, relative), gsu.sage_aggr(x.double(), ei, relative).float())
    assert torch.equal(gsu.gin_aggr(x, ei, 0.25), gsu.gin_aggr(x.double(), ei, 0.25).float())


# ---- premises of tests/test_gin_sage_scale_gpu.py's exact fixtures ------------------------------------------------------
def test_fp32_quotient_of_integers_is_the_rounded_fp64_quotient():
    """The SAGE kernels divide an exact integer numerator |a| < 2^22 by c <= 2^20 with one correctly rounded fp32
    division: that equals the fp64 quotient rounded to fp32 (double rounding is innocuous for division, 53 >= 2 * 24 +
    2), so the fp64 reference gives the kernel's bits.  Numerator and divisor uniform, and c a power of two or c - 1."""
    rng = np.random.default_rng(0)
    n = 4_000_000
    a = rng.integers(-(2**22) + 1, 2**22, n)
    c = rng.integers(1, 2**20 + 1, n)
    c[: n // 8] = 2 ** rng.integers(0, 21, n // 8)
    c[n // 8: n // 4] = np.maximum(2 ** rng.integers(1, 21, n // 8) - 1, 1)
    f32 = a.astype(np.float32) / c.astype(np.float32)
    f64 = (a.astype(np.float64) / c.astype(np.float64)).astype(np.float32)
    assert np.array_equal(f32, f64), int((f32 != f64).sum())


def test_backward_row_terms_are_exact_under_the_fixture_rule():
    """The backward's row terms with g_i = c_i k_i / 4, |k_i| <= 4 (SAGE, RSAGE): fl(g_i / c_i) = k_i / 4 for every
    c_i <= 2^20, and RSAGE's fl(fl(-(c_i - 1) g_i) / c_i) = -(c_i - 1) k_i / 4 for c_i <= 2048 and for every power of
    two up to 2^20 - the rows whose k_i the fixture keeps.  Past 2048 the product rounds for some c_i and k_i, so the
    rule is needed."""
    c = np.arange(1, 2**20 + 1, dtype=np.int64)[:, None]
    k = np.arange(-4, 5, dtype=np.int64)[None, :]
    cf = c.astype(np.float32)
    g = (c * k).astype(np.float32) / np.float32(4)               # exact: |c k| <= 2^22
    assert np.array_equal(g.astype(np.float64) * 4, (c * k).astype(np.float64))
    assert np.array_equal(g / cf, np.broadcast_to(k.astype(np.float32) / 4, g.shape))
    row = (-(cf - 1) * g) / cf
    exact = row.astype(np.float64) == -((c - 1) * k).astype(np.float64) / 4
    kept = (c[:, 0] <= 2048) | ((c[:, 0] & (c[:, 0] - 1)) == 0)
    assert exact[kept].all()
    assert not exact[~kept].all()


def _analog_graph():
    """A CPU-size graph with the planted degrees of ogb_graph_util.proteins_graph (the 10^6-edge row included) and
    random rows of degree 0 .. 2000, uniform sources (so self loops drawn at random on every row), edges shuffled."""
    g = torch.Generator().manual_seed(8)
    N = 300
    deg = torch.randint(0, 2000, (N,), generator=g)
    planted = {0: 1024, 10: 1023, 20: 4095, 30: 4096, 40: 4097, 50: 10**6, 60: 8192, N - 1: 8193}
    for r, d in planted.items():
        deg[r] = d
    dst = torch.repeat_interleave(torch.arange(N), deg)
    src = torch.randint(0, N, (dst.numel(),), generator=g)           # self loops drawn at random too
    perm = torch.randperm(dst.numel(), generator=g)
    return torch.stack((src[perm], dst[perm])), N, planted


def test_planted_self_loops_land_where_the_recipe_says():
    """plant_self_loops on a CPU analog of the proteins graph, read back in the row order of a stable CSR build: the
    loop counts, c values and segment placement loop_positions states, all-loop rows with c = 1, about 1 / 97 of the
    remaining edges looped, and the fp32 bounds that keep the exact fixtures exact."""
    ei, N, planted = _analog_graph()
    assert int((ei[0, ei[1] == 50] == 50).sum()) > 1000
    small = [r for r in range(100, 110)]
    fixed = gsu.plant_self_loops(ei, planted, small)
    assert fixed == sorted([0, 10, 30, 40, 50, 60] + small)
    order = torch.sort(ei[1], stable=True).indices                # the CSR's order within each row
    src, dst = ei[0, order], ei[1, order]
    rowptr = torch.zeros(N + 1, dtype=torch.long)
    rowptr[1:] = torch.bincount(dst, minlength=N).cumsum(0)
    c = gsu.sage_counts(ei, N)

    def loops_of(r):
        return (src[rowptr[r]:rowptr[r + 1]] == r).nonzero().squeeze(1)

    assert torch.equal(loops_of(0), torch.arange(1024)) and float(c[0]) == 1      # the first hub row
    assert torch.equal(loops_of(10), torch.arange(1023)) and float(c[10]) == 1    # the last one-warp row
    assert torch.equal(loops_of(30), torch.arange(32)) and float(c[30]) == 4096 - 32 + 1
    assert torch.equal(loops_of(40), torch.tensor([4096])) and float(c[40]) == 4097
    l60 = loops_of(60)
    assert l60.numel() == 2048 and int(l60.min()) >= gsu.SEG_EDGES and float(c[60]) == 8192 - 2048 + 1
    big = loops_of(50)
    assert big.numel() == gsu.BIG_ROW_LOOPS > 2**16 and float(c[50]) == 2**19
    per_seg = torch.bincount(big // gsu.SEG_EDGES, minlength=245)
    assert per_seg.numel() == 245 and bool((per_seg > 0).all())                    # every segment, the short last one too
    assert bool((per_seg[:-1] >= 32).all())                                         # ... with a full 32-edge chunk's worth
    for r in small:
        assert loops_of(r).numel() == rowptr[r + 1] - rowptr[r] and float(c[r]) == 1
    for r in (20, N - 1):                                                           # planted degree, no recipe
        assert 0 < loops_of(r).numel() < (rowptr[r + 1] - rowptr[r]) // 40
    other = ~torch.isin(dst, torch.tensor(fixed))
    frac = float((src[other] == dst[other]).double().mean())
    assert abs(frac - (1 / 97 + 96 / 97 / N)) < 2e-3, frac                    # planted, and drawn at random
    fwd, bwd = gsu.exact_magnitudes(ei, N)
    assert fwd < 2**22 and bwd < 2**22, (fwd, bwd)
    assert fwd >= 4 * 10**6                                                         # the 10^6-edge row is the bound


def test_chunked_references_match_the_plain_ones():
    """The chunked fp64 forms (a small REF_CHUNK_BYTES so that the graph takes many chunks) against gin_aggr /
    sage_aggr and against autograd of them."""
    g = torch.Generator().manual_seed(9)
    N, C = 97, 5
    ei = gsu.exact_graph(N, g, 0)
    x = torch.randn(N, C, generator=g, dtype=torch.float64, requires_grad=True)
    gout = torch.randn(N, C, generator=g, dtype=torch.float64)
    saved = gsu.REF_CHUNK_BYTES
    gsu.REF_CHUNK_BYTES = 8 * C * 7
    try:
        for rule in ("gin", "sage", "rsage"):
            ref = gsu.gin_aggr(x, ei, 0.25) if rule == "gin" else gsu.sage_aggr(x, ei, rule == "rsage")
            got = gsu.gin_aggr_chunked(x.detach(), ei, 0.25) if rule == "gin" else \
                gsu.sage_aggr_chunked(x.detach(), ei, rule == "rsage")
            torch.testing.assert_close(got, ref.detach(), rtol=1e-12, atol=1e-12)
            gx, = torch.autograd.grad(ref, x, gout)
            torch.testing.assert_close(gsu.gin_sage_grad_chunked(rule, gout, ei, 0.25), gx, rtol=1e-12, atol=1e-12)
    finally:
        gsu.REF_CHUNK_BYTES = saved
