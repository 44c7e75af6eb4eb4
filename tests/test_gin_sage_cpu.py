"""The sparse GIN / GraphSAGE layers without a GPU: constructor and state_dict layout against the reference's
(goldens of tests/golden/gen_golden_gin_sage.py), 'gat' / 'gcn' still refused, CPU tensors refused (no fallback),
and the premises of the exact fixtures of tests/test_gin_sage_gpu.py."""
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
