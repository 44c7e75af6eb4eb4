"""Shared pieces of the sparse GIN / GraphSAGE tests and of their golden generator (no GPU needed here):

- GINConvStandIn / SAGEConvStandIn / install_reference_stand_ins: torch_geometric's GINConv(nn, eps=0.,
  train_eps=False) and the older SAGEConv(in_channels, out_channels, normalize, bias) layout that the reference
  subclasses (gcn_lib/sparse/torch_vertex.py:136-205), restated over oracle/ref_shims.py's MessagePassing and put in
  place of ref_shims' placeholders before the reference is imported, so that the unmodified reference's GinConv,
  SAGEConv and RSAGEConv execute.  GINConv: out = nn(sum_{j->i} x_j + (1 + eps) x_i), the sum over edge_index as
  given, eps a buffer.  SAGEConv: weight (in, out) and bias (out) uniform in +-1/sqrt(in), mean aggregation,
  propagate handing x to update() as torch_geometric does.
- gin_aggr / sage_aggr: the aggregations restated functionally on any device and dtype (the fp64 references of the
  GPU tests): remove_self_loops + add_self_loops + mean for SAGE, exactly as torch_geometric composes them.
- exact_graph / exact_features: the exact-arithmetic fixtures of tests/test_gin_sage_gpu.py.
"""
import sys

import torch

from oracle import ref_shims


class GINConvStandIn(ref_shims.MessagePassing):
    """torch_geometric.nn.GINConv(nn, eps=0., train_eps=False)."""

    def __init__(self, nn, eps=0.0, train_eps=False, **kw):
        super().__init__(aggr="add", **kw)
        self.nn = nn
        self.initial_eps = eps
        if train_eps:
            self.eps = torch.nn.Parameter(torch.Tensor([eps]))
        else:
            self.register_buffer("eps", torch.Tensor([eps]))

    def forward(self, x, edge_index, size=None):
        out = self.propagate(edge_index, x=x, size=size)
        out = out + (1 + self.eps) * x
        return self.nn(out)


class SAGEConvStandIn(ref_shims.MessagePassing):
    """torch_geometric.nn.SAGEConv(in_channels, out_channels, normalize=False, bias=True) in the layout the
    reference's subclass reads (self.weight (in, out), self.bias, self.normalize); forward, message and update are
    the subclass's own."""

    def __init__(self, in_channels, out_channels, normalize=False, bias=True, **kw):
        super().__init__(aggr="mean", **kw)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.normalize = normalize
        self.weight = torch.nn.Parameter(torch.Tensor(in_channels, out_channels))
        if bias:
            self.bias = torch.nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        bound = 1.0 / in_channels ** 0.5
        for p in (self.weight, self.bias):
            if p is not None:
                p.data.uniform_(-bound, bound)

    def propagate(self, edge_index, size=None, x=None):
        n = x.size(0) if size is None else size[1]
        msg = self.message(x.index_select(0, edge_index[1]), x.index_select(0, edge_index[0]))
        return self.update(ref_shims.scatter(msg, edge_index[1], 0, dim_size=n, reduce="mean"), x)


def install_reference_stand_ins():
    """ref_shims' stand-in modules with GINConv and SAGEConv; call before ref_shims.load_reference()."""
    ref_shims._install_stubs()
    sys.modules["torch_geometric.nn"].GINConv = GINConvStandIn
    sys.modules["torch_geometric.nn"].SAGEConv = SAGEConvStandIn


def gin_aggr(x, edge_index, eps=0.0):
    """sum over every edge (j -> i) of x_j, plus (1 + eps) x_i, in x's dtype and on x's device."""
    src, dst = edge_index[0].long().to(x.device), edge_index[1].long().to(x.device)
    agg = torch.zeros_like(x).index_add_(0, dst, x.index_select(0, src))
    return agg + (1 + eps) * x


def sage_aggr(x, edge_index, relative=False):
    """remove_self_loops + add_self_loops, then the mean of x_j (x_j - x_i when relative) over each row's edges."""
    src, dst = edge_index[0].long().to(x.device), edge_index[1].long().to(x.device)
    keep = src != dst
    loop = torch.arange(x.shape[0], device=x.device)
    src, dst = torch.cat((src[keep], loop)), torch.cat((dst[keep], loop))
    msg = x.index_select(0, src) - (x.index_select(0, dst) if relative else 0)
    s = torch.zeros_like(x).index_add_(0, dst, msg)
    cnt = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return s / cnt.unsqueeze(1)


# ---- exact-arithmetic fixtures ----------------------------------------------------------------------------------
# Row kinds of exact_graph: (non-self in-degree, self loops on the row).  c_i = non-self + 1 is 1, 2, 4 or 8, so every
# mean is exact; one row carries several self loops, one row is empty, rows repeat a source (duplicate edges).
EXACT_ROWS = ((0, 0), (0, 1), (0, 3), (1, 0), (1, 1), (3, 0), (3, 2), (7, 0), (7, 1))


def exact_graph(N, g, hub=0):
    """(2, E) int64 over N nodes, in shuffled order: row r has EXACT_ROWS[r % 9] edges (random sources other than r,
    every third one repeating its predecessor, plus the self loops); with hub > 0 row N - 1 instead takes
    hub - 1 non-self edges and 2 self loops (hub - 1 + 1 a power of two keeps its mean exact)."""
    src, dst = [], []
    for r in range(N):
        n_other, n_self = EXACT_ROWS[r % len(EXACT_ROWS)]
        if hub and r == N - 1:
            n_other, n_self = hub - 1, 2
        s = torch.randint(0, N - 1, (n_other,), generator=g)
        s = s + (s >= r).long()                     # never r itself
        if n_other > 1:
            s[2::3] = s[1::3][:len(s[2::3])]        # duplicates
        s = torch.cat((s, torch.full((n_self,), r)))
        src.append(s)
        dst.append(torch.full((s.numel(),), r))
    ei = torch.stack((torch.cat(src), torch.cat(dst)))
    return ei[:, torch.randperm(ei.shape[1], generator=g)]


def exact_features(N, C, g):
    """(N, C) fp32 integers in [-4, 4]."""
    return torch.randint(-4, 5, (N, C), generator=g).float()


def sixteenths(shape, g):
    return torch.randint(-16, 17, shape, generator=g).float() / 16


def ppi_deepgcn(S, opt):
    """examples/ppi/architecture.py's DeepGCN (res or plain blocks) assembled from the drop-in sparse classes S, with
    its module layout (state_dict keys) and forward; the golden weights are loaded into it."""

    class DeepGCN(torch.nn.Module):
        def __init__(self):
            super().__init__()
            c, conv = opt["n_filters"], opt["conv"]
            args = (opt["act"], opt["norm"], opt["bias"], opt["n_heads"])
            self.n_blocks = opt["n_blocks"]
            self.head = S.GraphConv(opt["in_channels"], c, conv, *args)
            self.backbone = S.MultiSeq(*[S.ResGraphBlock(c, conv, *args, 1 if opt["block"] == "res" else 0)
                                         for _ in range(self.n_blocks - 1)])
            fusion_dims = c * self.n_blocks
            self.fusion_block = S.MLP([fusion_dims, 1024], opt["act"], None, opt["bias"])
            self.prediction = torch.nn.Sequential(
                S.MLP([1 + fusion_dims, 512], opt["act"], opt["norm"], opt["bias"]),
                torch.nn.Dropout(p=opt["dropout"]),
                S.MLP([512, 256], opt["act"], opt["norm"], opt["bias"]), torch.nn.Dropout(p=opt["dropout"]),
                S.MLP([256, opt["n_classes"]], None, None, opt["bias"]))

        def forward(self, x, edge_index):
            feats = [self.head(x, edge_index)]
            for i in range(self.n_blocks - 1):
                feats.append(self.backbone[i](feats[-1], edge_index)[0])
            feats = torch.cat(feats, 1)
            fusion, _ = torch.max(self.fusion_block(feats), 1, keepdim=True)
            return self.prediction(torch.cat((feats, fusion), 1))

    return DeepGCN()
