"""GENConv and the sparse-layout graph convolutions / blocks - API of the reference's
gcn_lib/sparse/torch_vertex.py (GENConv :12-88; MRConv :91-103; EdgConv :106-114; GraphConv :239-266; DynConv :267-281;
blocks :284-352)."""
import torch
from torch import nn

from ... import _native
from .._basic_conv import BasicConvLowering, update_running_stats
from .torch_nn import MLP, BondEncoder
from .torch_edge import DilatedKnnGraph
from .torch_message import GenMessagePassing, MsgNorm, _AggregateFn, csr_of

__all__ = ["GENConv", "MRConv", "EdgConv", "GraphConv", "DynConv", "PlainDynBlock", "ResDynBlock", "DenseDynBlock",
           "ResGraphBlock", "DenseGraphBlock"]


class GENConv(GenMessagePassing):
    """GENeralized graph convolution (softmax / power-mean aggregation).

    forward (torch_vertex.py:62-76): edge encoder -> [message + aggregate + MsgNorm
    + residual: ONE fused kernel over the cached CSR graph] -> MLP (torch)."""

    def __init__(self, in_dim, emb_dim, aggr="softmax", t=1.0, learn_t=False, p=1.0, learn_p=False,
                 y=0.0, learn_y=False, msg_norm=False, learn_msg_scale=True, encode_edge=False,
                 bond_encoder=False, edge_feat_dim=None, norm="batch", mlp_layers=2, eps=1e-7):
        super().__init__(aggr=aggr, t=t, learn_t=learn_t, p=p, learn_p=learn_p, y=y, learn_y=learn_y)
        channels = [in_dim] + [in_dim * 2] * (mlp_layers - 1) + [emb_dim]
        self.mlp = MLP(channels=channels, norm=norm, last_lin=True)
        self.msg_encoder = nn.ReLU()
        self.eps = eps
        self.encode_edge = encode_edge
        self.bond_encoder = bond_encoder
        self.msg_norm = MsgNorm(learn_msg_scale=learn_msg_scale) if msg_norm else None
        if self.encode_edge:
            if self.bond_encoder:
                self.edge_encoder = BondEncoder(emb_dim=in_dim)
            else:
                self.edge_encoder = nn.Linear(edge_feat_dim, in_dim)

    def forward(self, x, edge_index, edge_attr=None):
        if self.encode_edge and edge_attr is not None:
            edge_emb = self.edge_encoder(edge_attr)
        else:
            edge_emb = edge_attr
        scale = self.msg_norm.msg_scale if self.msg_norm is not None else None
        h = self.propagate(edge_index, x=x, edge_attr=edge_emb, msg_scale=scale, residual=True)
        if not torch.is_grad_enabled() and len(self.mlp) == 1 and isinstance(self.mlp[0], nn.Linear):
            lin = self.mlp[0]                      # inference, mlp_layers = 1: the Linear on the tensor cores
            if _native.linear_residual_supported(lin.in_features, lin.out_features) and h.data_ptr() % 16 == 0:
                return _native.linear_residual(h, lin.weight, lin.bias)
        return self.mlp(h)

    def message(self, x_j, edge_attr=None):
        """torch_vertex.py:78-85 (reference formula; the kernel fuses it)."""
        msg = x_j + edge_attr if edge_attr is not None else x_j
        return self.msg_encoder(msg) + self.eps

    def update(self, aggr_out):
        return aggr_out


class _RawAggr:
    """Carrier of the aggregator name for the autograd node (no parameters, no message transform)."""
    eps = 0.0

    def __init__(self, aggr):
        self.aggr = aggr

    def _check_aggr(self):
        return self.aggr


def _aggregate_rows(aggr, x, edge_index):
    """scatter_(aggr, x[src], dst) over the CSR-by-destination graph: the fused gather/reduce kernel on the raw
    source rows (empty rows -> 0, like torch_scatter)."""
    csr = csr_of(edge_index, x.size(0))
    return _AggregateFn.apply(_RawAggr(aggr), csr, True, False, x, None, 1.0, 1.0, 0.0, None), csr


class MRConv(nn.Module):
    """Max-Relative graph convolution, sparse layout (torch_vertex.py:91-103):
    nn(cat[x, scatter_(aggr, x_j - x_i, dst)]).  x_i is constant over a destination's edges and fp32 subtraction
    is monotone, so max_j fl(x_j - x_i) = fl(max_j x_j - x_i) bit for bit: the aggregation runs on the raw source
    rows in the CSR kernel and x_i is subtracted once per node ('add' / 'mean': sum_j x_j - deg * x_i, equal up to
    re-association)."""

    def __init__(self, in_channels, out_channels, act="relu", norm=None, bias=True, aggr="max"):
        super().__init__()
        self.nn = MLP([in_channels * 2, out_channels], act, norm, bias)
        self.aggr = aggr

    def forward(self, x, edge_index):
        if self.aggr not in ("add", "mean", "min", "max"):
            raise AssertionError(self.aggr)                      # utils/pyg_util.py:24
        if self.aggr == "min":
            m, csr = _aggregate_rows("max", -x, edge_index)
            m = -m
        else:
            m, csr = _aggregate_rows(self.aggr, x, edge_index)
        deg = (csr[0][1:] - csr[0][:-1]).to(x.dtype).unsqueeze(1)
        if self.aggr == "add":
            x_j = m - deg * x
        else:
            x_j = torch.where(deg > 0, m - x, torch.zeros_like(m))
        return self.nn(torch.cat([x, x_j], dim=1))


class _EdgeConvFn(torch.autograd.Function):
    """autograd node of EdgConv: dgcn_sparse_edge_conv_forward / _backward over the cached CSR graph."""

    @staticmethod
    def forward(ctx, owner, parts, csr, n_edges, x, weight, bias, prelu, bn_w, bn_b):
        prm = owner._conv_params(parts)
        out = _native.sparse_edge_conv_forward(x, csr, n_edges, prm)
        update_running_stats(parts[3], prm, n_edges)      # BatchNorm over the E edge rows
        ctx.prm, ctx.csr, ctx.n_edges = prm, csr, n_edges
        ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (x,) = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = _native.sparse_edge_conv_backward(x, ctx.csr, ctx.n_edges, ctx.prm, grad_out, need_x=need[4])
        pick = lambda i, key: g[key] if need[i] else None
        return (None, None, None, None, pick(4, "x"), pick(5, "weight"), pick(6, "bias"), pick(7, "prelu"),
                pick(8, "bn_weight"), pick(9, "bn_bias"))


class EdgConv(BasicConvLowering, nn.Module):
    """Edge convolution, sparse layout (torch_vertex.py:106-114, torch_geometric's EdgeConv around
    MLP([2*C_in, C_out], act, norm, bias): Linear -> norm -> act):
    out_i = max over edges (j -> i) of nn(cat[x_i, x_j - x_i]), 0 for a node without in-edges.  One CSR edge pass
    over the factorised Linear (z = P_i + Q_j, node-level GEMMs) keeps the max and min of z per node and channel;
    the BatchNorm runs over the E edge rows.  Gradient of the max: the first edge in edge_index order that attains
    it, as torch_scatter's scatter_max.  After nn.SyncBatchNorm.convert_sync_batchnorm, train-mode statistics are those
    of the edge rows of every rank in the BatchNorm's process group; the parameter gradients stay local."""

    def __init__(self, in_channels, out_channels, act="relu", norm=None, bias=True, aggr="max"):
        super().__init__()
        if aggr != "max":
            raise NotImplementedError("EdgConv aggr {}: the sparse-layout EdgeConv aggregates with 'max'".format(aggr))
        if norm is not None and str(norm).lower() not in ("none", "batch"):
            raise NotImplementedError("EdgConv norm {}: the sparse-layout EdgeConv covers None and 'batch'".format(norm))
        self.nn = MLP([in_channels * 2, out_channels], act, norm, bias)
        self.aggr = aggr

    def forward(self, x, edge_index):
        parts = self._parts()
        lin, act, prelu, bn = parts
        if isinstance(bn, nn.SyncBatchNorm) and not (x.is_cuda and edge_index.is_cuda):
            raise NotImplementedError("EdgConv: the sparse EdgeConv's SyncBatchNorm needs CUDA tensors")
        _native._require_cuda(x, edge_index)
        if x.dtype != torch.float32:
            raise RuntimeError("EdgConv computes in fp32, got %s features" % x.dtype)
        n_edges = int(edge_index.shape[1])
        # one edge row has no batch variance unless other ranks share the statistics (SyncBatchNorm's rule)
        if bn is not None and (self.training or bn.running_mean is None) and n_edges == 1 and \
                _native.sync_group(bn) is None:
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (torch.Size([1, lin.out_features]),))       # what BatchNorm1d raises
        csr = csr_of(edge_index, x.size(0))
        return _EdgeConvFn.apply(self, parts, csr, n_edges, x, lin.weight, lin.bias, prelu,
                                 None if bn is None else bn.weight, None if bn is None else bn.bias)


class GraphConv(nn.Module):
    """Static graph convolution, sparse layout (torch_vertex.py:239-266).  'edge' (EdgConv) and 'mr' (MRConv) run on
    the CSR kernels; the other variants are thin wrappers over third-party PyG convolutions in the reference
    (GATConv, GCNConv, GINConv, SAGEConv) and are not part of the rebuilt path."""

    def __init__(self, in_channels, out_channels, conv="edge", act="relu", norm=None, bias=True, heads=8):
        super().__init__()
        if conv.lower() == "edge":
            self.gconv = EdgConv(in_channels, out_channels, act, norm, bias)
        elif conv.lower() == "mr":
            self.gconv = MRConv(in_channels, out_channels, act, norm, bias)
        elif conv.lower() in ("gat", "gcn", "gin", "sage", "rsage"):
            raise NotImplementedError("conv {}: a torch_geometric layer in the reference; the sparse-layout path here "
                                      "covers 'edge' and 'mr'".format(conv))
        else:
            raise NotImplementedError("conv {} is not implemented".format(conv))

    def forward(self, x, edge_index):
        return self.gconv(x, edge_index)


class DynConv(GraphConv):
    """Dynamic graph convolution, sparse layout (torch_vertex.py:267-281): dilated kNN graph of the clouds in
    `batch` (dense selection kernels), then the static convolution."""

    def __init__(self, in_channels, out_channels, kernel_size=9, dilation=1, conv="edge", act="relu",
                 norm=None, bias=True, heads=8, **kwargs):
        super().__init__(in_channels, out_channels, conv, act, norm, bias, heads)
        self.k = kernel_size
        self.d = dilation
        self.dilated_knn_graph = DilatedKnnGraph(kernel_size, dilation, **kwargs)

    def forward(self, x, batch=None, edge_index=None):
        if edge_index is None:
            edge_index = self.dilated_knn_graph(x, batch)
        return super().forward(x, edge_index)


class PlainDynBlock(nn.Module):
    """torch_vertex.py:284-297."""

    def __init__(self, channels, kernel_size=9, dilation=1, conv="edge", act="relu", norm=None, bias=True,
                 res_scale=1, **kwargs):
        super().__init__()
        self.body = DynConv(channels, channels, kernel_size, dilation, conv, act, norm, bias, **kwargs)
        self.res_scale = res_scale

    def forward(self, x, batch=None, edge_index=None):
        return self.body(x, batch, edge_index), batch


class ResDynBlock(nn.Module):
    """torch_vertex.py:300-312."""

    def __init__(self, channels, kernel_size=9, dilation=1, conv="edge", act="relu", norm=None, bias=True,
                 res_scale=1, **kwargs):
        super().__init__()
        self.body = DynConv(channels, channels, kernel_size, dilation, conv, act, norm, bias, **kwargs)
        self.res_scale = res_scale

    def forward(self, x, batch=None, edge_index=None):
        return self.body(x, batch, edge_index) + x * self.res_scale, batch


class DenseDynBlock(nn.Module):
    """torch_vertex.py:315-326."""

    def __init__(self, in_channels, out_channels=64, kernel_size=9, dilation=1, conv="edge", act="relu", norm=None,
                 bias=True, **kwargs):
        super().__init__()
        self.body = DynConv(in_channels, out_channels, kernel_size, dilation, conv, act, norm, bias, **kwargs)

    def forward(self, x, batch=None, edge_index=None):
        dense = self.body(x, batch, edge_index)
        return torch.cat((x, dense), 1), batch


class ResGraphBlock(nn.Module):
    """torch_vertex.py:329-339."""

    def __init__(self, channels, conv="edge", act="relu", norm=None, bias=True, heads=8, res_scale=1):
        super().__init__()
        self.body = GraphConv(channels, channels, conv, act, norm, bias, heads)
        self.res_scale = res_scale

    def forward(self, x, edge_index):
        return self.body(x, edge_index) + x * self.res_scale, edge_index


class DenseGraphBlock(nn.Module):
    """torch_vertex.py:342-352."""

    def __init__(self, in_channels, out_channels, conv="edge", act="relu", norm=None, bias=True, heads=8):
        super().__init__()
        self.body = GraphConv(in_channels, out_channels, conv, act, norm, bias, heads)

    def forward(self, x, edge_index):
        dense = self.body(x, edge_index)
        return torch.cat((x, dense), 1), edge_index
