"""GENConv and the sparse-layout graph convolutions / blocks - API of the reference's
gcn_lib/sparse/torch_vertex.py (GENConv :12-88; MRConv :91-103; EdgConv :106-114; SAGEConv / RSAGEConv :136-205;
GinConv :224-233; GraphConv :239-266; DynConv :267-281; blocks :284-352)."""
import math

import torch
import torch.nn.functional as F
from torch import nn

from ... import _native
from .._basic_conv import BasicConvLowering, update_running_stats
from .torch_nn import MLP, BondEncoder
from .torch_edge import DilatedKnnGraph
from .torch_message import GenMessagePassing, MsgNorm, _AggregateFn, _GinSageFn, csr_of

__all__ = ["GENConv", "MRConv", "EdgConv", "GinConv", "SAGEConv", "RSAGEConv", "GraphConv", "DynConv", "PlainDynBlock", "ResDynBlock", "DenseDynBlock",
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
    re-association).  Any C: past the kernels' widest launch the aggregation runs on channel slices (raw messages
    are channel-separable), with the bits of one launch."""

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
        deg = (csr[0][1:] - csr[0][:-1]).unsqueeze(1)
        if self.aggr == "add":
            # deg * x_i in fp32 (at least): in bf16 / fp16 the product of a hub row's degree keeps 8 / 11 bits, and
            # the subtraction from the fp32 sum m cancels most of it
            x_j = m - deg.to(torch.promote_types(x.dtype, torch.float32)) * x
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


def _cuda_rows_input(layer, x, edge_index):
    """GIN / GraphSAGE node features: fp32, or bf16 / fp16 (torch.autocast), which the aggregate reads as they are."""
    _native._require_cuda(x, edge_index)
    if x.dtype not in _native._ROW_DTYPE:
        raise RuntimeError("%s takes fp32, bf16 or fp16 features, got %s" % (layer, x.dtype))


class GinConv(nn.Module):
    """GIN, sparse layout (torch_vertex.py:224-233): torch_geometric's GINConv(MLP([C_in, C_out], act, norm, bias))
    with eps = 0, not trained (the buffer `eps`, shape [1]):
        out = nn(agg + (1 + eps) * x),   agg_i = sum over every edge (j -> i) of edge_index of x_j,
    self loops and duplicate edges counted as given, agg = 0 on a row without in-edges.  In fp32 the order is
    torch_geometric's: the sum first, then + (1 + eps) * x (one rounding for the product, one for the add).  The
    aggregation is one pass of the CSR kernel over the cached graph (dgcn_gin_sage_aggregate, forward and backward);
    the MLP stays torch, so a BatchNorm in it may be an nn.SyncBatchNorm.  `aggr` is accepted and unused, as in the
    reference.  CUDA tensors, fp32 or bf16 / fp16 features: half rows give the bits of their fp32 upcast and their
    gradient comes back in their own dtype (the fp32 gradient rounded once)."""

    def __init__(self, in_channels, out_channels, act="relu", norm=None, bias=True, aggr="add"):
        super().__init__()
        self.initial_eps = 0.0
        self.register_buffer("eps", torch.Tensor([self.initial_eps]))
        self.nn = MLP([in_channels, out_channels], act, norm, bias)

    def forward(self, x, edge_index):
        _cuda_rows_input("GinConv", x, edge_index)
        csr = csr_of(edge_index, x.size(0))
        return self.nn(_GinSageFn.apply("gin", csr, x, self.eps))


class SAGEConv(nn.Module):
    """GraphSAGE, sparse layout: the reference's SAGEConv (torch_vertex.py:136-189) on torch_geometric's older
    SAGEConv(C_in, C_out, normalize, bias) layout - `weight` (C_in, C_out), `bias` (C_out) when `bias`, both uniform
    in +-1/sqrt(C_in); normalize = norm is not None - with the reference's message and update:
        forward(x, edge_index, size=None): every self loop removed and one added per node (skipped when `size` is
          given, as in the reference), so row i's set is {j : (j -> i), j != i} + {i}, c_i = its size;
        message x_j W, or (x_j - x_i) W when `relative` (the added self loop's message is 0); mean over the set;
        out = nn(cat[x, aggr]) (+ bias), then F.normalize(out, p=2, dim=-1) when normalize.
    The message is linear, so the mean runs on the raw rows in the CSR kernel over the cached graph
    (dgcn_gin_sage_aggregate: (sum_{j != i} x_j + x_i) / c_i, relative (sum_{j != i} x_j - (c_i - 1) x_i) / c_i,
    equal to the reference up to re-association) and W, nn, bias and the normalisation stay torch.  With `size`,
    the mean over edge_index as given (an empty row gives 0).  CUDA tensors, fp32 or bf16 / fp16 features, as in
    GinConv."""

    def __init__(self, in_channels, out_channels, nn, norm=True, bias=True, relative=False, **kwargs):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.relative = relative
        self.normalize = norm is not None
        self.weight = torch.nn.Parameter(torch.Tensor(in_channels, out_channels))
        if bias:
            self.bias = torch.nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()
        self.nn = nn

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.in_channels)
        for p in (self.weight, self.bias):
            if p is not None:
                p.data.uniform_(-bound, bound)

    def forward(self, x, edge_index, size=None):
        x = x.unsqueeze(-1) if x.dim() == 1 else x
        _cuda_rows_input(type(self).__name__, x, edge_index)
        if size is None:
            csr = csr_of(edge_index, x.size(0))
            aggr = _GinSageFn.apply("rsage" if self.relative else "sage", csr, x, None)
        else:
            if tuple(size) != (x.size(0), x.size(0)):
                raise NotImplementedError("SAGEConv: size must be None or (N, N) with N = x.size(0), got %s"
                                          % (tuple(size),))
            aggr, csr = _aggregate_rows("mean", x, edge_index)
            if self.relative:
                deg = (csr[0][1:] - csr[0][:-1]).unsqueeze(1)
                aggr = torch.where(deg > 0, aggr - x, torch.zeros_like(aggr))
        out = self.nn(torch.cat((x, torch.matmul(aggr, self.weight)), dim=1))
        if self.bias is not None:
            out = out + self.bias
        if self.normalize:
            out = F.normalize(out, p=2, dim=-1)
        return out


class RSAGEConv(SAGEConv):
    """torch_vertex.py:192-205: SAGEConv with nn = MLP([C_out + C_in, C_out], act, norm, bias)."""

    def __init__(self, in_channels, out_channels, act="relu", norm=None, bias=True, relative=False):
        nn_ = MLP([out_channels + in_channels, out_channels], act, norm, bias)
        super().__init__(in_channels, out_channels, nn_, norm, bias, relative)


class GraphConv(nn.Module):
    """Static graph convolution, sparse layout (torch_vertex.py:239-266).  'edge' (EdgConv), 'mr' (MRConv), 'gin'
    (GinConv), 'sage' and 'rsage' (RSAGEConv, relative False / True) run on the CSR kernels.  'gat' and 'gcn' wrap
    torch_geometric's GATConv / GCNConv in the reference, whose attention, normalisation and state_dict layout changed
    across the torch_geometric versions its install can pick; they are not part of the rebuilt path.  `heads` is
    accepted and unused."""

    def __init__(self, in_channels, out_channels, conv="edge", act="relu", norm=None, bias=True, heads=8):
        super().__init__()
        if conv.lower() == "edge":
            self.gconv = EdgConv(in_channels, out_channels, act, norm, bias)
        elif conv.lower() == "mr":
            self.gconv = MRConv(in_channels, out_channels, act, norm, bias)
        elif conv.lower() == "gin":
            self.gconv = GinConv(in_channels, out_channels, act, norm, bias)
        elif conv.lower() == "sage":
            self.gconv = RSAGEConv(in_channels, out_channels, act, norm, bias, False)
        elif conv.lower() == "rsage":
            self.gconv = RSAGEConv(in_channels, out_channels, act, norm, bias, True)
        elif conv.lower() in ("gat", "gcn"):
            raise NotImplementedError("conv {}: a torch_geometric layer in the reference; the sparse-layout path here "
                                      "covers 'edge', 'mr', 'gin', 'sage' and 'rsage'".format(conv))
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
