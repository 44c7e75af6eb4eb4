"""Dense vertex ops - API of the reference's gcn_lib/dense/torch_vertex.py.

EdgeConv2d / MRConv2d read the tensors of their `nn` (a BasicConv, so state_dict
keys match the reference) and run gather + conv1x1 + act + norm + max in libdgcn;
DynConv2d additionally fuses the dilated kNN selection so that the neighbour list
never reaches HBM in inference.
"""
import torch
from torch import nn

from ... import _native
from .._basic_conv import BasicConvLowering, update_running_stats
from .torch_nn import BasicConv
from .torch_edge import DenseDilatedKnnGraph, DilatedKnnGraph

__all__ = ["MRConv2d", "EdgeConv2d", "GraphConv2d", "DynConv2d", "PlainDynBlock2d", "ResDynBlock2d",
           "DenseDynBlock2d"]


class _GraphConvFn(torch.autograd.Function):
    """autograd node around the fused forward; backward = dgcn_graph_conv_backward.  ctx.prm carries the
    SyncBatchNorm process group (prm.sync_group) to backward, whose all-reduce then runs in the same order on
    every rank."""

    @staticmethod
    def forward(ctx, owner, parts, x, edge_index, fused, *params):
        prm = owner._conv_params(parts)
        if fused is not None:                       # dynamic graph, built in the same launch sequence
            k, dilation, cols, need_graph = fused[:4]
            block = fused[4] if len(fused) > 4 else {}      # block epilogue (inference): residual / res_scale / out
            out, nbr = _native.dyn_conv_forward(owner._conv, x, prm, k, dilation, cols, want_nbr=need_graph, **block)
        else:
            k, nbr = edge_index.shape[-1], None
            out = _native.graph_conv_forward(owner._conv, x, prm, edge_index=edge_index)
        # EdgeConv normalises the B*N*k edge activations, MRConv the B*N node activations
        update_running_stats(parts[3], prm, x.shape[0] * x.shape[2] * (k if owner._conv == "edge" else 1))
        ctx.owner, ctx.prm, ctx.nbr, ctx.edge_index = owner, prm, nbr, edge_index
        ctx.save_for_backward(x)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        (x,) = ctx.saved_tensors
        need = ctx.needs_input_grad
        g = _native.graph_conv_backward(ctx.owner._conv, x, ctx.prm, grad_out, edge_index=ctx.edge_index, nbr=ctx.nbr,
                                        need_x=need[2])
        if g["x"] is not None:
            g["x"] = g["x"].view(x.shape[0], x.shape[1], x.shape[2], 1)
        g["weight"] = g["weight"].view_as(ctx.owner.nn[0].weight)
        pick = lambda i, key: g[key] if need[i] else None
        return (None, None, pick(2, "x"), None, None, pick(5, "weight"), pick(6, "bias"), pick(7, "prelu"),
                pick(8, "bn_weight"), pick(9, "bn_bias"))


class _DenseGraphConv(BasicConvLowering, nn.Module):
    """Shared plumbing of EdgeConv2d / MRConv2d."""
    _conv = None

    def __init__(self, in_channels, out_channels, act="relu", norm=None, bias=True):
        super().__init__()
        self.nn = BasicConv([in_channels * 2, out_channels], act, norm, bias)
        for m in self.nn:
            if isinstance(m, nn.InstanceNorm2d):      # unreachable in the reference as well
                raise NotImplementedError("normalization layer [instance] is not supported by the graph convs")

    def _run(self, x, edge_index, fused=None, block=None):
        parts = self._parts()
        conv, act, prelu, bn = parts
        params = (conv.weight, conv.bias, prelu, None if bn is None else bn.weight, None if bn is None else bn.bias)
        if fused is not None:
            # the graph is kept (int32 neighbour list) only when a backward pass can follow
            need = torch.is_grad_enabled() and (x.requires_grad or any(
                p is not None and p.requires_grad for p in params))
            fused = tuple(fused) + (need,) + ((block,) if block else ())
        return _GraphConvFn.apply(self, parts, x, edge_index, fused, *params)

    def can_fuse_block(self, x):
        """The block epilogue (skip connection / slice write in the consumer's store) runs without autograd and
        without train-mode BatchNorm statistics."""
        bn = self._parts()[3]
        return (not torch.is_grad_enabled() and x.is_cuda and x.dtype == torch.float32 and
                (bn is None or not (self.training or bn.running_mean is None)))

    def forward(self, x, edge_index):
        return self._run(x, edge_index)


class MRConv2d(_DenseGraphConv):
    """Max-Relative graph convolution, torch_vertex.py:8-20."""
    _conv = "mr"


class EdgeConv2d(_DenseGraphConv):
    """Edge convolution, torch_vertex.py:23-35."""
    _conv = "edge"


class GraphConv2d(nn.Module):
    """Static graph convolution layer, torch_vertex.py:38-52."""

    def __init__(self, in_channels, out_channels, conv="edge", act="relu", norm=None, bias=True):
        super().__init__()
        if conv == "edge":
            self.gconv = EdgeConv2d(in_channels, out_channels, act, norm, bias)
        elif conv == "mr":
            self.gconv = MRConv2d(in_channels, out_channels, act, norm, bias)
        else:
            raise NotImplementedError("conv:{} is not supported".format(conv))

    def forward(self, x, edge_index):
        return self.gconv(x, edge_index)


class DynConv2d(GraphConv2d):
    """Dynamic graph convolution layer, torch_vertex.py:55-72."""

    def __init__(self, in_channels, out_channels, kernel_size=9, dilation=1, conv="edge", act="relu",
                 norm=None, bias=True, stochastic=False, epsilon=0.0, knn="matrix"):
        super().__init__(in_channels, out_channels, conv, act, norm, bias)
        self.k = kernel_size
        self.d = dilation
        if knn == "matrix":
            self.dilated_knn_graph = DenseDilatedKnnGraph(kernel_size, dilation, stochastic, epsilon)
        else:
            self.dilated_knn_graph = DilatedKnnGraph(kernel_size, dilation, stochastic, epsilon)

    def forward(self, x, edge_index=None, residual=None, res_scale=1.0, out=None):
        """`residual` / `res_scale` / `out` (beyond the reference's signature, used by the blocks below): fold the
        block's skip connection and the write into a channel slice of a wider buffer into the consumer's store -
        only on the fused dynamic path in inference; otherwise they are applied with plain torch ops."""
        g = self.dilated_knn_graph
        if edge_index is None and isinstance(g, DenseDilatedKnnGraph):
            # kNN selection and convolution in one call (dgcn_dyn_conv_forward)
            block = None
            if (residual is not None or out is not None) and self.gconv.can_fuse_block(x):
                block = {}
                if residual is not None:
                    block.update(residual=residual, res_scale=res_scale)
                if out is not None:
                    block.update(out=out)
            y = self.gconv._run(x, None, fused=(g.k, g.dilation, g.columns()), block=block)
            if block is not None:
                return y
        else:
            y = self.gconv(x, edge_index if edge_index is not None else g(x))
        if residual is not None:
            y = y + residual * res_scale
        if out is not None:
            out.copy_(y)
            return out
        return y


class PlainDynBlock2d(nn.Module):
    """torch_vertex.py:75-86."""

    def __init__(self, in_channels, kernel_size=9, dilation=1, conv="edge", act="relu", norm=None,
                 bias=True, stochastic=False, epsilon=0.0, knn="matrix"):
        super().__init__()
        self.body = DynConv2d(in_channels, in_channels, kernel_size, dilation, conv, act, norm, bias,
                              stochastic, epsilon, knn)

    def forward(self, x, edge_index=None):
        return self.body(x, edge_index)


class ResDynBlock2d(nn.Module):
    """torch_vertex.py:89-101."""

    def __init__(self, in_channels, kernel_size=9, dilation=1, conv="edge", act="relu", norm=None,
                 bias=True, stochastic=False, epsilon=0.0, knn="matrix", res_scale=1):
        super().__init__()
        self.body = DynConv2d(in_channels, in_channels, kernel_size, dilation, conv, act, norm, bias,
                              stochastic, epsilon, knn)
        self.res_scale = res_scale

    def forward(self, x, edge_index=None, out=None):
        """torch_vertex.py:101: body(x) + x * res_scale; the skip connection rides in the consumer's store in
        inference.  `out` (optional, beyond the reference): a channel slice of the model's fusion buffer."""
        return self.body(x, edge_index, residual=x, res_scale=self.res_scale, out=out)


class DenseDynBlock2d(nn.Module):
    """torch_vertex.py:104-116."""

    def __init__(self, in_channels, out_channels=64, kernel_size=9, dilation=1, conv="edge", act="relu",
                 norm=None, bias=True, stochastic=False, epsilon=0.0, knn="matrix"):
        super().__init__()
        self.body = DynConv2d(in_channels, out_channels, kernel_size, dilation, conv, act, norm, bias,
                              stochastic, epsilon, knn)

    def forward(self, x, edge_index=None):
        """torch_vertex.py:116: cat((x, body(x)), 1); in inference the convolution writes its channel slice of the
        result directly."""
        if self.body.gconv.can_fuse_block(x) and edge_index is None:
            c_in, c_out = x.shape[1], self.body.gconv.nn[0].out_channels
            res = torch.empty((x.shape[0], c_in + c_out) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)
            res[:, :c_in].copy_(x)
            self.body(x, None, out=res[:, c_in:])
            return res
        return torch.cat((x, self.body(x, edge_index)), 1)
