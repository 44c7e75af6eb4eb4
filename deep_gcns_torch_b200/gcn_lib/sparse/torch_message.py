"""Generalised message passing - API of the reference's gcn_lib/sparse/torch_message.py
without PyG / torch_scatter: the aggregation runs in the fused CSR kernel of libdgcn."""
import collections
import os
import threading

import torch
from torch import nn

from ... import _native

__all__ = ["GenMessagePassing", "MsgNorm", "csr_of"]

_SOFTMAX = ("softmax_sg", "softmax", "softmax_sum")
_POWER = ("power", "power_sum")

# Non-persistent cache of destination-sorted graphs (SURVEY.md 8b: derived tensors must
# not show up in state_dict).  All layers of a model share one edge_index, so one
# entry serves a whole forward; entries pin the tensor they were built from.  An entry
# remembers the stream it was built on and the event that ends the build: a consumer on
# another stream waits for that event (no host sync), so a CSR is never read before it exists.
_csr_cache = collections.OrderedDict()
_csr_lock = threading.Lock()
CSR_CACHE_SIZE = int(os.environ.get("DGCN_CSR_CACHE", "4"))      # graphs kept; 0 disables the cache


def clear_csr_cache():
    with _csr_lock:
        _csr_cache.clear()


def csr_of(edge_index, num_nodes, cache=True):
    """(rowptr, src, eid, hubs) int32 for edge_index (2,E): rows = targets (edge_index[1]),
    stable within a row.  Built once per (tensor, version) by dgcn_csr_build.  cache=False
    for one-off graphs (GenMessagePassing.aggregate on explicit messages)."""
    if not cache or CSR_CACHE_SIZE <= 0:
        return _native.csr_build(edge_index, int(num_nodes))
    key = (edge_index.data_ptr(), tuple(edge_index.shape), edge_index._version, str(edge_index.device),
           int(num_nodes))
    cur = torch.cuda.current_stream(edge_index.device) if edge_index.is_cuda else None
    with _csr_lock:
        hit = _csr_cache.get(key)
        if hit is not None:
            _csr_cache.move_to_end(key)
            _, csr, stream_id, done = hit
            if cur is not None and stream_id is not None and stream_id != cur.cuda_stream:
                # first use from another stream: the build must be complete before this stream reads it.  Settle it
                # once on the host (afterwards the entry is valid for every stream, including a graph-capture stream,
                # where neither an event wait on uncaptured work nor an event query is legal).
                if torch.cuda.is_current_stream_capturing():
                    raise RuntimeError("csr_of: this graph's CSR was built on another stream and has not been used from "
                                       "a second stream yet - run one warm-up forward before CUDA-graph capture")
                done.synchronize()
                hit[2] = None
            return csr
    csr = _native.csr_build(edge_index, int(num_nodes))
    done, stream_id = None, None
    if cur is not None:
        done = torch.cuda.Event()
        done.record(cur)
        stream_id = cur.cuda_stream
    with _csr_lock:
        _csr_cache[key] = [edge_index, csr, stream_id, done]
        while len(_csr_cache) > CSR_CACHE_SIZE:
            _csr_cache.popitem(last=False)
    return csr


class _AggregateFn(torch.autograd.Function):
    """x_dst + MsgNorm(aggregate(relu(x_src[src] + edge_attr) + eps)); see dgcn.h."""

    @staticmethod
    def forward(ctx, owner, csr, raw, residual, x, edge_attr, t, p, y, msg_scale):
        ctx.aggr = owner._check_aggr()                    # None -> 'add' (PyG default), like the reference
        prm, keep = _native.genconv_params(ctx.aggr, t, p, y, getattr(owner, "eps", 1e-7),
                                           msg_scale, add_residual=residual)
        prm.raw_message = int(raw)
        out = _native.genconv_aggregate(x, x, csr, prm, edge_attr) if not raw else \
            _native.genconv_aggregate(x, None, csr, prm, None)
        ctx.owner, ctx.csr, ctx.raw, ctx.residual = owner, csr, raw, residual
        ctx.scalars = (t, p, y, msg_scale)
        ctx.save_for_backward(x, edge_attr)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from .. import _backward
        return _backward.genconv_aggregate_backward(ctx, grad_out)


class _GinSageFn(torch.autograd.Function):
    """GIN's sum_j x_j + (1 + eps) x_i, or GraphSAGE's mean over {j -> i, j != i} + {i} of x_j ('sage') / x_j - x_i
    ('rsage'), over the cached CSR graph; see dgcn_gin_sage_aggregate.  eps: GIN's (1,) buffer (no gradient) or None.
    The output is fp32 for fp32, bf16 and fp16 x; the gradient is returned in x's dtype."""

    @staticmethod
    def forward(ctx, rule, csr, x, eps):
        ctx.rule, ctx.csr, ctx.eps, ctx.x_dtype = rule, csr, eps, x.dtype
        return _native.gin_sage_aggregate(rule, x, csr, eps)

    @staticmethod
    def backward(ctx, grad_out):
        gx = _native.gin_sage_aggregate_backward(ctx.rule, grad_out, ctx.csr, ctx.eps).to(ctx.x_dtype) \
            if ctx.needs_input_grad[2] else None
        return None, None, gx, None


class GenMessagePassing(nn.Module):
    """torch_message.py:8-85."""

    def __init__(self, aggr="softmax", t=1.0, learn_t=False, p=1.0, learn_p=False, y=0.0, learn_y=False):
        super().__init__()
        self.aggr = aggr
        self.node_dim = 0
        if aggr in _SOFTMAX:
            if learn_t and aggr in ("softmax", "softmax_sum"):
                self.learn_t = True
                self.t = nn.Parameter(torch.Tensor([t]), requires_grad=True)
            else:
                self.learn_t = False
                self.t = t
            if aggr == "softmax_sum":
                self.y = nn.Parameter(torch.Tensor([y]), requires_grad=learn_y)
        elif aggr in _POWER:
            if learn_p:
                self.p = nn.Parameter(torch.Tensor([p]), requires_grad=True)
            else:
                self.p = p
            if aggr == "power_sum":
                self.y = nn.Parameter(torch.Tensor([y]), requires_grad=learn_y)

    def _scalars(self):
        t = getattr(self, "t", 1.0)
        p = getattr(self, "p", 1.0)
        y = getattr(self, "y", 0.0)
        if self.aggr in ("softmax_sum", "power_sum"):
            self.sigmoid_y = torch.sigmoid(self.y)          # read by callers (print_params)
        return t, p, y

    def _check_aggr(self):
        if self.aggr not in _SOFTMAX + _POWER + ("add", "mean", "max", None):
            raise NotImplementedError("To be implemented")
        return "add" if self.aggr is None else self.aggr

    def propagate(self, edge_index, x, edge_attr=None, msg_scale=None, residual=False, size=None):
        """message + aggregate (+ MsgNorm + residual) for flow source_to_target; the
        PyG `propagate` of torch_vertex.py:68 with message() of :78-85 folded in."""
        self._check_aggr()
        t, p, y = self._scalars()
        csr = csr_of(edge_index, x.size(0))
        return _AggregateFn.apply(self, csr, False, residual, x, edge_attr, t, p, y, msg_scale)

    def aggregate(self, inputs, index, ptr=None, dim_size=None):
        """torch_message.py:44-85 on explicit per-edge messages `inputs` (E,C)."""
        self._check_aggr()
        t, p, y = self._scalars()
        n = int(dim_size) if dim_size is not None else int(index.max()) + 1
        pos = torch.arange(index.numel(), device=index.device)
        csr = csr_of(torch.stack((pos, index)), n, cache=False)     # throw-away graph: do not evict real ones
        return _AggregateFn.apply(self, csr, True, False, inputs, None, t, p, y, None)


class MsgNorm(nn.Module):
    """torch_message.py:88-99.  Inside GENConv the normalisation is fused into the
    aggregation kernel; this module owns `msg_scale` and keeps a standalone forward."""

    def __init__(self, learn_msg_scale=False):
        super().__init__()
        self.msg_scale = nn.Parameter(torch.Tensor([1.0]), requires_grad=learn_msg_scale)

    def forward(self, x, msg, p=2):
        msg = torch.nn.functional.normalize(msg, p=p, dim=1)
        return msg * x.norm(p=p, dim=1, keepdim=True) * self.msg_scale
