"""Fused 'res+' block of DeeperGCN (SURVEY.md 8f rank 1) - opt-in, inference only.

The reference writes the block as separate modules (examples/ogb/ogbn_arxiv/model.py:91-106):

    h2 = norms[l-1](h); h2 = relu(h2); h2 = dropout(h2); h = gcns[l](h2, edge_index) + h

In eval mode the BatchNorm1d is a per-channel affine, dropout is the identity and GENConv with
mlp_layers=1 ends in one Linear.  `res_plus_block` runs the same arithmetic in two launches:

    dgcn_genconv_aggregate_fused   reads h rows as relu(s*h + t) (gathered rows and the residual row),
                                   message + aggregate + MsgNorm + (z_i + m_i)     -> a
    dgcn_linear_residual           h_out = h + a W^T + b on the tensor cores (wgmma; two-plane bf16 split of both
                                   operands, fp32 accumulation; bias and skip connection in the epilogue)

so the normalised / activated copy of h and the GENConv output before the skip connection are never
written to HBM (three N x C passes fewer per layer).  A model opts in by replacing the four lines above
with `h = res_plus_block(self.gcns[l], self.norms[l-1], h, edge_index)`; with autograd enabled, a
training-mode norm or an unsupported layer shape the call falls back to the unfused module sequence.
"""
import torch
import torch.nn.functional as F
from torch import nn

from ... import _native
from .torch_message import csr_of

__all__ = ["bn_eval_affine", "res_plus_block", "res_plus_block_partitioned", "fusable"]


def bn_eval_affine(norm):
    """(scale, shift) with norm(h) = scale * h + shift for an eval-mode BatchNorm1d (running statistics).
    Cached on the module (a plain attribute, not a buffer: nothing new in state_dict) until one of the four
    tensors it derives from changes (tensor version counters / identity)."""
    src = (norm.running_var, norm.running_mean, norm.weight, norm.bias)
    key = tuple((id(t), t._version, t.device) if t is not None else None for t in src) + (norm.eps,)
    hit = norm.__dict__.get("_dgcn_eval_affine")
    if hit is not None and hit[0] == key:
        return hit[1], hit[2]
    var, mean = norm.running_var, norm.running_mean
    scale = torch.rsqrt(var + norm.eps)
    if norm.weight is not None:
        scale = scale * norm.weight
    shift = -mean * scale
    if norm.bias is not None:
        shift = shift + norm.bias
    scale, shift = scale.detach().contiguous(), shift.detach().contiguous()
    norm.__dict__["_dgcn_eval_affine"] = (key, scale, shift)
    return scale, shift


def fusable(conv, norm, h):
    """The fused kernels cover: no autograd, eval-mode BatchNorm1d (or the SyncBatchNorm that
    convert_sync_batchnorm made of it, on (N, C) rows) with running statistics, GENConv whose MLP is a single
    Linear (mlp_layers = 1) and no edge features."""
    is_bn = isinstance(norm, nn.BatchNorm1d) or (isinstance(norm, nn.SyncBatchNorm) and h.dim() == 2)
    return (not torch.is_grad_enabled() and is_bn and not norm.training and
            norm.running_var is not None and len(conv.mlp) == 1 and isinstance(conv.mlp[0], nn.Linear) and
            not conv.encode_edge and h.is_cuda and h.dtype == torch.float32 and h.shape[1] % 4 == 0 and
            h.shape[1] <= 512)


def _prm(conv):
    t, p, y = conv._scalars()
    scale = conv.msg_norm.msg_scale if conv.msg_norm is not None else None
    return _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, scale, add_residual=True)


def _linear_plus(lin, a, h, out=None):
    """h + a W^T + b: the tensor-core row-Linear with bias and skip connection in its epilogue (one pass over a, h and
    the result); shapes it does not cover keep cuBLAS with the skip connection riding on the GEMM's beta."""
    if a.is_cuda and _native.linear_residual_supported(lin.in_features, lin.out_features) and \
            a.data_ptr() % 16 == 0 and h.data_ptr() % 16 == 0 and (out is None or out.data_ptr() % 16 == 0):
        return _native.linear_residual(a, lin.weight, lin.bias, h, out=out)
    res = torch.addmm(h, a, lin.weight.t(), out=out)
    if lin.bias is not None:
        res.add_(lin.bias)
    return res


def res_plus_block(conv, norm, h, edge_index, out=None, dropout=0.0):
    """h <- GENConv(dropout(relu(norm(h))), edge_index) + h   (model.py:91-106), fused when `fusable`."""
    if not fusable(conv, norm, h):
        h2 = F.dropout(F.relu(norm(h)), p=dropout, training=conv.training)
        return conv(h2, edge_index) + h
    h = h.contiguous()
    prm, _keep = _prm(conv)
    scale, shift = bn_eval_affine(norm)
    a = _native.genconv_aggregate(h, h, csr_of(edge_index, h.size(0)), prm, pre=(scale, shift, True))
    return _linear_plus(conv.mlp[0], a, h, out=out)


def res_plus_block_partitioned(conv, norm, part, channels, slot, scratch=None, group=None, overlap=True):
    """The same block on a node partition (deep_gcns_torch_b200.partition): the layer input is the raw h in
    part.local_rows(channels, slot); the halo exchange ships raw rows (the kernel applies norm -> relu on
    read) and overlaps the interior rows; the result is written into the OTHER buffer slot, which is
    returned, so a layer stack ping-pongs between the two persistent buffers without copies."""
    from ... import partition as P
    h = part.local_rows(channels, slot)
    if not fusable(conv, norm, h):
        raise RuntimeError("res_plus_block_partitioned: inference-only fused path (eval BatchNorm1d, mlp_layers=1)")
    scale, shift = bn_eval_affine(norm)
    a = P.aggregate_partitioned(conv, part, channels, slot=slot, pre=(scale, shift, True), out=scratch, group=group,
                                overlap=overlap)
    return _linear_plus(conv.mlp[0], a, h, out=part.local_rows(channels, slot ^ 1))
