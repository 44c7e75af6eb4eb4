"""Fused 'res+' block of DeeperGCN (SURVEY.md 8f rank 1) - opt-in, inference and (fused_training=True) training.

The reference writes the block as separate modules (examples/ogb/ogbn_arxiv/model.py:91-106):

    h2 = norms[l-1](h); h2 = relu(h2); h2 = dropout(h2); h = gcns[l](h2, edge_index) + h

In eval mode the BatchNorm1d is a per-channel affine, dropout is the identity and GENConv with
mlp_layers=1 ends in one Linear.  `res_plus_block` runs the same arithmetic in two launches:

    dgcn_genconv_aggregate         reads h rows as relu(s*h + t) (gathered rows and the residual row),
                                   message + aggregate + MsgNorm + (z_i + m_i)     -> a
    dgcn_linear_residual           h_out = h + a W^T + b on the tensor cores (wgmma; two-plane bf16 split of both
                                   operands, fp32 accumulation; bias and skip connection in the epilogue)

so the normalised / activated copy of h and the GENConv output before the skip connection are never
written to HBM (three N x C passes fewer per layer).  A model opts in by replacing the four lines above
with `h = res_plus_block(self.gcns[l], self.norms[l-1], h, edge_index)`; with autograd enabled, a
training-mode norm or an unsupported layer shape the call falls back to the unfused module sequence.

Training (`fused_training=True`, `trainable`): one autograd node per block.  Forward: BatchNorm1d statistics of h
(batch or running) folded to (scale, shift) on the device; a dropout mask drawn as
`torch.empty((N, C), device=h.device).bernoulli_(1 - dropout)` and bit-packed (the fp32 draw is freed before the
aggregate runs); the aggregate reads every row as `keep ? relu(scale*h + shift) / (1 - dropout) : 0`; then
`h + a W^T + b`.  It saves h, a, the bits and C-sized vectors - not the normalised, activated and dropped copies
of h nor a byte mask.  Backward: the Linear by torch matmuls, the aggregate backward recomputes the activated rows
from h with the forward's instructions, and one epilogue kernel pair takes the row gradients back through dropout,
ReLU and BatchNorm.  The mask is a different sample from the one F.dropout would draw, so the path is opt-in.
Not covered (they run the four lines): LayerNorm, edge features / encode_edge, mlp_layers > 1, half-precision rows,
a SyncBatchNorm that syncs, the partitioned multi-GPU block.
"""
import torch
import torch.nn.functional as F
from torch import nn

from ... import _native
from .torch_message import csr_of
from .torch_vertex import GENConv

__all__ = ["bn_eval_affine", "res_plus_block", "res_plus_block_partitioned", "fusable", "trainable"]


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


def _uses_batch_stats(norm):
    """nn.BatchNorm1d's rule: batch statistics in training mode or when no running statistics are kept."""
    return norm.training or (norm.running_mean is None and norm.running_var is None)


def trainable(conv, norm, h, dropout):
    """The fused training path covers: autograd on or a training-mode norm; a BatchNorm1d, or a SyncBatchNorm that
    does not sync, on (N, C) rows (affine or not, running statistics or not); GENConv with mlp_layers = 1 and no
    edge encoder; a contiguous CUDA fp32 h with C % 4 == 0 and C <= 512; 0 <= dropout < 1."""
    is_bn = isinstance(norm, nn.BatchNorm1d) or (isinstance(norm, nn.SyncBatchNorm) and _native.sync_group(norm) is None)
    return ((torch.is_grad_enabled() or norm.training) and is_bn and isinstance(conv, GENConv) and
            len(conv.mlp) == 1 and isinstance(conv.mlp[0], nn.Linear) and not conv.encode_edge and
            h.dim() == 2 and h.is_cuda and h.dtype == torch.float32 and h.is_contiguous() and
            h.shape[1] % 4 == 0 and h.shape[1] <= 512 and h.shape[1] == norm.num_features and
            0.0 <= dropout < 1.0 and (h.shape[0] > 1 or not _uses_batch_stats(norm)))


def bn_batch_affine(norm, h):
    """Batch statistics of h (N, C) as nn.BatchNorm1d computes them in training mode: returns (scale, shift, mean,
    invstd) with norm(h) = scale * h + shift, and updates the running statistics as the module does (momentum,
    momentum=None as a cumulative average, unbiased variance, num_batches_tracked).  Device-side only."""
    with torch.no_grad():
        var, mean = torch.var_mean(h, dim=0, unbiased=False)
        invstd = torch.rsqrt(var + norm.eps)
        if norm.training and norm.track_running_stats and norm.running_mean is not None:
            norm.num_batches_tracked.add_(1)
            if norm.momentum is None:
                factor = 1.0 / norm.num_batches_tracked.double()
            else:
                factor = norm.momentum
            n = h.shape[0]
            norm.running_mean.mul_(1 - factor).add_(mean * factor)
            norm.running_var.mul_(1 - factor).add_(var * (factor * n / (n - 1)))
        scale = invstd * norm.weight.detach() if norm.weight is not None else invstd
        shift = -mean * scale
        if norm.bias is not None:
            shift = shift + norm.bias.detach()
    return scale.contiguous(), shift.contiguous(), mean, invstd


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


class _ResPlusTrainFn(torch.autograd.Function):
    """h + Linear(aggregate(dropout(relu(norm(h))))) with the block's statistics, mask and activations folded into
    the kernels' reads (module docstring).  Inputs after the modules: h, Linear weight / bias, BatchNorm weight / bias
    and GENConv's scalars t, p, y, msg_scale (tensors are differentiated, floats are not)."""

    @staticmethod
    def forward(ctx, conv, norm, csr, dropout, out_box, h, weight, bias, gamma, beta, t, p, y, msg_scale):
        N, C = h.shape
        batch = _uses_batch_stats(norm)
        if batch:
            scale, shift, mean, invstd = bn_batch_affine(norm, h)
        else:
            scale, shift = bn_eval_affine(norm)
            mean = norm.running_mean.clone()
            invstd = torch.rsqrt(norm.running_var + norm.eps)
        keep = None
        if dropout > 0 and conv.training:
            draw = torch.empty((N, C), device=h.device).bernoulli_(1 - dropout)
            keep = (_native.keep_bits(draw), 1.0 / (1.0 - dropout))
            del draw
        prm, _keep = _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, msg_scale, add_residual=True)
        a = _native.genconv_aggregate(h, h, csr, prm, pre=(scale, shift, True), keep=keep)
        res = _linear_plus(conv.mlp[0], a, h, out=out_box[0])
        ctx.conv, ctx.csr, ctx.batch, ctx.scalars = conv, csr, batch, (t, p, y, msg_scale)
        ctx.keep_scale = None if keep is None else keep[1]
        bits = keep[0] if keep is not None else None
        ctx.save_for_backward(h, a, bits, scale, shift, mean, invstd, weight)
        return res

    @staticmethod
    def backward(ctx, g_out):
        h, a, bits, scale, shift, mean, invstd, weight = ctx.saved_tensors
        need = ctx.needs_input_grad
        conv = ctx.conv
        t, p, y, msg_scale = ctx.scalars
        g_out = g_out.contiguous()
        g_a = g_out @ weight
        g_w = g_out.t() @ a if need[6] else None
        g_b = g_out.sum(0) if need[7] else None
        prm, _keep = _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, msg_scale, add_residual=True)
        keep = None if bits is None else (bits, ctx.keep_scale)
        gsrc, gdst, _gea, gsc = _native.genconv_aggregate_backward(
            h, h, ctx.csr, prm, g_a, softmax_grad=getattr(conv, "learn_t", False), pre=(scale, shift, True),
            keep=keep)
        del g_a
        # g_y = dL/d norm(h) (over gsrc), sums = [sum g_y | sum g_y * xhat] per channel
        sums = _native.res_plus_backward_gy(h, scale, shift, keep, gsrc, gdst, mean, invstd)
        g_y, n = gsrc, h.shape[0]
        g_beta, g_gamma = sums[0].float(), sums[1].float()       # d beta = sum g_y, d gamma = sum g_y * xhat
        if ctx.batch:   # g_h = gamma * invstd * (g_y - mean(g_y) - xhat * mean(g_y * xhat)), scale = gamma * invstd
            c_b = -scale * invstd * (sums[1] / n).float()
            c_d = -scale * (sums[0] / n).float() - c_b * mean
            g_h = _native.res_plus_backward_dh(g_y, h, scale, c_b, c_d, grad_skip=g_out, out=g_y)
        else:           # running statistics: norm(h) is the affine scale * h + shift
            g_h = _native.res_plus_backward_dh(g_y, h, scale, grad_skip=g_out, out=g_y)

        def scalar_grad(i, v, idx):
            return gsc[idx:idx + 1].clone() if (need[i] and torch.is_tensor(v)) else None
        return (None, None, None, None, None, g_h if need[5] else None, g_w, g_b,
                g_gamma if need[8] else None, g_beta if need[9] else None,
                scalar_grad(10, t, 0), scalar_grad(11, p, 1), scalar_grad(12, y, 2), scalar_grad(13, msg_scale, 3))


def _res_plus_train(conv, norm, h, edge_index, out, dropout):
    t, p, y = conv._scalars()
    msg_scale = conv.msg_norm.msg_scale if conv.msg_norm is not None else None
    lin = conv.mlp[0]
    return _ResPlusTrainFn.apply(conv, norm, csr_of(edge_index, h.size(0)), float(dropout), (out,), h, lin.weight,
                                 lin.bias, norm.weight, norm.bias, t, p, y, msg_scale)


def res_plus_block(conv, norm, h, edge_index, out=None, dropout=0.0, fused_training=False):
    """h <- GENConv(dropout(relu(norm(h))), edge_index) + h   (model.py:91-106).

    Fused in inference when `fusable`; with fused_training=True also in training when `trainable` (the dropout
    mask is then the block's own draw, see the module docstring).  Everything else runs the four lines."""
    if fused_training and trainable(conv, norm, h, dropout):
        return _res_plus_train(conv, norm, h, edge_index, out, dropout)
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
