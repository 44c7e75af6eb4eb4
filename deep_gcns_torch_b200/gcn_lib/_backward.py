"""Backward glue of GENConv's aggregate autograd node: unpack what forward saved, call the native gradient
kernels (dgcn_genconv_aggregate_backward), hand the gradients back in the order of the forward's inputs."""
from .. import _native


def genconv_aggregate_backward(ctx, grad_out):
    """Inputs of _AggregateFn.forward: (owner, csr, raw, residual, x, edge_attr, t, p, y, msg_scale)."""
    import torch
    x, edge_attr = ctx.saved_tensors
    owner = ctx.owner
    t, p, y, msg_scale = ctx.scalars
    prm, keep = _native.genconv_params(ctx.aggr, t, p, y, getattr(owner, "eps", 1e-7), msg_scale,
                                       add_residual=ctx.residual)
    prm.raw_message = int(ctx.raw)
    need = ctx.needs_input_grad
    gsrc, gdst, gea, gsc = _native.genconv_aggregate_backward(
        x, None if ctx.raw else x, ctx.csr, prm, grad_out, edge_attr,
        softmax_grad=getattr(owner, "learn_t", False), need_edge_attr=need[5])
    gx = None
    if need[4]:
        gx = gsrc if gdst is None else gsrc + gdst
    def scalar_grad(i, v, idx):
        return gsc[idx:idx + 1].clone() if (need[i] and torch.is_tensor(v)) else None
    return (None, None, None, None, gx, gea if need[5] else None, scalar_grad(6, t, 0), scalar_grad(7, p, 1),
            scalar_grad(8, y, 2), scalar_grad(9, msg_scale, 3))
