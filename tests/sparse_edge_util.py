"""Shared pieces of the sparse-layout EdgeConv tests and of their golden generator (no GPU needed here):

- EdgeConvStandIn / install_reference_stand_ins: torch_geometric's EdgeConv(nn, aggr='max') restated - message
  nn(cat[x_i, x_j - x_i]) with x_i = x[edge_index[1]], x_j = x[edge_index[0]], aggregated at edge_index[1] by
  oracle/ref_shims.py's scatter (empty groups -> 0; duplicate edges and self-loops are ordinary edges) - put in place
  of ref_shims' placeholder before the reference is imported, so that the unmodified reference's EdgConv
  (gcn_lib/sparse/torch_vertex.py:106-114) executes.  Its reset_parameters is not restated: the generator sets every
  parameter explicitly.  The stand-in's torch_scatter.scatter_max / scatter_min also return a copy of the
  reduction: utils/pyg_util.py:31 zeroes entries of the result in place, which autograd allows on torch_scatter's
  own result but not on the output that scatter_reduce's backward reads (the model golden takes a backward).
- edge_conv: the CPU restatement of EdgConv (fp32, or fp64 for autograd references), its max routed to the first
  edge in edge_index order as torch_scatter's scatter_max does (seg_max_first);
- edge_tie_mask: the sparse analogue of backward_util.edge_tie_mask.
"""
import sys

import torch
import torch.nn.functional as F

from oracle import ref_shims


class EdgeConvStandIn(ref_shims.MessagePassing):
    """torch_geometric.nn.EdgeConv(nn, aggr='max')."""

    def __init__(self, nn, aggr="max", **kw):
        super().__init__(aggr=aggr, **kw)
        self.nn = nn

    def forward(self, x, edge_index):
        return self.propagate(edge_index, x=x)

    def message(self, x_i, x_j):
        return self.nn(torch.cat([x_i, x_j - x_i], dim=-1))


def _scatter_max_copy(src, index, dim=-1, out=None, dim_size=None):
    return ref_shims.scatter(src, index, dim, out, dim_size, "max").clone(), None


def _scatter_min_copy(src, index, dim=-1, out=None, dim_size=None):
    return ref_shims.scatter(src, index, dim, out, dim_size, "min").clone(), None


def install_reference_stand_ins():
    """ref_shims' stand-in modules, with EdgeConv and the copying scatter_max / scatter_min; call before
    ref_shims.load_reference()."""
    ref_shims._install_stubs()
    sys.modules["torch_geometric.nn"].EdgeConv = EdgeConvStandIn
    sys.modules["torch_scatter"].scatter_max = _scatter_max_copy
    sys.modules["torch_scatter"].scatter_min = _scatter_min_copy


def edge_conv_params(mlp, dtype=torch.float32):
    """Functional parameters of EdgConv's MLP([2*C_in, C_out], act, norm, bias) (gcn_lib/sparse/torch_nn.py:50-68):
    weight, bias, slope (PReLU weight), norm {weight, bias, running_mean, running_var, eps}; only those that exist."""
    cast = lambda v: v.detach().cpu().to(dtype).clone()
    lin = mlp[0]
    p = {"weight": cast(lin.weight)}
    if lin.bias is not None:
        p["bias"] = cast(lin.bias)
    for m in list(mlp)[1:]:
        if isinstance(m, torch.nn.PReLU):
            p["slope"] = cast(m.weight)
        elif isinstance(m, torch.nn.BatchNorm1d):
            p["norm"] = {"weight": cast(m.weight), "bias": cast(m.bias), "running_mean": cast(m.running_mean),
                         "running_var": cast(m.running_var), "eps": m.eps}
    return p


def _act(u, act, slope=None):
    act = None if act is None else str(act).lower()
    if act in (None, "none"):
        return u
    if act == "relu":
        return F.relu(u)
    if act == "leakyrelu":
        return F.leaky_relu(u, 0.2)
    if act == "prelu":
        return F.prelu(u, slope)
    raise NotImplementedError(act)


def seg_max_first(y, dst, n):
    """(out, arg): per destination and channel the max over its edges and the FIRST edge (in edge order) that
    attains it - torch_scatter's scatter_max, whose gradient goes to that edge only; empty rows -> 0, arg -1.
    out is y gathered at arg, so autograd routes the gradient the same way (torch's scatter_reduce amax would split
    a tied gradient evenly)."""
    C = y.shape[1]
    idx = dst.view(-1, 1).expand(-1, C)
    top = torch.full((n, C), float("-inf"), dtype=y.dtype).scatter_reduce(0, idx, y.detach(), "amax",
                                                                          include_self=True)
    E = y.shape[0]
    pos = torch.arange(E).view(-1, 1).expand(-1, C)
    cand = torch.where(y.detach() == top.index_select(0, dst), pos, torch.full_like(pos, E))
    arg = torch.full((n, C), E, dtype=torch.long).scatter_reduce(0, idx, cand, "amin", include_self=True)
    has = arg < E
    out = y.gather(0, arg.clamp(max=max(E - 1, 0))) if E > 0 else torch.zeros((n, C), dtype=y.dtype)
    out = torch.where(has, out, torch.zeros_like(out))
    return out, torch.where(has, arg, torch.full_like(arg, -1))


def edge_conv(x, edge_index, p, act="relu", training=False, return_stats=False):
    """gcn_lib/sparse/torch_vertex.py:106-114 (EdgConv) in x's dtype: torch_geometric's EdgeConv
    out_i = max_{e=(j->i)} nn(cat[x_i, x_j - x_i]) with nn = Linear -> BatchNorm1d over the E edge rows (batch
    statistics when `training`, biased variance for the normalisation) -> act; empty rows -> 0; the max routes its
    gradient to the first edge in edge_index order (seg_max_first).  p: edge_conv_params (in x's dtype).
    return_stats: also (batch mean, biased batch variance) of the edge rows, or None."""
    src, dst = edge_index[0].long(), edge_index[1].long()
    xi, xj = x.index_select(0, dst), x.index_select(0, src)
    z = F.linear(torch.cat([xi, xj - xi], 1), p["weight"], p.get("bias"))
    stats = None
    if "norm" in p:
        q = p["norm"]
        if training:
            mean, var = z.mean(0), z.var(0, unbiased=False)
            stats = (mean, var)
        else:
            mean, var = q["running_mean"], q["running_var"]
        z = (z - mean) / torch.sqrt(var + q["eps"]) * q["weight"] + q["bias"]
    y = _act(z, act, p.get("slope"))
    out, _ = seg_max_first(y, dst, x.shape[0])
    return (out, stats) if return_stats else out


def mlp_act(mlp):
    """The activation name of an EdgConv MLP ('relu', 'leakyrelu', 'prelu' or None)."""
    for m in list(mlp)[1:]:
        if isinstance(m, torch.nn.PReLU):
            return "prelu"
        if isinstance(m, torch.nn.LeakyReLU):
            return "leakyrelu"
        if isinstance(m, torch.nn.ReLU):
            return "relu"
    return None


def edge_tie_mask(mlp, x, edge_index, tie_rel, kink_rel, training):
    """(N, C_out) bool, fp64: the EdgConv maxima whose winning edge an fp32 evaluation may legitimately pick
    differently, or whose activation derivative it may take on the other side of the kink.  y = act(s z + t) with
    (s, t) the BatchNorm affine (batch statistics of the edge rows when `training`) or (1, 0).  A (node, channel) is
    masked when the runner-up's y is within tie_rel * |s| * max(1, |z|) of the top (fp32 errors live in z; edges
    from the winner's own source - duplicates - carry the same z on every evaluation and are not runners-up) - unless
    s == 0, where every edge ties exactly and both sides take the first, or the winner sits in ReLU's flat part,
    where any choice carries zero gradient - or when the winner's |s z + t| is below kink_rel * max(1, |s z|)."""
    p = edge_conv_params(mlp, torch.float64)
    act = mlp_act(mlp)
    src, dst = edge_index[0].long().cpu(), edge_index[1].long().cpu()
    xd = x.detach().cpu().double()
    xi, xj = xd.index_select(0, dst), xd.index_select(0, src)
    z = F.linear(torch.cat([xi, xj - xi], 1), p["weight"], p.get("bias"))
    s = torch.ones(z.shape[1], dtype=torch.float64)
    t = torch.zeros_like(s)
    if "norm" in p:
        q = p["norm"]
        mean, var = (z.mean(0), z.var(0, unbiased=False)) if training else (q["running_mean"], q["running_var"])
        s = q["weight"] / torch.sqrt(var + q["eps"])
        t = q["bias"] - mean * s
    u = s * z + t
    y = _act(u, act, p.get("slope"))
    n, C, E = xd.shape[0], z.shape[1], z.shape[0]
    top, arg = seg_max_first(y, dst, n)
    has = arg >= 0
    a = arg.clamp(min=0)
    if E == 0:
        return torch.zeros((n, C), dtype=torch.bool)
    z_w, u_w = z.gather(0, a), u.gather(0, a)
    win_src = src[a]                                                       # the winner's source, per (row, channel)
    y2 = y.masked_fill(src.view(-1, 1) == win_src.index_select(0, dst), float("-inf"))   # its edges out ...
    second = torch.full((n, C), float("-inf"), dtype=y.dtype).scatter_reduce(
        0, dst.view(-1, 1).expand(-1, C), y2, "amax", include_self=True)   # ... the runner-up's y
    scale = s.abs().view(1, -1) * z_w.abs().clamp_min(1.0)
    tie = (top - second) < tie_rel * scale
    tie &= s.view(1, -1) != 0
    if act == "relu":
        tie &= ~(u_w < -kink_rel * (s.view(1, -1) * z_w).abs().clamp_min(1.0))
    kink = u_w.abs() < kink_rel * (s.view(1, -1) * z_w).abs().clamp_min(1.0) if act is not None \
        else torch.zeros_like(tie)
    return (tie | kink) & has
