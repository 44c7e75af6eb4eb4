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
- edge_tie_mask: the sparse analogue of backward_util.edge_tie_mask;
- exact_fixture: the exact-arithmetic EdgConv fixtures of tests/test_sparse_edgeconv_shapes_gpu.py.

The restatement and the mask run on the device of their inputs (the fp64 references of E = 1 M edges run on the GPU).
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


def edge_conv_params(mlp, dtype=torch.float32, device="cpu"):
    """Functional parameters of EdgConv's MLP([2*C_in, C_out], act, norm, bias) (gcn_lib/sparse/torch_nn.py:50-68):
    weight, bias, slope (PReLU weight), norm {weight, bias, running_mean, running_var, eps}; only those that exist
    (a BatchNorm1d without affine or without running statistics has None there)."""
    cast = lambda v: None if v is None else v.detach().to(device=device, dtype=dtype).clone()
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
    C, dev = y.shape[1], y.device
    idx = dst.view(-1, 1).expand(-1, C)
    top = torch.full((n, C), float("-inf"), dtype=y.dtype, device=dev).scatter_reduce(0, idx, y.detach(), "amax",
                                                                                      include_self=True)
    E = y.shape[0]
    pos = torch.arange(E, device=dev).view(-1, 1).expand(-1, C)
    cand = torch.where(y.detach() == top.index_select(0, dst), pos, torch.full_like(pos, E))
    arg = torch.full((n, C), E, dtype=torch.long, device=dev).scatter_reduce(0, idx, cand, "amin", include_self=True)
    has = arg < E
    out = y.gather(0, arg.clamp(max=max(E - 1, 0))) if E > 0 else torch.zeros((n, C), dtype=y.dtype, device=dev)
    out = torch.where(has, out, torch.zeros_like(out))
    return out, torch.where(has, arg, torch.full_like(arg, -1))


def edge_conv(x, edge_index, p, act="relu", training=False, return_stats=False, retain_z=None):
    """gcn_lib/sparse/torch_vertex.py:106-114 (EdgConv) in x's dtype: torch_geometric's EdgeConv
    out_i = max_{e=(j->i)} nn(cat[x_i, x_j - x_i]) with nn = Linear -> BatchNorm1d over the E edge rows (batch
    statistics when `training`, biased variance for the normalisation) -> act; empty rows -> 0; the max routes its
    gradient to the first edge in edge_index order (seg_max_first).  p: edge_conv_params (in x's dtype, on x's
    device); a BatchNorm1d without affine has weight / bias None.
    return_stats: also (batch mean, biased batch variance) of the edge rows, or None.  retain_z: a list that receives
    the Linear's output z (E, C_out), its gradient retained."""
    src, dst = edge_index[0].long(), edge_index[1].long()
    xi, xj = x.index_select(0, dst), x.index_select(0, src)
    z = F.linear(torch.cat([xi, xj - xi], 1), p["weight"], p.get("bias"))
    if retain_z is not None:
        z.retain_grad()
        retain_z.append(z)
    stats = None
    if "norm" in p:
        q = p["norm"]
        if training:
            mean, var = z.mean(0), z.var(0, unbiased=False)
            stats = (mean, var)
        else:
            mean, var = q["running_mean"], q["running_var"]
        z = (z - mean) / torch.sqrt(var + q["eps"])
        if q["weight"] is not None:
            z = z * q["weight"] + q["bias"]
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


def edge_tie_mask(mlp, x, edge_index, tie_rel, kink_rel, training, exact=False):
    """(N, C_out) bool, fp64, on x's device: the EdgConv maxima whose winning edge an fp32 evaluation may
    legitimately pick differently, or whose activation derivative it may take on the other side of the kink.
    y = act(s z + t) with (s, t) the BatchNorm affine (batch statistics of the edge rows when `training`) or (1, 0).
    A (node, channel) is masked when the runner-up's y is within tie_rel * |s| * max(1, |z|) of the top (fp32 errors
    live in z; edges from the winner's own source - duplicates - carry the same z on every evaluation and are not
    runners-up) - unless s == 0, where every edge ties exactly and both sides take the first, or the winner sits in
    ReLU's flat part, where any choice carries zero gradient - or when the winner's |s z + t| is below
    kink_rel * max(1, |s z|).  exact: z is exact in fp32 (exact_fixture), so every edge whose z equals the
    winner's - a duplicate, or an edge from a copied source row - ties exactly on every evaluation and is not a
    runner-up either; what remains masked is a real near-tie, which such a fixture must not have."""
    dev = x.device
    p = edge_conv_params(mlp, torch.float64, dev)
    act = mlp_act(mlp)
    src, dst = edge_index[0].long().to(dev), edge_index[1].long().to(dev)
    xd = x.detach().double()
    xi, xj = xd.index_select(0, dst), xd.index_select(0, src)
    z = F.linear(torch.cat([xi, xj - xi], 1), p["weight"], p.get("bias"))
    s = torch.ones(z.shape[1], dtype=torch.float64, device=dev)
    t = torch.zeros_like(s)
    if "norm" in p:
        q = p["norm"]
        mean, var = (z.mean(0), z.var(0, unbiased=False)) if training else (q["running_mean"], q["running_var"])
        s = (q["weight"] if q["weight"] is not None else 1.0) / torch.sqrt(var + q["eps"])
        t = (q["bias"] if q["bias"] is not None else 0.0) - mean * s
    u = s * z + t
    y = _act(u, act, p.get("slope"))
    n, C, E = xd.shape[0], z.shape[1], z.shape[0]
    top, arg = seg_max_first(y, dst, n)
    has = arg >= 0
    a = arg.clamp(min=0)
    if E == 0:
        return torch.zeros((n, C), dtype=torch.bool, device=dev)
    z_w, u_w = z.gather(0, a), u.gather(0, a)
    if exact:
        same = z == z_w.index_select(0, dst)                               # the winner's z, per (row, channel)
    else:
        same = src.view(-1, 1) == src[a].index_select(0, dst)              # the winner's source, per (row, channel)
    y2 = y.masked_fill(same, float("-inf"))                                # its edges out ...
    second = torch.full((n, C), float("-inf"), dtype=y.dtype, device=dev).scatter_reduce(
        0, dst.view(-1, 1).expand(-1, C), y2, "amax", include_self=True)   # ... the runner-up's y
    scale = s.abs().view(1, -1) * z_w.abs().clamp_min(1.0)
    tie = (top - second) < tie_rel * scale
    tie &= s.view(1, -1) != 0
    if act == "relu":
        tie &= ~(u_w < -kink_rel * (s.view(1, -1) * z_w).abs().clamp_min(1.0))
    kink = u_w.abs() < kink_rel * (s.view(1, -1) * z_w).abs().clamp_min(1.0) if act is not None \
        else torch.zeros_like(tie)
    return (tie | kink) & has


# ---- exact-arithmetic fixtures ----------------------------------------------------------------------------------
OFFSET = 1024                                    # added to the offset input channels: un-centred features
ROW_LENGTHS = (0, 1, 31, 32, 33, 63, 64, 65)     # in-degrees every exact graph has, around the kernels' 32-edge chunks
HUB = 1100                                       # in-degree of the hub row (> 1024) of the graphs built with one


def exact_graph(N, hub, g):
    """(2, E) int64 edge_index over N nodes, in shuffled order: one row of each length in ROW_LENGTHS (and one of HUB
    edges when `hub`), every other row 0 to 6 edges; random sources, with self-loops (every 7th edge), duplicates
    (every 5th edge repeats its predecessor's source within a row) and edges from the copied rows of exact_features
    (the sources of edges 3 and 4 mod 11)."""
    rows = torch.randperm(N, generator=g)
    deg = torch.randint(0, 7, (N,), generator=g)
    special = list(ROW_LENGTHS) + ([HUB] if hub else [])
    deg[rows[:len(special)]] = torch.tensor(special)
    dst = torch.repeat_interleave(torch.arange(N), deg)
    src = torch.randint(0, N, (dst.numel(),), generator=g)
    k = torch.arange(dst.numel())
    a, b = copied_rows(N)
    src = torch.where(k % 11 == 3, a, torch.where(k % 11 == 4, b, src))
    src = torch.where(k % 7 == 0, dst, src)
    dup = (k % 5 == 0) & (k > 0)
    dup[1:] &= dst[1:] == dst[:-1]
    src[1:] = torch.where(dup[1:], src[:-1], src[1:])
    return torch.stack((src, dst))[:, torch.randperm(dst.numel(), generator=g)]


def copied_rows(N):
    """(original, copy) node pair of exact_features."""
    return N // 3, N - N // 3 - 1


def offset_channels(ci):
    return sorted({0, ci // 2})


def exact_features(N, ci, g):
    """(N, ci) fp32: integers in [-4, 4], the last three rows zero, row copied_rows(N)[1] a copy of [0], then OFFSET
    added to the offset channels (so the zero rows are zero elsewhere)."""
    x = torch.randint(-4, 5, (N, ci), generator=g).float()
    x[N - 3:] = 0
    a, b = copied_rows(N)
    x[b] = x[a]
    x[:, offset_channels(ci)] += OFFSET
    return x


def exact_fixture(N, ci, co, act, slope, train, seed, hub=False):
    """(EdgConv module on the CPU, x, edge_index, upstream gradient) of the exact tests: every P, Q and z is exact
    in fp32 whatever the summation order (|z| < 2^20 in sixteenths).

    Linear weights and biases in sixteenths.  Output channel 1 is dead (weight and bias 0: z == 0, a zero batch
    variance in train mode).  The offset input channels carry OFFSET in x: their W1 column is 0 except in the last
    output channel, so every other channel's P and Q carry +-W2 * OFFSET that cancels in z = P_i + Q_j exactly; the
    last output channel (C_out >= 3) reads only the first offset channel of the source, z = x_j + b, a channel of
    |mean| / std ~ 400 whose distinct values lie at least 1 apart.  BatchNorm gammas cycle through exact_util.GAMMAS (channel 2: gamma = 0, every edge ties).
    Eval (train False): eps = 0, running mean and beta in eighths, running variance in {1/4, 1, 4} - every u = s z + t
    is exact too.  Train: the default eps, beta in odd eighths (no z sits at the batch mean at beta = 0), running
    statistics as in eval (the update rule is checked on them); under a V-shaped activation (PReLU weight < 0) the
    un-centred channel gets gamma = 0, because the two branches of the V put values of that channel within
    edge_tie_mask's bound (1e-4 |s| |z|, |z| ~ OFFSET) of each other.  Upstream gradient: quarters in [-1, 1]."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    import exact_util as eu
    g = torch.Generator().manual_seed(seed)
    x = exact_features(N, ci, g)
    ei = exact_graph(N, hub, g)
    mod = S.EdgConv(ci, co, act, "batch", True)
    lin = mod.nn[0]
    with torch.no_grad():
        w = eu.sixteenths(lin.weight.shape, g)
        b = eu.sixteenths((co,), g)
        off = offset_channels(ci)
        w[:, off] = 0
        if co >= 3:
            w[co - 1] = 0
            w[co - 1, off[0]] = 1.0
            w[co - 1, ci + off[0]] = 1.0
        if co >= 2:
            w[1] = 0
            b[1] = 0
        lin.weight.copy_(w)
        lin.bias.copy_(b)
        for m in mod.nn:
            if isinstance(m, torch.nn.PReLU):
                m.weight.fill_(slope)
            if isinstance(m, torch.nn.BatchNorm1d):
                m.weight.copy_(torch.tensor(eu.GAMMAS)[torch.arange(co) % len(eu.GAMMAS)])
                if train and co >= 3 and slope is not None and slope < 0:
                    m.weight[co - 1] = 0.0
                if train:
                    m.bias.copy_((2 * torch.randint(-4, 4, (co,), generator=g) + 1).float() / 8)
                else:
                    m.eps = 0.0
                    m.bias.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_mean.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_var.copy_(4.0 ** torch.randint(-1, 2, (co,), generator=g).float())
    gout = torch.randint(-4, 5, (N, co), generator=g).float() / 4
    return mod.train(train), x, ei, gout


# name: (N, C_in, C_out, hub row, seed); tests/test_sparse_edgeconv_shapes_gpu.py's table says what each reaches.
# Each seed is the first, counting up from the shape's index, whose train-mode fixtures meet the preconditions.
EXACT_SHAPES = {
    "n33-co2": (33, 3, 2, False, 1),
    "n97-co1": (97, 5, 1, False, 2),
    "n159-co32": (159, 7, 32, True, 3),
    "n256-co33": (256, 16, 33, False, 4),
    "n543-co64": (543, 9, 64, False, 6),
    "n2048-ci128": (2048, 128, 16, False, 6),
    "n1313-co65": (1313, 12, 65, True, 7),
    "n1030-ci130-co129": (1030, 130, 129, True, 53),
}
ALL_ACTS = (("relu", None), ("leakyrelu", None), ("prelu", 0.25), ("prelu", -0.5))
BIG_SHAPES = ("n1313-co65", "n1030-ci130-co129")     # every activation; relu elsewhere


def exact_cases():
    """(shape name, act, PReLU slope, train) of every exact case."""
    out = []
    for name in EXACT_SHAPES:
        for act, slope in (ALL_ACTS if name in BIG_SHAPES else ALL_ACTS[:1]):
            for train in (False, True):
                out.append((name, act, slope, train))
    return out
