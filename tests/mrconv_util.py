"""Shared pieces of the sparse MRConv tests (no GPU needed here):

- mr_aggr_chunked / mr_grad_chunked / MRAggr64: the reference's aggregation scatter(aggr, x[src] - x[dst], dst) (empty
  rows 0) and its gradient written out, in fp64 over a whole graph a chunk of edges at a time; a max or min routes its
  gradient to the first edge of the row, in edge_index order, that attains it (torch_scatter's scatter_max / min).
  MRAggr64 is the autograd node of the two, the fp64 stand-in of MRConv's aggregation in restated models.
- raw_aggr_chunked: the same over the raw source rows, scatter(aggr, x[src], dst), what dgcn_genconv_aggregate
  returns in raw-message mode, and raw_grad_chunked its gradient.
- mr_graph / mr_features: the exact-arithmetic fixtures of tests/test_mrconv_sparse_gpu.py: planted row lengths at
  the one-warp / hub / segment boundaries, repeated sources, self loops, twin nodes and an all-equal channel.
- mr_error_bound: the random-data bound 2^-24 (deg + 2) (sum_j |x_j| + deg |x_i|) per row and channel.
- reference_mrconv: an MRConv's forward restated on MRAggr64 (for fp64 copies of whole models).
"""
import torch

from gin_sage_util import edge_chunks

AGGRS = ("add", "mean", "max", "min")
# planted row lengths: short rows, one warp's 32-edge chunk, the last one-warp row and the first hub row
# (HUB_MIN_DEGREE = 1024), one and two hub segments (HUB_SEG_EDGES = 4096) and one edge past them
ROW_LENGTHS = (0, 1, 2, 31, 32, 33, 1023, 1024, 4096, 4097, 8193)
POW2_LENGTHS = (0, 1, 2, 32, 1024, 4096, 8192)          # mean: S / deg and every g / deg exact
BACKGROUND = (0, 1, 2, 3, 5, 8)                           # the other rows' in-degrees ...
POW2_BACKGROUND = (0, 1, 2, 4, 8)                         # ... of a mean graph
FEATURE_MAX = 8                                           # mr_features: integers in [-8, 8]


def _pick(aggr, msg):
    return msg if aggr != "min" else -msg


def _scatter_chunked(x, edge_index, aggr, relative, dtype):
    N, C = x.shape
    dev = x.device
    deg = torch.bincount(edge_index[1].to(dev), minlength=N)
    if aggr in ("add", "mean"):
        acc = torch.zeros((N, C), dtype=dtype, device=dev)
    else:
        acc = torch.full((N, C), -float("inf"), dtype=dtype, device=dev)
    for src, dst in edge_chunks(edge_index, C, dev):
        msg = x.index_select(0, src).to(dtype)
        if relative:
            msg -= x.index_select(0, dst).to(dtype)
        if aggr in ("add", "mean"):
            acc.index_add_(0, dst, msg)
        else:
            acc.scatter_reduce_(0, dst.unsqueeze(1).expand_as(msg), _pick(aggr, msg), "amax")
    if aggr == "mean":
        acc /= deg.clamp(min=1).to(dtype).unsqueeze(1)
    elif aggr in ("max", "min"):
        acc = _pick(aggr, acc)
        acc[deg == 0] = 0
    return acc


def mr_aggr_chunked(x, edge_index, aggr, dtype=torch.float64):
    """scatter(aggr, x[src] - x[dst], dst) in `dtype`, an empty row 0."""
    return _scatter_chunked(x, edge_index, aggr, True, dtype)


def raw_aggr_chunked(x, edge_index, aggr, dtype=torch.float64):
    """scatter(aggr, x[src], dst) in `dtype`, an empty row 0."""
    return _scatter_chunked(x, edge_index, aggr, False, dtype)


def first_winner(x, edge_index, aggr):
    """(N, C) int64: for max / min, the position in edge_index of the first edge j -> i whose x_j attains row i's
    max / min in channel c (x_i is common to the row's edges, so it does not change the choice); E on empty rows."""
    N, C = x.shape
    dev = x.device
    E = edge_index.shape[1]
    best = _scatter_chunked(x, edge_index, aggr, False, x.dtype)
    first = torch.full((N, C), E, dtype=torch.int64, device=dev)
    e0 = 0
    for src, dst in edge_chunks(edge_index, C, dev):
        hit = x.index_select(0, src) == best.index_select(0, dst)
        pos = torch.arange(e0, e0 + src.numel(), device=dev).unsqueeze(1).expand_as(hit)
        first.scatter_reduce_(0, dst.unsqueeze(1).expand_as(hit), torch.where(hit, pos, E), "amin")
        e0 += src.numel()
    return first


def raw_grad_chunked(x, edge_index, aggr, grad_out, dtype=torch.float64):
    """The gradient w.r.t. x of sum(grad_out * raw_aggr_chunked(x)): every edge j -> i sends g_i (add), g_i / deg_i
    (mean) or, for max / min, g_i where it is row i's first winning edge, to row j."""
    N, C = x.shape
    dev = x.device
    g = grad_out.to(dtype, copy=True)
    if aggr == "mean":
        g /= torch.bincount(edge_index[1].to(dev), minlength=N).clamp(min=1).to(dtype).unsqueeze(1)
    first = first_winner(x, edge_index, aggr) if aggr in ("max", "min") else None
    gx = torch.zeros((N, C), dtype=dtype, device=dev)
    e0 = 0
    for src, dst in edge_chunks(edge_index, C, dev):
        ge = g.index_select(0, dst)
        if first is not None:
            pos = torch.arange(e0, e0 + src.numel(), device=dev).unsqueeze(1)
            ge = torch.where(first.index_select(0, dst) == pos, ge, torch.zeros_like(ge))
        gx.index_add_(0, src, ge)
        e0 += src.numel()
    return gx


def mr_grad_chunked(x, edge_index, aggr, grad_out, dtype=torch.float64):
    """The gradient w.r.t. x of sum(grad_out * mr_aggr_chunked(x)): raw_grad_chunked for the x_j, and row i's own
    -deg_i g_i (add) or -g_i (mean, max, min on a non-empty row) for the x_i of its edges."""
    deg = torch.bincount(edge_index[1].to(x.device), minlength=x.shape[0]).to(dtype).unsqueeze(1)
    own = deg if aggr == "add" else (deg > 0).to(dtype)
    return raw_grad_chunked(x, edge_index, aggr, grad_out, dtype) - own * grad_out.to(dtype)


class MRAggr64(torch.autograd.Function):
    """mr_aggr_chunked with mr_grad_chunked as its backward, in x's dtype (fp64 in the tests)."""

    @staticmethod
    def forward(ctx, x, edge_index, aggr):
        ctx.save_for_backward(x)
        ctx.edge_index, ctx.aggr = edge_index, aggr
        return mr_aggr_chunked(x, edge_index, aggr, x.dtype)

    @staticmethod
    def backward(ctx, grad_out):
        (x,) = ctx.saved_tensors
        return mr_grad_chunked(x, ctx.edge_index, ctx.aggr, grad_out, x.dtype), None, None


def reference_mrconv(layer):
    """forward(x, edge_index) of an MRConv `layer` restated on MRAggr64: layer.nn(cat[x, aggr(x_j - x_i)])."""
    def forward(x, edge_index):
        return layer.nn(torch.cat([x, MRAggr64.apply(x, edge_index, layer.aggr)], dim=1))
    return forward


def use_reference_mrconv(model):
    """Every MRConv in `model` (an fp64 copy) computes through reference_mrconv from here on."""
    from deep_gcns_torch_b200.gcn_lib.sparse import MRConv
    for m in model.modules():
        if isinstance(m, MRConv):
            m.forward = reference_mrconv(m)
    return model


# ---- exact-arithmetic fixtures -------------------------------------------------------------------------------------
def planted_rows(N, lengths, reverse=False):
    """{row: length}: the lengths at rows spread evenly over 0 .. N - 1 (the first at row 0, the last at row N - 1),
    in reverse order when `reverse`."""
    lengths = tuple(reversed(lengths)) if reverse else tuple(lengths)
    n = len(lengths)
    return {round(k * (N - 1) / (n - 1)): L for k, L in enumerate(lengths)}


TWINS = (3, 5)        # mr_features gives node 5 node 3's row; mr_graph adds the edges 3 -> r and 5 -> r to rows


def mr_graph(N, g, lengths=ROW_LENGTHS, background=BACKGROUND, reverse=False):
    """(2, E) int64, rows in shuffled order.  The planted_rows get their lengths, every other row the in-degree
    background[row % len(background)].  Sources are random, except: every 5th edge of a row repeats its
    predecessor's source, every 7th is a self loop, and rows of at least 3 edges take both twins (3 and 5) as their
    first two sources, so their max and min tie across distinct sources."""
    plant = planted_rows(N, lengths, reverse)
    src, dst = [], []
    for r in range(N):
        d = plant.get(r, background[r % len(background)])
        s = torch.randint(0, N, (d,), generator=g)
        if d >= 3:
            s[0], s[1] = TWINS
        k = torch.arange(d)
        s[1:] = torch.where(k[1:] % 5 == 0, s[:-1], s[1:])
        s[k % 7 == 6] = r
        src.append(s)
        dst.append(torch.full((d,), r))
    ei = torch.stack((torch.cat(src), torch.cat(dst)))
    # rows in random order, each row's edges kept together in their order (the order a stable CSR build keeps)
    key = torch.randperm(N, generator=g)[ei[1]]
    return ei[:, torch.sort(key, stable=True).indices]


def mr_features(N, C, g):
    """(N, C) fp32 integers in [-FEATURE_MAX, FEATURE_MAX]; channel 0 all equal (every edge of a row ties) and
    node TWINS[1]'s row a copy of node TWINS[0]'s."""
    x = torch.randint(-FEATURE_MAX, FEATURE_MAX + 1, (N, C), generator=g).float()
    x[:, 0] = 3.0
    x[TWINS[1]] = x[TWINS[0]]
    return x


def quarters(shape, g, k=8):
    """Upstream gradients k' / 4, k' integer in [-k, k]."""
    return torch.randint(-k, k + 1, shape, generator=g).float() / 4


def exact_bounds(edge_index, N, C_in, c_out, g_max=2.0):
    """Bounds on every partial sum the fixtures form, in units of the smallest step they hold (all must stay below
    2^24 for fp32 to hold them exactly in any order): (aggregate: add's deg * (|x_j| + |x_i|) in units of 1;
    backward: a row's collected g / deg plus its own deg * |g|, in quarters; module Linear: 2 C_in products of a
    weight in eighths with |x| or |x_j|, in eighths)."""
    deg = torch.bincount(edge_index[1], minlength=N).double()
    outdeg = torch.bincount(edge_index[0], minlength=N).double()
    fwd = float((deg * 2 * FEATURE_MAX).max())
    bwd = float(((outdeg + deg) * g_max).max()) * 4
    lin = (C_in * FEATURE_MAX + C_in * fwd) * 8
    return fwd, bwd, lin


# ---- random data ---------------------------------------------------------------------------------------------------
def mr_error_bound(x, edge_index, aggr):
    """(N, C) fp64 bound on |fp32 - exact| of MRConv's x_j = aggr(x_j - x_i) computed as the kernel does: an fp32 sum
    of the row's deg x_j in any order of depth at most deg (each addition rounds to within 2^-24 of its result, which
    is at most sum_j |x_j|), then minus deg x_i (one rounding each for the product and the difference) or divided by
    deg and minus x_i:  2^-24 (deg + 2) (sum_j |x_j| + deg |x_i|), over deg for mean.  max / min are exact up to the
    one rounding of the difference: 2^-24 |x_j - x_i| <= 2^-24 (max_j |x_j| + |x_i|)."""
    N = x.shape[0]
    deg = torch.bincount(edge_index[1].to(x.device), minlength=N).double().unsqueeze(1)
    xa = x.abs().double()
    if aggr in ("max", "min"):
        return 2.0**-24 * (raw_aggr_chunked(xa, edge_index, "max") + xa) * (deg > 0)
    b = 2.0**-24 * (deg + 2) * (raw_aggr_chunked(xa, edge_index, "add") + deg * xa)
    return b / deg.clamp(min=1) if aggr == "mean" else b
