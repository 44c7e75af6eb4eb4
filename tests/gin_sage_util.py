"""Shared pieces of the sparse GIN / GraphSAGE tests and of their golden generator (no GPU needed here):

- GINConvStandIn / SAGEConvStandIn / install_reference_stand_ins: torch_geometric's GINConv(nn, eps=0.,
  train_eps=False) and the older SAGEConv(in_channels, out_channels, normalize, bias) layout that the reference
  subclasses (gcn_lib/sparse/torch_vertex.py:136-205), restated over oracle/ref_shims.py's MessagePassing and put in
  place of ref_shims' placeholders before the reference is imported, so that the unmodified reference's GinConv,
  SAGEConv and RSAGEConv execute.  GINConv: out = nn(sum_{j->i} x_j + (1 + eps) x_i), the sum over edge_index as
  given, eps a buffer.  SAGEConv: weight (in, out) and bias (out) uniform in +-1/sqrt(in), mean aggregation,
  propagate handing x to update() as torch_geometric does.
- gin_aggr / sage_aggr: the aggregations restated functionally on any device and dtype (the fp64 references of the
  GPU tests): remove_self_loops + add_self_loops + mean for SAGE, exactly as torch_geometric composes them.
- exact_graph / exact_features: the exact-arithmetic fixtures of tests/test_gin_sage_gpu.py.
- gin_aggr_chunked / sage_aggr_chunked / gin_sage_grad_chunked: the same aggregations and their gradient written out,
  in fp64 over a whole ogbn-sized graph a chunk of edges at a time (tests/test_gin_sage_scale_gpu.py).
- loop_positions / plant_self_loops / exact_magnitudes: the self loops that test file plants at the hub kernels'
  segment and ballot boundaries, and the bounds that keep its integer fixtures exact in fp32.
"""
import sys

import torch

from oracle import ref_shims


class GINConvStandIn(ref_shims.MessagePassing):
    """torch_geometric.nn.GINConv(nn, eps=0., train_eps=False)."""

    def __init__(self, nn, eps=0.0, train_eps=False, **kw):
        super().__init__(aggr="add", **kw)
        self.nn = nn
        self.initial_eps = eps
        if train_eps:
            self.eps = torch.nn.Parameter(torch.Tensor([eps]))
        else:
            self.register_buffer("eps", torch.Tensor([eps]))

    def forward(self, x, edge_index, size=None):
        out = self.propagate(edge_index, x=x, size=size)
        out = out + (1 + self.eps) * x
        return self.nn(out)


class SAGEConvStandIn(ref_shims.MessagePassing):
    """torch_geometric.nn.SAGEConv(in_channels, out_channels, normalize=False, bias=True) in the layout the
    reference's subclass reads (self.weight (in, out), self.bias, self.normalize); forward, message and update are
    the subclass's own."""

    def __init__(self, in_channels, out_channels, normalize=False, bias=True, **kw):
        super().__init__(aggr="mean", **kw)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.normalize = normalize
        self.weight = torch.nn.Parameter(torch.Tensor(in_channels, out_channels))
        if bias:
            self.bias = torch.nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        bound = 1.0 / in_channels ** 0.5
        for p in (self.weight, self.bias):
            if p is not None:
                p.data.uniform_(-bound, bound)

    def propagate(self, edge_index, size=None, x=None):
        n = x.size(0) if size is None else size[1]
        msg = self.message(x.index_select(0, edge_index[1]), x.index_select(0, edge_index[0]))
        return self.update(ref_shims.scatter(msg, edge_index[1], 0, dim_size=n, reduce="mean"), x)


def install_reference_stand_ins():
    """ref_shims' stand-in modules with GINConv and SAGEConv; call before ref_shims.load_reference()."""
    ref_shims._install_stubs()
    sys.modules["torch_geometric.nn"].GINConv = GINConvStandIn
    sys.modules["torch_geometric.nn"].SAGEConv = SAGEConvStandIn


def gin_aggr(x, edge_index, eps=0.0):
    """sum over every edge (j -> i) of x_j, plus (1 + eps) x_i, in x's dtype and on x's device."""
    src, dst = edge_index[0].long().to(x.device), edge_index[1].long().to(x.device)
    agg = torch.zeros_like(x).index_add_(0, dst, x.index_select(0, src))
    return agg + (1 + eps) * x


def sage_aggr(x, edge_index, relative=False):
    """remove_self_loops + add_self_loops, then the mean of x_j (x_j - x_i when relative) over each row's edges."""
    src, dst = edge_index[0].long().to(x.device), edge_index[1].long().to(x.device)
    keep = src != dst
    loop = torch.arange(x.shape[0], device=x.device)
    src, dst = torch.cat((src[keep], loop)), torch.cat((dst[keep], loop))
    msg = x.index_select(0, src) - (x.index_select(0, dst) if relative else 0)
    s = torch.zeros_like(x).index_add_(0, dst, msg)
    cnt = torch.zeros(x.shape[0], dtype=x.dtype, device=x.device).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return s / cnt.unsqueeze(1)


# ---- exact-arithmetic fixtures ----------------------------------------------------------------------------------
# Row kinds of exact_graph: (non-self in-degree, self loops on the row).  c_i = non-self + 1 is 1, 2, 4 or 8, so every
# mean is exact; one row carries several self loops, one row is empty, rows repeat a source (duplicate edges).
EXACT_ROWS = ((0, 0), (0, 1), (0, 3), (1, 0), (1, 1), (3, 0), (3, 2), (7, 0), (7, 1))


def exact_graph(N, g, hub=0):
    """(2, E) int64 over N nodes, in shuffled order: row r has EXACT_ROWS[r % 9] edges (random sources other than r,
    every third one repeating its predecessor, plus the self loops); with hub > 0 row N - 1 instead takes
    hub - 1 non-self edges and 2 self loops (hub - 1 + 1 a power of two keeps its mean exact)."""
    src, dst = [], []
    for r in range(N):
        n_other, n_self = EXACT_ROWS[r % len(EXACT_ROWS)]
        if hub and r == N - 1:
            n_other, n_self = hub - 1, 2
        s = torch.randint(0, N - 1, (n_other,), generator=g)
        s = s + (s >= r).long()                     # never r itself
        if n_other > 1:
            s[2::3] = s[1::3][:len(s[2::3])]        # duplicates
        s = torch.cat((s, torch.full((n_self,), r)))
        src.append(s)
        dst.append(torch.full((s.numel(),), r))
    ei = torch.stack((torch.cat(src), torch.cat(dst)))
    return ei[:, torch.randperm(ei.shape[1], generator=g)]


def exact_features(N, C, g):
    """(N, C) fp32 integers in [-4, 4]."""
    return torch.randint(-4, 5, (N, C), generator=g).float()


# ---- whole-graph fp64 references, a chunk of edges at a time --------------------------------------------------------
# At the ogbn shapes one gather of every edge's row would take tens of GiB; the chunked forms keep one chunk's gathered
# rows (in the reference's dtype) below REF_CHUNK_BYTES and sum with index_add_ into one (N, C) accumulator.
REF_CHUNK_BYTES = 2**30


def edge_chunks(edge_index, width, device, drop_self=False, itemsize=8):
    """(src, dst) int64 on `device` for consecutive chunks of edge_index's edges, each chunk small enough that its
    gathered (chunk, width) rows of `itemsize`-byte values stay below REF_CHUNK_BYTES; drop_self: without the self
    loops."""
    step = max(1, REF_CHUNK_BYTES // (itemsize * max(width, 1)))
    for e0 in range(0, edge_index.shape[1], step):
        src, dst = (t.long().to(device) for t in edge_index[:, e0:e0 + step])
        if drop_self:
            keep = src != dst
            src, dst = src[keep], dst[keep]
        yield src, dst


def sage_counts(edge_index, N, device=None, dtype=torch.float64):
    """c_i = (number of edges j -> i with j != i) + 1: the size of row i's set after remove_self_loops +
    add_self_loops, counted on edge_index (not on any CSR)."""
    device = edge_index.device if device is None else device
    c = torch.ones(N, dtype=dtype, device=device)
    for _src, dst in edge_chunks(edge_index, 1, device, drop_self=True):
        c.index_add_(0, dst, torch.ones_like(dst, dtype=dtype))
    return c


def gin_aggr_chunked(x, edge_index, eps=0.0, dtype=torch.float64):
    """gin_aggr in `dtype` (x in any dtype: rows are converted as they are gathered)."""
    agg = torch.zeros(x.shape, dtype=dtype, device=x.device)
    for src, dst in edge_chunks(edge_index, x.shape[1], x.device):
        agg.index_add_(0, dst, x.index_select(0, src).to(dtype))
    return agg.add_(x.to(dtype), alpha=1 + eps)


def sage_aggr_chunked(x, edge_index, relative=False, dtype=torch.float64):
    """sage_aggr in `dtype`: s_i = sum over the edges j -> i, j != i of x_j, then (s_i + x_i) / c_i, or with
    relative (s_i - (c_i - 1) x_i) / c_i - the sum of the messages x_j - x_i over the same set, where the added self
    loop's message is 0."""
    s = torch.zeros(x.shape, dtype=dtype, device=x.device)
    for src, dst in edge_chunks(edge_index, x.shape[1], x.device, drop_self=True):
        s.index_add_(0, dst, x.index_select(0, src).to(dtype))
    c = sage_counts(edge_index, x.shape[0], x.device, dtype).unsqueeze(1)
    if relative:
        s.addcmul_(c - 1, x.to(dtype), value=-1)
    else:
        s.add_(x.to(dtype))
    return s.div_(c)


def gin_sage_grad_chunked(rule, grad_out, edge_index, eps=0.0, dtype=torch.float64):
    """The gradient w.r.t. x of sum(out * grad_out) for out = gin_aggr / sage_aggr, written out: every edge j -> i
    (j != i for SAGE) sends g_i (GIN) or g_i / c_i (SAGE, RSAGE) to row j, and row i receives (1 + eps) g_i, g_i / c_i
    or -(c_i - 1) / c_i g_i.  In `dtype`, a chunk of edges at a time."""
    ge = grad_out.to(dtype, copy=True)
    if rule == "gin":
        gx = ge * (1 + eps)
    else:
        c = sage_counts(edge_index, ge.shape[0], ge.device, dtype).unsqueeze(1)
        ge.div_(c)
        gx = ge.clone() if rule == "sage" else ge * -(c - 1)
    for src, dst in edge_chunks(edge_index, ge.shape[1], ge.device, drop_self=rule != "gin"):
        gx.index_add_(0, src, ge.index_select(0, dst))
    return gx


# ---- self loops planted at the hub kernels' boundaries -------------------------------------------------------------
SEG_EDGES = 4096                      # _native.HUB_SEG_EDGES: edges per hub segment
BIG_ROW_LOOPS = 475_713               # on the 10^6-edge row: c = 10^6 - 475,713 + 1 = 2^19


def loop_positions(deg):
    """Which of a planted row's edges (0 .. deg - 1, in the row's order) become self loops, by the row's degree:
    1023 / 1024 all of them (c = 1 on the last one-warp row and on the first hub row); 4096 its first 32 (one full
    ballot chunk); 4097 its last (the only edge of its second segment); 8192 every other edge of its second segment
    only; 10^6 BIG_ROW_LOOPS spread evenly over all 245 segments (a count above 2^16 carried through the merge,
    c = 2^19).  None for any other degree."""
    if deg in (1023, 1024):
        return torch.arange(deg)
    if deg == 4096:
        return torch.arange(32)
    if deg == 4097:
        return torch.tensor([4096])
    if deg == 8192:
        return torch.arange(SEG_EDGES, 8192, 2)
    if deg == 10**6:
        return torch.arange(BIG_ROW_LOOPS) * deg // BIG_ROW_LOOPS
    return None


def plant_self_loops(edge_index, planted, loop_rows=(), every=97):
    """Turns edges of edge_index into self loops in place (edge_index[0] = edge_index[1]):
    - planted ({row: degree}): the edges loop_positions(degree) of the row, counted in edge_index order - the order a
      stable CSR build keeps within a row - and no other edge of the row (a loop drawn there moves to another source);
    - loop_rows: every edge of these rows;
    - of every other row, the edges at the indices of edge_index divisible by `every`.
    Returns the rows the first two rules fixed (planted rows of another degree take the third)."""
    plan = {r: loop_positions(int(d)) for r, d in planted.items()}
    plan = {r: pos for r, pos in plan.items() if pos is not None}
    plan.update({r: None for r in loop_rows})
    for r, pos in plan.items():
        at = (edge_index[1] == r).nonzero().squeeze(1)
        assert r not in planted or at.numel() == planted[r], (r, at.numel(), planted[r])
        if pos is not None:
            drawn = at[edge_index[0, at] == r]
            edge_index[0, drawn] = r - 1 if r > 0 else 1
            at = at[pos.to(at.device)]
        edge_index[0, at] = r
    idx = torch.arange(0, edge_index.shape[1], every, device=edge_index.device)
    fixed = torch.tensor(sorted(plan), dtype=edge_index.dtype, device=edge_index.device)
    idx = idx[~torch.isin(edge_index[1, idx], fixed)]
    edge_index[0, idx] = edge_index[1, idx]
    return sorted(plan)


def exact_magnitudes(edge_index, N):
    """Bounds, on integer features in [-4, 4] and upstream gradients g_i = k_i / 4 (GIN) or c_i k_i / 4 (SAGE) with
    |k_i| <= 4, of every fp32 value the GIN / SAGE kernels form, forward and backward, on this graph: (forward, the
    largest |partial sum| of a row's messages plus its own term; backward, the largest |sum| one row's gradient
    collects).  Below 2^22 every such value is a multiple of 1/16 (GIN's fl(1.25 x_i) and fl(1.25 g_i)) or 1/4 held
    exactly, in any order of the additions."""
    dev = edge_index.device
    indeg = torch.bincount(edge_index[1], minlength=N)
    outdeg = torch.bincount(edge_index[0], minlength=N)
    c = sage_counts(edge_index, N, dev, torch.float64)
    fwd = max(float(indeg.max()) * 4 + 5, float(((c - 1) * 4 * 2).max()))       # GIN; RSAGE sum - (c - 1) x_i
    bwd = float((outdeg.double() + (c - 1).clamp(min=1.25)).max())                # each scatter |k/4| <= 1
    return fwd, bwd


def sixteenths(shape, g):
    return torch.randint(-16, 17, shape, generator=g).float() / 16


def ppi_deepgcn(S, opt):
    """examples/ppi/architecture.py's DeepGCN (res or plain blocks) assembled from the drop-in sparse classes S, with
    its module layout (state_dict keys) and forward; the golden weights are loaded into it."""

    class DeepGCN(torch.nn.Module):
        def __init__(self):
            super().__init__()
            c, conv = opt["n_filters"], opt["conv"]
            args = (opt["act"], opt["norm"], opt["bias"], opt["n_heads"])
            self.n_blocks = opt["n_blocks"]
            self.head = S.GraphConv(opt["in_channels"], c, conv, *args)
            self.backbone = S.MultiSeq(*[S.ResGraphBlock(c, conv, *args, 1 if opt["block"] == "res" else 0)
                                         for _ in range(self.n_blocks - 1)])
            fusion_dims = c * self.n_blocks
            self.fusion_block = S.MLP([fusion_dims, 1024], opt["act"], None, opt["bias"])
            self.prediction = torch.nn.Sequential(
                S.MLP([1 + fusion_dims, 512], opt["act"], opt["norm"], opt["bias"]),
                torch.nn.Dropout(p=opt["dropout"]),
                S.MLP([512, 256], opt["act"], opt["norm"], opt["bias"]), torch.nn.Dropout(p=opt["dropout"]),
                S.MLP([256, opt["n_classes"]], None, None, opt["bias"]))

        def forward(self, x, edge_index):
            feats = [self.head(x, edge_index)]
            for i in range(self.n_blocks - 1):
                feats.append(self.backbone[i](feats[-1], edge_index)[0])
            feats = torch.cat(feats, 1)
            fusion, _ = torch.max(self.fusion_block(feats), 1, keepdim=True)
            return self.prediction(torch.cat((feats, fusion), 1))

    return DeepGCN()
