"""Node-partitioned GENConv over several GPUs (SURVEY.md 8e, BASELINE config 5).

New functionality - the reference has no multi-GPU sparse path (its products training drops
cross-partition edges, utils/data_util.py:43-61); parity oracle = the single-device full-graph
forward.  Destination nodes (CSR rows) are split into `world` contiguous ranges.  Rank r owns
x rows [lo_r, hi_r) and every edge whose TARGET lies in its range; sources outside the range
are its halo.  Everything a rank needs is derived ON ITS DEVICE from the edges it owns (sort /
unique / searchsorted; no pass over the global edge list on the host, no N-sized table).

Per layer (`aggregate_partitioned`), with persistent buffers - nothing is allocated or
concatenated in steady state:

    xbuf = [ local rows (n_local, C) | halo rows (n_halo, C) ]     one buffer, written in place
    comm stream : dgcn_gather_rows(local rows peers asked for) -> send buffer
                  all_to_all_single(send -> xbuf[n_local:])        NCCL over NVLink, async
    main stream : dgcn_genconv_aggregate(rows = interior)          rows whose sources are all local
                  wait(all_to_all)
                  dgcn_genconv_aggregate(rows = boundary)          rows that read halo rows (+ hub rows)

The exchange is the only collective of the forward; BatchNorm1d (eval) / MLP are row-local.
Training: `HaloExchange` / `PartitionedAggregate` are autograd nodes, the backward of the
exchange is the reverse all-to-all followed by a scatter-add into the rows that were sent.
One process per GPU.
"""
import torch
import torch.distributed as dist


def high_priority_group(ranks=None):
    """A NCCL process group whose kernels run on a high-priority stream: a halo all-to-all launched next to a
    grid-filling aggregate kernel is scheduled as CTAs retire instead of after the whole grid has been dispatched.
    (gloo / single process: the default group.)"""
    if not dist.is_initialized() or dist.get_backend() != "nccl":
        return None
    opts = dist.ProcessGroupNCCL.Options()
    opts.is_high_priority_stream = True
    return dist.new_group(ranks=ranks, backend="nccl", pg_options=opts)


def row_ranges(num_nodes, world):
    """Contiguous, balanced row ranges [(lo, hi)] * world."""
    base, rem = divmod(num_nodes, world)
    out, lo = [], 0
    for r in range(world):
        hi = lo + base + (1 if r < rem else 0)
        out.append((lo, hi))
        lo = hi
    return out


class GraphPartition:
    """Everything rank `rank` needs about its share of the graph (index tensors on `device`)."""

    def __init__(self, edge_index, num_nodes, rank, world, device=None):
        """From the GLOBAL edge list (2, E) (any device): keeps the edges whose target this rank owns."""
        device = torch.device(device) if device is not None else edge_index.device
        ei = edge_index.to(device)
        lo, hi = row_ranges(num_nodes, world)[rank]
        mine = (ei[1] >= lo) & (ei[1] < hi)
        self.edge_ids = mine.nonzero(as_tuple=True)[0]              # positions in the global edge list
        self._build(ei[0][mine], ei[1][mine], num_nodes, rank, world, device)

    @classmethod
    def from_local_edges(cls, src, dst, num_nodes, rank, world, device=None):
        """From the edges this rank owns already (global ids, every dst inside the rank's range)."""
        self = cls.__new__(cls)
        device = torch.device(device) if device is not None else src.device
        self.edge_ids = None
        self._build(src.to(device), dst.to(device), num_nodes, rank, world, device)
        return self

    def _build(self, src, dst, num_nodes, rank, world, device):
        self.rank, self.world, self.num_nodes, self.device = rank, world, num_nodes, device
        self.ranges = row_ranges(num_nodes, world)
        lo, hi = self.ranges[rank]
        self.lo, self.hi, self.n_local = lo, hi, hi - lo
        if src.numel() and (int(dst.min()) < lo or int(dst.max()) >= hi):
            raise RuntimeError("GraphPartition: an edge's target lies outside this rank's row range")
        remote = (src < lo) | (src >= hi)
        halo_nodes = torch.unique(src[remote])                      # sorted global ids => grouped by owner
        bounds = torch.tensor([r[0] for r in self.ranges] + [num_nodes], device=device)
        owner = torch.bucketize(halo_nodes, bounds, right=True) - 1
        self.recv_counts = torch.bincount(owner, minlength=world).tolist()     # one small device->host read
        self.n_halo = int(halo_nodes.numel())
        # local numbering of sources: own rows first, then halo rows in the order they arrive
        src_local = torch.where(remote, self.n_local + torch.searchsorted(halo_nodes, src), src - lo)
        dst_local = dst - lo
        self.local_edge_index = torch.stack((src_local, dst_local))
        self.halo_nodes = halo_nodes                                # global ids I need, grouped by owner rank
        # rows that read at least one halo row must wait for the exchange; the others overlap it
        touches_halo = torch.zeros(self.n_local, dtype=torch.bool, device=device)
        touches_halo[dst_local[remote]] = True
        self.interior_rows = (~touches_halo).nonzero(as_tuple=True)[0].to(torch.int32)
        self.boundary_rows = touches_halo.nonzero(as_tuple=True)[0].to(torch.int32)
        self.n_remote_edges = int(remote.sum())
        self.send_rows = None                                       # filled by exchange_halo_lists()
        self.send_counts = None
        self._csr = None
        self._buffers = {}
        self._comm_stream = None
        self.group = None

    # ---- one-time setup --------------------------------------------------------------------------
    def exchange_halo_lists(self, group=None):
        """Tell every owner which of its rows I need; learn which of mine the others need."""
        world = self.world
        offs = [0]
        for c in self.recv_counts:
            offs.append(offs[-1] + c)
        want = torch.cat([self.halo_nodes[offs[r]:offs[r + 1]] - self.ranges[r][0] for r in range(world)]) \
            if world > 0 else self.halo_nodes
        counts = torch.tensor(self.recv_counts, dtype=torch.long)
        comm_dev = self.device if dist.get_backend(group) == "nccl" else torch.device("cpu")
        theirs = torch.empty(world, dtype=torch.long, device=comm_dev)
        dist.all_to_all_single(theirs, counts.to(comm_dev), group=group)
        self.send_counts = [int(v) for v in theirs.cpu()]
        recv = torch.empty(sum(self.send_counts), dtype=torch.long, device=comm_dev)
        dist.all_to_all_single(recv, want.to(comm_dev), output_split_sizes=self.send_counts,
                               input_split_sizes=self.recv_counts, group=group)
        self.send_rows = recv.to(self.device, torch.int32)          # local row ids, grouped by destination rank
        self.group = group                                          # the exchanges of this partition use it too
        return self

    def csr(self):
        if self._csr is None:
            from . import _native
            self._csr = _native.csr_build(self.local_edge_index, self.n_local)
        return self._csr

    # ---- persistent buffers ------------------------------------------------------------------------
    def buffers(self, channels, slot=0):
        """(xbuf (n_local + n_halo, C), send (n_send, C)) - allocated once per (C, slot); two slots give a
        layer stack its ping-pong pair (layer l reads slot l&1, its MLP writes slot (l+1)&1)."""
        key = (int(channels), int(slot))
        buf = self._buffers.get(key)
        if buf is None:
            xbuf = torch.empty((self.n_local + self.n_halo, channels), dtype=torch.float32, device=self.device)
            send = torch.empty((int(self.send_rows.numel()), channels), dtype=torch.float32, device=self.device)
            buf = self._buffers[key] = (xbuf, send)
        return buf

    def local_rows(self, channels, slot=0):
        """View of the local-row region of the persistent buffer: producers write the layer input here."""
        return self.buffers(channels, slot)[0][:self.n_local]

    def comm_stream(self):
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(self.device, priority=-1)      # ahead of the aggregate's grid
        return self._comm_stream

    def halo_bytes(self, channels):
        """Bytes this rank receives per exchange = n_halo * C * 4 (every halo row arrives exactly once)."""
        return self.n_halo * channels * 4


# ---- exchange ------------------------------------------------------------------------------------
def _pack(x_local, rows, out=None):
    if x_local.is_cuda:
        from . import _native
        return _native.gather_rows(x_local, rows, out=out)
    res = x_local.index_select(0, rows.long())                      # host-logic tests (gloo)
    if out is not None:
        out.copy_(res)
        return out
    return res


def start_halo_exchange(part, channels, slot=0, group=None):
    """Pack + all-to-all of the rows in part.local_rows(C, slot) into the halo region of the same buffer.
    CUDA: runs on the partition's communication stream behind everything queued on the current stream and
    returns a handle whose wait() makes the CURRENT stream wait for the halo.  CPU (gloo): synchronous."""
    xbuf, send = part.buffers(channels, slot)
    local, halo = xbuf[:part.n_local], xbuf[part.n_local:]
    group = group if group is not None else part.group
    if not xbuf.is_cuda:
        _pack(local, part.send_rows, out=send)
        dist.all_to_all_single(halo, send, output_split_sizes=part.recv_counts, input_split_sizes=part.send_counts,
                               group=group)
        return None
    main, comm = torch.cuda.current_stream(part.device), part.comm_stream()
    ready = torch.cuda.Event()
    ready.record(main)
    with torch.cuda.stream(comm):
        comm.wait_event(ready)
        _pack(local, part.send_rows, out=send)
        work = dist.all_to_all_single(halo, send, output_split_sizes=part.recv_counts,
                                      input_split_sizes=part.send_counts, group=group, async_op=True)
    return work


def halo_exchange(x_local, part, gather=None, group=None):
    """[local rows | halo rows] as a NEW tensor in x_local's dtype (simple, allocation per call): packs the rows
    the peers asked for and swaps them all-to-all.  The persistent-buffer path is start_halo_exchange()."""
    group = group if group is not None else part.group
    send = gather(x_local, part.send_rows) if gather is not None else _pack(x_local, part.send_rows)
    recv = torch.empty((part.n_halo, x_local.shape[1]), dtype=x_local.dtype, device=x_local.device)
    dist.all_to_all_single(recv, send, output_split_sizes=part.recv_counts, input_split_sizes=part.send_counts,
                           group=group)
    return torch.cat((x_local, recv), 0)


class HaloExchange(torch.autograd.Function):
    """x_local (n_local, C) -> [local | halo] (n_local + n_halo, C), differentiable: the gradient of a halo row
    travels back to its owner (reverse all-to-all) and is added to the gradient of the row that was sent."""

    @staticmethod
    def forward(ctx, x_local, part, group):
        ctx.part, ctx.group = part, group
        return halo_exchange(x_local.contiguous(), part, group=group)

    @staticmethod
    def backward(ctx, grad):
        part = ctx.part
        g_local = grad[:part.n_local].clone()
        g_halo = grad[part.n_local:].contiguous()
        back = torch.empty((int(part.send_rows.numel()), grad.shape[1]), dtype=grad.dtype, device=grad.device)
        dist.all_to_all_single(back, g_halo, output_split_sizes=part.send_counts, input_split_sizes=part.recv_counts,
                               group=ctx.group if ctx.group is not None else part.group)
        g_local.index_add_(0, part.send_rows.long(), back)
        return g_local, None, None


class PartitionedAggregate(torch.autograd.Function):
    """x_dst + MsgNorm(aggregate(relu(x_src[src]) + eps)) on this rank's CSR with separate source / destination
    row sets (dgcn_genconv_aggregate / _backward); scalars t, p, y, msg_scale as in GenMessagePassing."""

    @staticmethod
    def forward(ctx, x_src, x_dst, part, aggr, eps, learn_t, t, p, y, msg_scale):
        from . import _native
        prm, _keep = _native.genconv_params(aggr, t, p, y, eps, msg_scale, add_residual=True)
        ctx.part, ctx.cfg, ctx.scalars = part, (aggr, eps, learn_t), (t, p, y, msg_scale)
        ctx.save_for_backward(x_src, x_dst)
        return _native.genconv_aggregate(x_src, x_dst, part.csr(), prm)

    @staticmethod
    def backward(ctx, grad_out):
        from . import _native
        x_src, x_dst = ctx.saved_tensors
        aggr, eps, learn_t = ctx.cfg
        t, p, y, msg_scale = ctx.scalars
        prm, _keep = _native.genconv_params(aggr, t, p, y, eps, msg_scale, add_residual=True)
        gsrc, gdst, _gea, gsc = _native.genconv_aggregate_backward(x_src, x_dst, ctx.part.csr(), prm,
                                                                   grad_out.contiguous(), None, softmax_grad=learn_t)
        need = ctx.needs_input_grad

        def sg(i, v, idx):
            return gsc[idx:idx + 1].clone() if (need[i] and torch.is_tensor(v)) else None
        return (gsrc if need[0] else None, gdst if need[1] else None, None, None, None, None,
                sg(6, t, 0), sg(7, p, 1), sg(8, y, 2), sg(9, msg_scale, 3))


# ---- layer-level entry points ------------------------------------------------------------------------
def aggregate_partitioned(conv, part, channels, slot=0, pre=None, out=None, overlap=True, group=None):
    """Fused message + aggregate + MsgNorm + residual of `conv` (a GENConv) on this rank's rows.  The layer
    input must already sit in part.local_rows(channels, slot) (raw h when `pre` = (scale, shift, relu) folds
    the block's norm -> relu into the kernel's reads).  Inference path: the halo all-to-all runs on the
    communication stream while the interior rows are aggregated."""
    from . import _native
    xbuf, _send = part.buffers(channels, slot)
    x_local = xbuf[:part.n_local]
    t, p, y = conv._scalars()
    scale = conv.msg_norm.msg_scale if conv.msg_norm is not None else None
    prm, _keep = _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, scale, add_residual=True)
    csr = part.csr()
    if out is None:
        out = torch.empty((part.n_local, channels), dtype=torch.float32, device=part.device)
    with torch.no_grad():
        work = start_halo_exchange(part, channels, slot, group)
        if not overlap:
            if work is not None:
                work.wait()
            return _native.genconv_aggregate(xbuf, x_local, csr, prm, out=out, pre=pre)
        _native.genconv_aggregate(xbuf, x_local, csr, prm, out=out, pre=pre, rows=part.interior_rows, skip_hubs=True)
        if work is not None:
            work.wait()
        _native.genconv_aggregate(xbuf, x_local, csr, prm, out=out, pre=pre, rows=part.boundary_rows, skip_hubs=False)
    return out


def genconv_forward_partitioned(conv, x_local, part, edge_attr_local=None, group=None):
    """GENConv.forward (gcn_lib/sparse/torch_vertex.py:62-76) on this rank's rows: halo exchange, fused
    aggregate over the local CSR, row-local MLP.  Differentiable (training path, no overlap); under
    torch.no_grad() and without edge features it takes the overlapped persistent-buffer path."""
    from . import _native
    channels = x_local.shape[1]
    if not torch.is_grad_enabled() and edge_attr_local is None:
        part.local_rows(channels).copy_(x_local)
        return conv.mlp(aggregate_partitioned(conv, part, channels, group=group))
    t, p, y = conv._scalars()
    scale = conv.msg_norm.msg_scale if conv.msg_norm is not None else None
    if edge_attr_local is not None:                                  # edge features: inference only
        with torch.no_grad():
            x_src = halo_exchange(x_local, part, group=group)
            prm, _keep = _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, scale, add_residual=True)
            ea = conv.edge_encoder(edge_attr_local) if conv.encode_edge else edge_attr_local
            return conv.mlp(_native.genconv_aggregate(x_src, x_local, part.csr(), prm, ea))
    x_src = HaloExchange.apply(x_local, part, group)
    h = PartitionedAggregate.apply(x_src, x_local, part, conv._check_aggr(), conv.eps,
                                   bool(getattr(conv, "learn_t", False)), t, p, y, scale)
    return conv.mlp(h)


# ---- locality: Cuthill-McKee style ordering ---------------------------------------------------------------
def bfs_order(edge_index, num_nodes):
    """Breadth-first (Cuthill-McKee) ordering of the undirected version of the graph, level-synchronous and
    entirely in device tensor ops: returns `order` with order[new_id] = old_id.  Nodes of a level are sorted
    by degree; components are started from their lowest-degree unvisited node.  Relabelling with
    perm = argsort(order) turns a graph with geometric / banded locality whose ids were shuffled back into
    one whose contiguous row ranges have a bounded halo (SURVEY.md 7 "Halo volume")."""
    dev = edge_index.device
    s = torch.cat((edge_index[0], edge_index[1]))
    d = torch.cat((edge_index[1], edge_index[0]))
    key = torch.argsort(s, stable=True)
    col = d[key]
    deg = torch.bincount(s, minlength=num_nodes)
    rowptr = torch.zeros(num_nodes + 1, dtype=torch.long, device=dev)
    rowptr[1:] = torch.cumsum(deg, 0)
    visited = torch.zeros(num_nodes, dtype=torch.bool, device=dev)
    by_degree = torch.argsort(deg, stable=True)
    seed_ptr = 0
    order = []
    done = 0
    while done < num_nodes:
        while bool(visited[by_degree[seed_ptr]]):
            seed_ptr += 1
        frontier = by_degree[seed_ptr:seed_ptr + 1]
        visited[frontier] = True
        while frontier.numel():
            order.append(frontier)
            done += int(frontier.numel())
            cnt = deg[frontier]
            total = int(cnt.sum())
            if total == 0:
                break
            start = torch.repeat_interleave(rowptr[frontier], cnt)
            first = torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
            nb = col[start + (torch.arange(total, device=dev) - first)]
            nb = torch.unique(nb[~visited[nb]])
            nb = nb[torch.argsort(deg[nb], stable=True)]
            visited[nb] = True
            frontier = nb
    return torch.cat(order)


def relabel(edge_index, order):
    """Edge list in the numbering of `order` (new id of old node v = position of v in order)."""
    perm = torch.empty_like(order)
    perm[order] = torch.arange(order.numel(), device=order.device)
    return perm[edge_index], perm
