"""Synthetic graphs with the node and edge counts of the OGB node-property datasets DeeperGCN trains on, drawn on the
device from seeded generators (no download), and the compact subgraph an fp64 reference of a row sample needs.

- products_edges: ogbn-products' 2,449,029 nodes and 61,859,140 edges, uniform sources and destinations (the graph
  bench_sparse.py --products times).
- proteins_graph: ogbn-proteins' 132,534 nodes and ~80 M directed edges, in-degrees ~ Exp(mean 600) (a fifth of the
  rows reach HUB_MIN_DEGREE), rows planted at the hub kernels' boundaries, empty rows, shuffled edge order.
"""
import torch

PRODUCTS = (2_449_029, 61_859_140)
PROTEINS_N = 132_534

# csr_build.cu: edges per radix-sort block (RS_CHUNK = RS_THREADS * RS_ITEMS); the histogram has 256 entries per
# block, and scan_totals_kernel scans exclusive_scan's per-1024-entry totals in strips of 1024, so a scan of more
# than 2^20 entries takes a second strip and its carry
RS_CHUNK = 2048


def ceil_div(a, b):
    return -(-a // b)


def radix_passes(n):
    """8-bit passes dgcn_csr_build's LSD sort makes for n rows."""
    bits = 1
    while (1 << bits) < n:
        bits += 1
    return (bits + 7) // 8


def products_edges(seed=0):
    N, E = PRODUCTS
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, N, (2, E), generator=g, device="cuda")


def proteins_graph(seed=0):
    """(edge_index (2, E) int64 on the device, {row: planted degree}, empty rows (list)).

    Planted: 1023 / 1024 (the last warp-per-row degree and the first hub degree), 4095 / 4096 / 4097 and
    8192 / 8193 (one segment short of, at and past a HUB_SEG_EDGES boundary), and one row of 10^6 edges (245
    segments).  Row 0 and row N - 1 are planted too.  Edges are listed in a random order, so a row's edges are
    scattered over edge_index and only a stable CSR build keeps their order."""
    N = PROTEINS_N
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand(N, generator=g, device="cuda").clamp_min(1e-12)
    deg = (-600.0 * torch.log(u)).long()                         # Exp(mean 600): P(deg >= 1024) ~ e^-1.7 ~ 0.18
    planted = {0: 1024, 1000: 1023, 20000: 4095, 40000: 4096, 60000: 4097, 70001: 1_000_000, 80000: 8192,
               N - 1: 8193}
    empty = [7, 8, 9, 50000, 131000]
    for r, d in planted.items():
        deg[r] = d
    deg[empty] = 0
    dst = torch.repeat_interleave(torch.arange(N, device="cuda"), deg)
    src = torch.randint(0, N, (dst.numel(),), generator=g, device="cuda")
    perm = torch.randperm(dst.numel(), generator=g, device="cuda")
    ei = torch.stack((src[perm], dst[perm]))
    return ei, planted, empty


def compact_subgraph(edge_index, rows):
    """The in-edges of `rows` (found with torch.isin on edge_index, independently of any CSR) renumbered onto
    nodes = rows + their sources: (nodes (sorted), edge_index of the subgraph in that numbering, positions of `rows`
    in nodes).  Every value of an aggregate row - and, with the upstream gradient non-zero only on `rows`, every
    gradient - depends on nothing else."""
    sub = edge_index[:, torch.isin(edge_index[1], rows)]
    nodes = torch.unique(torch.cat((rows, sub[0])))
    return nodes, torch.searchsorted(nodes, sub), torch.searchsorted(nodes, rows)
