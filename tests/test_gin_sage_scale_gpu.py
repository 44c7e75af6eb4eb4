"""The sparse GIN / GraphSAGE aggregates (dgcn_gin_sage_aggregate and its backward) bit for bit against fp64, at
every channel dispatch and at the ogbn-proteins and ogbn-products shapes.

Exact arithmetic: integer features in [-4, 4] keep every partial sum an integer below 2^22 (gin_sage_util.
exact_magnitudes checks the bound on each graph), so the order of the additions - hub segments, their merge, the
backward's atomics - cannot change a bit.  GIN adds fl(1.25 x_i), exact too (eps = 0.25).  SAGE's one correctly
rounded division equals fp64's quotient rounded to fp32.  The backward's upstream gradient is k_i / 4 (GIN) or
c_i k_i / 4 (SAGE), integer k_i in [-4, 4], so each scattered g_i / c_i is the quarter k_i / 4; RSAGE's row term
fl(fl(-(c_i - 1) g_i) / c_i) is exact for c_i <= 2048 and for powers of two, and k_i = 0 on its other rows.
(tests/test_gin_sage_cpu.py checks these premises.)  So the kernels must equal the fp64 references of
gin_sage_util - whole-graph, a chunk of edges at a time, never through the kernel's CSR - over every row.

- channel sweep (N = 3001, planted rows of 1100, 5000 and 9000 edges): every forward (VEC, NBLK) and backward NCH
  branch at its edges, float4 rows and misaligned rows, with and without the hub list; C > 1024 refused.
- ogbn-proteins (132,534 nodes, ~80 M edges): self loops planted where the self-loop count can go wrong - rows made
  only of loops at the hub boundary, a full 32-edge ballot chunk, a loop alone in its segment, loops confined to one
  segment, 475,713 loops (> 2^16) spread over the 245 segments of the 10^6-edge row - and MODE 1 CTAs and MODE 2
  warps that loop over several work items.
- ogbn-products (2,449,029 nodes, 61.9 M uniform edges, C = 100): MODE 0 over its full grid, no hub rows.
- random data on a proteins row sample and ResGraphBlock(64, conv) forward and backward against fp64 autograd on a
  compact subgraph.

Each test prints its wall time and peak device memory.
"""
import re
import time
import types

import pytest
import torch

import backward_util as bu
import gin_sage_util as gsu
import ogb_graph_util as ogb
from test_gin_sage_gpu import reference_forward
from test_sparse_scale_gpu import MODE1_CTAS_PER_SM, MODE2_WARPS, ONE_WARP_TIGHT_DEGREE, _hub_table, _sms

pytestmark = pytest.mark.gpu

MAX_PEAK = 12 * 2**30                 # the GPUs are shared: no test may hold more device memory than this
RTOL, ATOL = 2e-3, 2e-4               # random fp32 data against fp64 (test_sparse_scale_gpu.py's)
CONVS = ("gin", "sage", "rsage")
EPS = 0.25
# every forward dispatch branch at its edges (VEC 4: NBLK 1 / 2 / 4 / 8 up to 128 / 256 / 512 / 1024 channels;
# VEC 1: NBLK 1 / 2 / 4 / 8 / 16 / 32 up to 32 / 64 / 128 / 256 / 512 / 1024) and every backward NCH
SWEEP_C = (1, 31, 32, 33, 64, 65, 100, 127, 128, 129, 130, 132, 255, 256, 257, 260, 384, 511, 512, 516, 602, 1000,
           1023, 1024)
ALIGN_C = (64, 128, 256, 512, 1024)


@pytest.fixture(autouse=True)
def _time_and_peak(request):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    print("\n%s: %.2f s, peak %.2f GiB" % (request.node.name, time.perf_counter() - t0, peak / 2**30))
    assert peak <= MAX_PEAK, "%s held %.2f GiB of device memory" % (request.node.name, peak / 2**30)


def _teardown():
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import clear_csr_cache
    clear_csr_cache()
    torch.cuda.empty_cache()


def _native():
    from deep_gcns_torch_b200 import _native
    return _native


def _eps():
    return torch.tensor([EPS], device="cuda")


def _misaligned(x):
    """x's values in rows that start 4 bytes past a 16-byte boundary (the VEC 1 kernels)."""
    N, C = x.shape
    y = torch.empty(N * C + 1, device=x.device)[1:].view(N, C)
    y.copy_(x)
    assert y.data_ptr() % 16 == 4 and y.is_contiguous()
    return y


def _exact_x(N, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-4, 5, (N, C), generator=g, device="cuda").float()


def _exact_gout(conv, c, C, seed):
    """g_i = k_i / 4 (GIN) or c_i k_i / 4 (SAGE, RSAGE), k_i integer in [-4, 4]; k_i = 0 on the RSAGE rows whose
    row term would round (c_i > 2048 and not a power of two).  c: sage_counts (fp64, (N,))."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.randint(-4, 5, (c.numel(), C), generator=g, device="cuda").float()
    if conv == "gin":
        return k.div_(4)
    if conv == "rsage":
        ci = c.long()
        k[(ci > 2048) & ((ci & (ci - 1)) != 0)] = 0
    return k.mul_(c.float().unsqueeze(1) / 4)


def _ref_forward(conv, x, ei):
    return gsu.gin_aggr_chunked(x, ei, EPS) if conv == "gin" else gsu.sage_aggr_chunked(x, ei, conv == "rsage")


def _assert_bits(what, got, want, deg):
    """got, want: (N, C) fp32, bit for bit over every row; a failure names the first rows that differ and their
    in-degree."""
    bad = (got != want).any(1)
    if not bool(bad.any()):
        return
    rows = bad.nonzero().squeeze(1)
    lines = []
    for r in rows[:5].tolist():
        ch = int((got[r] != want[r]).nonzero()[0, 0])
        lines.append("row %d (in-degree %d), channel %d: got %r, want %r" % (r, int(deg[r]), ch, float(got[r, ch]),
                                                                              float(want[r, ch])))
    raise AssertionError("%s: %d of %d rows differ\n  %s" % (what, rows.numel(), got.shape[0], "\n  ".join(lines)))


def _forward_exact(G, conv, C, seed, what, misaligned=False):
    """The forward with the hub list and without it (one warp per row), bit for bit against fp64 over every row."""
    nat = _native()
    x = _exact_x(G.N, C, seed)
    want = _ref_forward(conv, x, G.ei).float()
    if misaligned:
        x = _misaligned(x)
    for name, csr in (("hub list", G.csr), ("one warp per row", G.csr[:3])):
        got = nat.gin_sage_aggregate(conv, x, csr, _eps())
        _assert_bits("%s %s C=%d %s%s" % (what, conv, C, name, ", misaligned rows" if misaligned else ""), got, want,
                     G.deg)
        del got
    del want, x


def _backward_exact(G, conv, C, seed, what):
    """The backward against the written-out fp64 gradient, bit for bit over every row; returns the call's time."""
    nat = _native()
    gout = _exact_gout(conv, G.c, C, seed)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    got = nat.gin_sage_aggregate_backward(conv, gout, G.csr, _eps())
    t1.record()
    want = gsu.gin_sage_grad_chunked(conv, gout, G.ei, EPS).float()
    _assert_bits("%s %s C=%d backward" % (what, conv, C), got, want, G.deg)
    t1.synchronize()
    return t0.elapsed_time(t1)


def _graph(ei, N, **extra):
    """What the tests of one graph share: edge_index, the kernel's CSR, in-degrees and SAGE's c_i (from edge_index),
    and the exactness bounds, which must hold."""
    nat = _native()
    csr = nat.csr_build(ei, N)
    deg = torch.bincount(ei[1], minlength=N)
    fwd, bwd = gsu.exact_magnitudes(ei, N)
    assert fwd < 2**22 and bwd < 2**22, (fwd, bwd)
    return types.SimpleNamespace(ei=ei, N=N, csr=csr, deg=deg, c=gsu.sage_counts(ei, N), **extra)


# ---- channel sweep -------------------------------------------------------------------------------------------------
def _sweep_edges(N, E, g, hubs=(1100, 5000, 9000)):
    """E random edges over N nodes with self loops (every 9th edge) and duplicates (every 7th repeats its
    predecessor), plus rows 1, 2, 3 with `hubs` extra in-edges, every 50th a self loop (9000 edges: three hub
    segments)."""
    src, dst = torch.randint(0, N, (E,), generator=g), torch.randint(0, N, (E,), generator=g)
    k = torch.arange(E)
    src = torch.where(k % 9 == 0, dst, src)
    src[1:] = torch.where(k[1:] % 7 == 0, src[:-1], src[1:])
    dst[1:] = torch.where(k[1:] % 7 == 0, dst[:-1], dst[1:])
    parts = [torch.stack((src, dst))]
    for row, n in zip((1, 2, 3), hubs):
        s = torch.randint(0, N, (n,), generator=g)
        s[::50] = row
        parts.append(torch.stack((s, torch.full((n,), row))))
    ei = torch.cat(parts, 1)
    return ei[:, torch.randperm(ei.shape[1], generator=g)]


@pytest.fixture(scope="module")
def sweep():
    N = 3001                                                 # N % 4 != 0
    ei = _sweep_edges(N, 4 * N, torch.Generator().manual_seed(12)).cuda()
    G = _graph(ei, N)
    assert G.csr[3] is not None and int(G.deg[3]) >= 9000
    yield G
    G.__dict__.clear()
    _teardown()


def _expected_widths(C, aligned):
    """(VEC, NBLK) of dispatch_gin_sage, and the backward's NCH."""
    nch = next(n for n in (1, 2, 4, 8, 16, 32) if 32 * n >= C)
    if aligned and C % 4 == 0:
        return (4, next(b for b in (1, 2, 4, 8) if 128 * b >= C)), nch
    return (1, next(b for b in (1, 2, 4, 8, 16, 32) if 32 * b >= C)), nch


@pytest.mark.parametrize("C", SWEEP_C)
@pytest.mark.parametrize("conv", CONVS)
def test_channel_sweep_bit_exact(sweep, conv, C):
    """Forward (with and without the hub list, float4 and misaligned rows) and backward at C, bit for bit against
    fp64 over every row; on randn data the misaligned (VEC 1) call gives the bits of the float4 call: both sum each
    channel over the same edges in the same order."""
    G = sweep
    _forward_exact(G, conv, C, 100 + C, "sweep")
    _forward_exact(G, conv, C, 100 + C, "sweep", misaligned=True)
    _backward_exact(G, conv, C, 200 + C, "sweep")
    if C in ALIGN_C:
        nat = _native()
        x = torch.randn(G.N, C, generator=torch.Generator(device="cuda").manual_seed(C), device="cuda")
        xm = _misaligned(x)
        for name, csr in (("hub list", G.csr), ("one warp per row", G.csr[:3])):
            _assert_bits("%s C=%d %s: VEC 1 vs VEC 4 on randn" % (conv, C, name),
                         nat.gin_sage_aggregate(conv, xm, csr, _eps()), nat.gin_sage_aggregate(conv, x, csr, _eps()),
                         G.deg)


_KERNEL = re.compile(r"genconv_aggregate_kernel<float, (?:\(int\))?(\d+), (?:\(int\))?(\d+), (?:\(int\))?\d+, "
                     r"(?:\(int\))?(\d+)")
_BWD = re.compile(r"gin_sage_bwd_kernel<(?:\(int\))?(\d+),")


@pytest.mark.parametrize("C", (1, 33, 100, 128, 130, 256, 257, 516, 1023, 1024))
def test_dispatch_launches_the_expected_widths(sweep, C):
    """Which (VEC, NBLK) the forward launches (the hub list given: MODE 0, 1 and 2 all take it) and which NCH the
    backward launches, for float4-able and misaligned rows.  A capture that recorded none of the kernels is taken
    again (CUPTI can drop a session's kernel records)."""
    G, nat = sweep, _native()
    x = _exact_x(G.N, C, 7)

    def widths(fn, pattern):
        for _ in range(3):
            _, names = bu.kernel_names(fn)
            got = {m.groups() for m in map(pattern.search, names) if m}
            if got:
                return got, names
        return got, names

    for aligned, rows in ((True, x), (False, _misaligned(x))):
        (vec, nblk), nch = _expected_widths(C, aligned)
        got, names = widths(lambda: nat.gin_sage_aggregate("sage", rows, G.csr, None), _KERNEL)
        assert got and {g[:2] for g in got} == {(str(vec), str(nblk))}, (C, aligned, sorted(names))
    got, names = widths(lambda: nat.gin_sage_aggregate_backward("sage", x, G.csr, None), _BWD)
    assert got == {(str(nch),)}, (C, sorted(names))


def test_channels_past_1024_raise(sweep):
    """C = 1025 is refused (NotImplementedError), forward and backward, float4-able or misaligned rows, and through
    GraphConv's forward."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    G, nat = sweep, _native()
    x = torch.zeros(G.N, 1028, device="cuda")[:, :1025].contiguous()
    x4 = torch.zeros(G.N, 1028, device="cuda")
    for conv in CONVS:
        for rows in (x, x4, _misaligned(x4)):
            with pytest.raises(NotImplementedError):
                nat.gin_sage_aggregate(conv, rows, G.csr, _eps())
            with pytest.raises(NotImplementedError):
                nat.gin_sage_aggregate_backward(conv, rows, G.csr, _eps())
        with pytest.raises(NotImplementedError):
            S.GraphConv(1025, 8, conv).cuda()(x, G.ei)
    torch.cuda.synchronize()


# ---- ogbn-proteins shape -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def proteins():
    """ogb_graph_util.proteins_graph with self loops planted (gin_sage_util.plant_self_loops): the planted rows'
    recipes, six short rows made only of loops, and every 97th edge of the other rows; plus a row sample (the
    planted, loop-only and empty rows, rows 0 and N - 1, 128 ordinary hub rows, 128 rows below HUB_MIN_DEGREE) and its
    compact subgraph."""
    nat = _native()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    ei, planted, empty = ogb.proteins_graph(seed=0)
    N = ogb.PROTEINS_N
    deg = torch.bincount(ei[1], minlength=N)
    special = torch.zeros(N, dtype=torch.bool, device="cuda")
    special[list(planted) + empty] = True
    short = ((deg > 0) & (deg < 64) & ~special).nonzero().squeeze(1)
    loop_rows = short[torch.linspace(0, short.numel() - 1, 6, device="cuda").long()].tolist()
    fixed = gsu.plant_self_loops(ei, planted, loop_rows)
    G = _graph(ei, N, planted=planted, empty=empty, loop_rows=loop_rows, fixed=fixed)
    special[loop_rows] = True
    hub = ((G.deg >= nat.HUB_MIN_DEGREE) & ~special).nonzero().squeeze(1)
    low = ((G.deg > 0) & (G.deg < nat.HUB_MIN_DEGREE) & ~special).nonzero().squeeze(1)
    pick = lambda v, k: v[torch.linspace(0, v.numel() - 1, k, device="cuda").long()]
    rows = torch.cat((torch.tensor(list(planted) + empty + loop_rows + [0, N - 1], device="cuda"), pick(hub, 128),
                      pick(low, 128)))
    G.rows = torch.unique(rows)
    G.nodes, G.ei_c, G.rows_c = ogb.compact_subgraph(ei, G.rows)
    torch.cuda.synchronize()
    print("\nproteins graph: N=%d E=%d, %d sampled rows, subgraph of %d nodes: %.2f s, peak %.2f GiB" % (
        N, ei.shape[1], G.rows.numel(), G.nodes.numel(), time.perf_counter() - t0,
        torch.cuda.max_memory_allocated() / 2**30))
    yield G
    G.__dict__.clear()
    _teardown()


def test_proteins_planted_loops_and_hub_rounds(proteins):
    """The planted rows have the c_i they were planted for (counted on edge_index), and the hub kernels loop: more
    MODE 1 items than its 4 x SMs CTAs, more hub rows than MODE 2's 256 warps, sampled hub rows past the first round
    of both."""
    G, nat = proteins, _native()
    c = G.c.long().cpu()
    want = {0: 1, 1000: 1, 40000: 4096 - 32 + 1, 60000: 4097, 80000: 8192 - 2048 + 1, 70001: 2**19}
    assert {r: int(c[r]) for r in want} == want
    assert all(int(c[r]) == 1 for r in G.loop_rows) and all(int(c[r]) == 1 for r in G.empty)
    assert int(G.deg[0]) >= nat.HUB_MIN_DEGREE > int(G.deg[1000])
    loops = int(G.deg.sum()) - int(G.c.sum()) + G.N
    assert loops > G.ei.shape[1] // 100, loops                 # ~1/97 of the other edges too
    items, table = _hub_table(G.csr)
    grid1 = MODE1_CTAS_PER_SM * _sms()
    assert items.shape[0] > grid1 and table.shape[0] > MODE2_WARPS, (items.shape[0], table.shape[0])
    where = torch.isin(table[:, 0], G.rows.cpu()).nonzero().squeeze(1)
    assert int(where.numel()) >= 100
    assert bool((where >= MODE2_WARPS).any())
    assert bool((table[where, 1] + table[where, 2] > grid1).any())


@pytest.mark.parametrize("C", (8, 64, 256))
@pytest.mark.parametrize("conv", CONVS)
def test_proteins_exact_over_every_row(proteins, conv, C):
    """Forward with the hub list and without it, and the backward (one warp per row, the 10^6-edge row included),
    bit for bit against fp64 over all 132,534 rows."""
    _forward_exact(proteins, conv, C, 300 + C, "proteins")
    ms = _backward_exact(proteins, conv, C, 400 + C, "proteins")
    print("\nproteins %s C=%d: backward %.2f ms" % (conv, C, ms))


@pytest.mark.parametrize("conv", CONVS)
def test_proteins_random_rows_against_fp64(proteins, conv):
    """randn at C = 64 against fp64 on the sampled rows (rounding that integer data cannot show): with the hub list
    on every sampled row, without it (one warp per row) on the rows below ONE_WARP_TIGHT_DEGREE.  One warp sums the
    10^6-edge row in one fp32 chain per lane, and randn's cancellation leaves that chain's error unbounded relative to
    the GIN sum (the exact tests hold the row bit for bit on that path; csr_build always gives such a graph a hub
    list)."""
    G, nat = proteins, _native()
    x = torch.randn(G.N, 64, generator=torch.Generator(device="cuda").manual_seed(5), device="cuda")
    xr = x[G.nodes].double()
    ref = (gsu.gin_aggr(xr, G.ei_c, EPS) if conv == "gin" else gsu.sage_aggr(xr, G.ei_c, conv == "rsage"))[G.rows_c]
    short = G.deg[G.rows] < ONE_WARP_TIGHT_DEGREE
    assert int((~short).sum()) == 1
    for name, csr, keep in (("hub list", G.csr, torch.ones_like(short)), ("one warp per row", G.csr[:3], short)):
        got = nat.gin_sage_aggregate(conv, x, csr, _eps())[G.rows]
        ok = torch.isclose(got.double(), ref, rtol=RTOL, atol=ATOL).all(1) | ~keep
        assert bool(ok.all()), "%s %s: rows %s out of tolerance" % (conv, name, G.rows[~ok][:5].tolist())


@pytest.mark.parametrize("conv", CONVS)
def test_proteins_res_graph_block(proteins, conv):
    """ResGraphBlock(64, conv, 'relu', 'batch') in eval mode, forward and backward, with the upstream gradient non-zero
    only on the sampled rows: against fp64 autograd on the compact subgraph; grad x outside it exactly 0."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    G = proteins
    torch.manual_seed(6)
    blk = S.ResGraphBlock(64, conv, "relu", "batch").cuda().eval()
    with torch.no_grad():
        for b in blk.modules():
            if isinstance(b, torch.nn.BatchNorm1d):
                b.weight.uniform_(0.5, 1.5)
                b.bias.uniform_(-0.5, 0.5)
                b.running_mean.uniform_(-0.3, 0.3)
                b.running_var.uniform_(0.5, 1.5)
        if conv == "gin":
            blk.body.gconv.eps.fill_(EPS)
    gen = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(G.N, 64, generator=gen, device="cuda").requires_grad_(True)
    wgt = torch.zeros(G.N, 64, device="cuda")
    wgt[G.rows] = torch.randn(G.rows.numel(), 64, generator=gen, device="cuda")
    y, _ = blk(x, G.ei)
    y.backward(wgt)
    x64 = x.detach()[G.nodes].double().requires_grad_(True)
    body, _lay = reference_forward(blk.body, x64, G.ei_c, conv)
    y64 = body + x64 * blk.res_scale
    (y64 * wgt[G.nodes].double()).sum().backward()
    bu.assert_grads_close(conv + " ResGraphBlock forward", y.detach()[G.rows], y64.detach()[G.rows_c])
    gx = x.grad
    # GIN's backward adds g_i to row i once per self loop: on the 10^6-edge row 475,713 fp32 additions of one value,
    # whose rounding errors share a sign - the recursive-summation bound L_i 2^-24 |sum|, not a fixed rtol, holds
    # there.  Those rows are held to that bound, apart, so that their size sets no other row's tolerance.
    ei_c = G.ei_c
    loops = torch.bincount(ei_c[1][ei_c[0] == ei_c[1]], minlength=G.nodes.numel())
    heavy = loops > 2**16
    assert int(heavy.sum()) == 1
    got, ref = gx[G.nodes], x64.grad
    bu.assert_grads_close(conv + " ResGraphBlock grad x", got[~heavy], ref[~heavy])
    slack = loops[heavy].unsqueeze(1).double() * 2.0**-24 * ref[heavy].abs() if conv == "gin" else 0.0
    bu.assert_grads_close(conv + " ResGraphBlock grad x, rows of > 2^16 self loops", got[heavy], ref[heavy],
                          slack=slack)
    gx[G.nodes] = 0
    outside = gx.abs().amax(1)
    assert not bool(outside.any()), "%s: grad x is non-zero at %d nodes outside the subgraph, e.g. node %d" % (
        conv, int((outside != 0).sum()), int(outside.argmax()))


# ---- ogbn-products shape -------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def products():
    N, _E = ogb.PRODUCTS
    G = _graph(ogb.products_edges(), N)
    yield G
    G.__dict__.clear()
    _teardown()


@pytest.mark.parametrize("conv", CONVS)
def test_products_exact_over_every_row(products, conv):
    """C = 100 (ogbn-products' feature width: 25 float4 lanes of a warp's 32 live), forward and backward over all
    2,449,029 rows, bit for bit against fp64.  Uniform degrees make no hub rows: MODE 0 over its full grid."""
    G = products
    assert G.csr[3] is None and -(-G.N // 8) > 300_000
    _forward_exact(G, conv, 100, 500, "products")
    ms = _backward_exact(G, conv, 100, 600, "products")
    print("\nproducts %s: backward %.2f ms" % (conv, ms))
