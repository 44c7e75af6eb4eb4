"""The sparse MRConv (GraphConv(conv='mr')) on the GPU against fp64: the GENConv aggregate in raw-message mode
(dgcn_genconv_aggregate / _backward with raw_message = 1, 'min' as max on -x) and the layer around it.

- exact fixtures (mrconv_util.mr_graph / mr_features): integer features in [-8, 8] with repeated sources, self loops,
  twin nodes and an all-equal channel, rows of 0 .. 8193 edges at the one-warp / hub / segment boundaries, upstream
  gradients in quarters.  Every partial sum is an integer (quarter, eighth) far below 2^24 (exact_bounds, checked),
  so any order of the additions gives the fp64 value, and a tied max / min goes to the first edge in edge_index
  order in the kernel as in torch_scatter.  'mean' graphs have power-of-two degrees, so S / deg and g / deg are exact;
  elsewhere the mean is checked on the aggregate, one correctly rounded division of an exact sum.
- every forward (VEC, NBLK) and backward NCH dispatch, float4 and misaligned rows, with and without the hub list, and
  hub work lists longer than one round of MODE 1's and MODE 2's grids.
- randn and un-centred data against fp64 within mrconv_util.mr_error_bound; GraphConv(mr, relu, batch) in train mode
  against fp64 autograd.
- C past the kernels' widest launch (the binding's channel slices), forward and backward, and a DenseGraphBlock stack
  whose width crosses 512 and 1024.
- bf16 / fp16 features under autocast: the bits of the module fed x.float().
- the reference's PPI DeepGCN with conv='mr' (golden of tests/golden/gen_golden_ppi_mr.py), and one training step at
  a PPI batch's size against fp64 autograd.

Each test prints its wall time and peak device memory.
"""
import copy
import re
import time

import pytest
import torch

import backward_util as bu
import gin_sage_util as gsu
import golden_util as gu
import mrconv_util as mu
from test_gin_sage_scale_gpu import _KERNEL, _assert_bits, _misaligned
from test_sparse_scale_gpu import MODE1_CTAS_PER_SM, MODE2_WARPS, _sms
from deep_gcns_torch_b200 import _native
from deep_gcns_torch_b200.gcn_lib import sparse as S
from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import clear_csr_cache, csr_of
from deep_gcns_torch_b200.gcn_lib.sparse.torch_vertex import _aggregate_rows

pytestmark = pytest.mark.gpu

MAX_PEAK = 12 * 2**30                 # the GPUs are shared: no test may hold more device memory than this
AGGRS = mu.AGGRS
SWEEP_VEC4 = (4, 128, 132, 256, 260, 512, 516, 1024)
SWEEP_VEC1 = (1, 31, 32, 33, 63, 65, 127, 129, 255, 256)
SWEEP_BWD = (1, 32, 33, 64, 65, 128, 129, 256, 257, 512)
PAST_LIMITS = (258, 513, 640, 1024, 1025, 1792)
_BWD = re.compile(r"genconv_aggregate_bwd_kernel<float, (?:\(int\))?(\d+)")


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


def _capture(module, store, key, output=False):
    """Keeps the first input (or output) of module's forward in store[key]; the hook returns None, so the forward's
    output is unchanged."""
    def hook(m, inp, out):
        if key not in store:
            store[key] = (out if output else inp[0]).detach()
    module.register_forward_hook(hook)


def _prm(aggr):
    prm, _ = _native.genconv_params("max" if aggr == "min" else aggr, add_residual=False)
    prm.raw_message = 1
    return prm


def raw_forward(x, csr, aggr):
    """The raw aggregate as MRConv runs it: scatter(aggr, x[src], dst), 'min' as -max(-x)."""
    if aggr == "min":
        return -_native.genconv_aggregate(-x, None, csr, _prm(aggr))
    return _native.genconv_aggregate(x, None, csr, _prm(aggr))


def raw_backward(x, csr, aggr, gout):
    """The gradient w.r.t. x of sum(gout * raw_forward(x))."""
    if aggr == "min":
        return _native.genconv_aggregate_backward(-x, None, csr, _prm(aggr), gout)[0]
    return _native.genconv_aggregate_backward(x, None, csr, _prm(aggr), gout)[0]


class _Graph:
    def __init__(self, ei, N):
        self.ei, self.N = ei, N
        self.csr = _native.csr_build(ei, N)
        self.deg = torch.bincount(ei[1], minlength=N)


def _exact_graph(N, seed, pow2):
    g = torch.Generator().manual_seed(seed)
    lengths, background = (mu.POW2_LENGTHS, mu.POW2_BACKGROUND) if pow2 else (mu.ROW_LENGTHS, mu.BACKGROUND)
    ei = mu.mr_graph(N, g, lengths, background, reverse=pow2)
    fwd, bwd, _ = mu.exact_bounds(ei, N, 1, 1)
    assert fwd < 2**24 and bwd < 2**24
    G = _Graph(ei.cuda(), N)
    assert G.csr[3] is not None
    return G


@pytest.fixture(scope="module")
def graphs():
    """{False: the general exact graph (add, max, min; mean on the aggregate), True: the power-of-two one (mean)}."""
    gs = {False: _exact_graph(3001, 1, False), True: _exact_graph(3001, 2, True)}
    yield gs
    gs.clear()
    clear_csr_cache()
    torch.cuda.empty_cache()


def _x(N, C, seed):
    return mu.mr_features(N, C, torch.Generator().manual_seed(seed)).cuda()


def _gout(N, C, seed):
    return mu.quarters((N, C), torch.Generator().manual_seed(seed)).cuda()


def _check_exact(G, aggr, C, seed, what, misaligned=False, backward=True):
    """Forward with and without the hub list, and backward, bit for bit (by value) against fp64 over every row."""
    x = _x(G.N, C, seed)
    want = mu.raw_aggr_chunked(x, G.ei, aggr).float()
    xr = _misaligned(x) if misaligned else x
    for name, csr in (("hub list", G.csr), ("one warp per row", G.csr[:3])):
        _assert_bits("%s %s C=%d forward, %s%s" % (what, aggr, C, name, ", misaligned" if misaligned else ""),
                     raw_forward(xr, csr, aggr), want, G.deg)
    if backward:
        gout = _gout(G.N, C, seed + 1)
        _assert_bits("%s %s C=%d backward" % (what, aggr, C), raw_backward(xr, G.csr, aggr, gout),
                     mu.raw_grad_chunked(x, G.ei, aggr, gout).float(), G.deg)


# ---- a. exact fixtures -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aggr", AGGRS)
def test_exact_aggregate_and_gradient(graphs, aggr):
    """Raw aggregate and gradient at C = 16 and 64; 'mean' also on the general graph's aggregate."""
    for C in (16, 64):
        _check_exact(graphs[aggr == "mean"], aggr, C, C, "exact")
    if aggr == "mean":
        _check_exact(graphs[False], aggr, 64, 5, "exact, any degree", backward=False)


def _exact_module(C_in, C_out, aggr, g):
    mod = S.MRConv(C_in, C_out, "relu", None, True, aggr).cuda()
    with torch.no_grad():
        for p in mod.parameters():
            p.copy_(torch.randint(-8, 9, p.shape, generator=g).float() / 8)
    return mod


@pytest.mark.parametrize("aggr", AGGRS)
def test_exact_mrconv_module(graphs, aggr):
    """MRConv(8, 8, aggr) without norm, weights in eighths, TF32 off: x_j = aggr(x_j - x_i), the output and x's
    gradient equal fp64 (the reference's formula, first-edge max / min gradient) bit for bit."""
    assert not torch.backends.cuda.matmul.allow_tf32
    G = graphs[aggr == "mean"]
    C = 8
    g = torch.Generator().manual_seed(31)
    mod = _exact_module(C, 8, aggr, g)
    fwd, bwd, lin = mu.exact_bounds(G.ei.cpu(), G.N, C, 8, g_max=16.0)   # |gout @ W| <= 8 * 2 * 1, in 32nds
    assert lin < 2**24 and bwd * 8 < 2**24
    seen = {}
    _capture(mod.nn, seen, "h")
    x = _x(G.N, C, 41).requires_grad_(True)
    y = mod(x, G.ei)
    x64 = x.detach().double().requires_grad_(True)
    ref = copy.deepcopy(mod).double()
    mu.use_reference_mrconv(ref)
    y64 = ref(x64, G.ei)
    _assert_bits("MRConv %s x_j" % aggr, seen["h"][:, C:], mu.mr_aggr_chunked(x.detach(), G.ei, aggr).float(), G.deg)
    _assert_bits("MRConv %s output" % aggr, y, y64.float(), G.deg)
    gout = _gout(G.N, 8, 43)
    y.backward(gout)
    y64.backward(gout.double())
    _assert_bits("MRConv %s grad x" % aggr, x.grad, x64.grad.float(), G.deg)


# ---- b. channel sweep --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", sorted(set(SWEEP_VEC4 + SWEEP_VEC1 + SWEEP_BWD)))
def test_channel_sweep_exact(graphs, C):
    """Every dispatch branch at its edges: float4 rows (VEC 4), ragged C and misaligned rows (VEC 1), and the
    backward's NCH, for all four aggregators, with and without the hub list."""
    for aggr in AGGRS:
        G = graphs[aggr == "mean"]
        _check_exact(G, aggr, C, 1000 + C, "sweep", backward=C in SWEEP_BWD)
        if C in SWEEP_VEC1:
            _check_exact(G, aggr, C, 2000 + C, "sweep", misaligned=True, backward=False)


def _widths(fn, pattern):
    for _ in range(3):
        _, names = bu.kernel_names(fn)
        got = {m.groups() for m in map(pattern.search, names) if m}
        if got:
            return got, names
    return got, names


@pytest.mark.parametrize("C", (1, 33, 128, 132, 255, 256, 260, 516, 1024))
def test_dispatch_launches_the_expected_widths(graphs, C):
    """The (VEC, NBLK) the raw forward launches on float4-able and misaligned rows, and the backward's NCH."""
    G = graphs[False]
    x = _x(G.N, C, 7)
    for aligned, rows in ((True, x), (False, _misaligned(x))):
        if not aligned and C > 256:
            continue
        if aligned and C % 4 == 0:
            want = ("4", str(next(b for b in (1, 2, 4, 8) if 128 * b >= C)))
        else:
            want = ("1", str(next(b for b in (1, 2, 4, 8) if 32 * b >= C)))
        got, names = _widths(lambda: raw_forward(rows, G.csr, "max"), _KERNEL)
        assert got and {w[:2] for w in got} == {want}, (C, aligned, sorted(names))
    if C <= 512:
        nch = str(next(n for n in (1, 2, 4, 8, 16) if 32 * n >= C))
        got, names = _widths(lambda: raw_backward(x, G.csr, "max", x), _BWD)
        assert got == {(nch,)}, (C, sorted(names))


# ---- c. hub rounds ---------------------------------------------------------------------------------------------------
def test_hub_work_lists_longer_than_one_round():
    """More hub segments than MODE 1's 4 x SMs CTAs and more hub rows than MODE 2's 256 warps: every row against fp64
    and against the call without the hub list."""
    sms = _sms()
    lengths = (1024, 4096, 4097, 8193)                     # 1, 1, 2, 3 segments
    n_rows = MODE2_WARPS + 64
    N = 4 * n_rows + 1
    g = torch.Generator().manual_seed(5)
    src, dst = [], []
    for k in range(n_rows):
        d = lengths[k % 4]
        src.append(torch.randint(0, N, (d,), generator=g))
        dst.append(torch.full((d,), 4 * k + 1))
    ei = torch.stack((torch.cat(src), torch.cat(dst)))
    ei = ei[:, torch.randperm(ei.shape[1], generator=g)].cuda()
    G = _Graph(ei, N)
    n_items = G.csr[3][3]
    assert n_items > MODE1_CTAS_PER_SM * sms and int(G.csr[3][2][1]) > MODE2_WARPS, (n_items, sms)
    x = _x(N, 32, 9)
    for aggr in AGGRS:
        want = mu.raw_aggr_chunked(x, ei, aggr).float()
        got = raw_forward(x, G.csr, aggr)
        _assert_bits("hub rounds %s" % aggr, got, want, G.deg)
        _assert_bits("hub rounds %s, one warp per row" % aggr, raw_forward(x, G.csr[:3], aggr), got, G.deg)
    clear_csr_cache()


# ---- d. random data --------------------------------------------------------------------------------------------------
def _random_x(N, C, seed):
    """randn, with channels 1 and 2 shifted to means of +100 and -100 (|mean| / std = 100)."""
    x = torch.randn(N, C, generator=torch.Generator().manual_seed(seed))
    x[:, 1] += 100.0
    x[:, 2] -= 100.0
    return x.cuda()


@pytest.mark.parametrize("aggr", AGGRS)
def test_random_x_j_within_bound(graphs, aggr):
    """MRConv's x_j on randn and un-centred channels within mr_error_bound of fp64, every row, C = 64."""
    G = graphs[False]
    x = _random_x(G.N, 64, 3)
    mod = S.MRConv(64, 8, "relu", None, True, aggr).cuda()
    seen = {}
    _capture(mod.nn, seen, "h")
    with torch.no_grad():
        mod(x, G.ei)
    got = seen["h"][:, 64:].double()
    want = mu.mr_aggr_chunked(x, G.ei, aggr)
    bound = mu.mr_error_bound(x, G.ei, aggr)
    err = (got - want).abs()
    assert bool((err <= bound).all()), float((err / bound.clamp_min(1e-300)).max())


@pytest.mark.parametrize("aggr", AGGRS)
def test_graphconv_train_against_fp64_autograd(graphs, aggr):
    """GraphConv(48, 32, 'mr', 'relu', 'batch') in train mode, forward and backward, against fp64 autograd; the
    upstream gradient is zeroed where the fp64 pre-activation sits within 1e-5 of ReLU's kink."""
    G = graphs[False]
    torch.manual_seed(11)
    mod = S.GraphConv(48, 32, "mr", "relu", "batch", True).cuda().train()
    for p in mod.parameters():
        p.data.uniform_(-0.5, 0.5)
    ref = mu.use_reference_mrconv(copy.deepcopy(mod).double())
    x = _random_x(G.N, 48, 13).requires_grad_(True)
    x64 = x.detach().double().requires_grad_(True)
    z = {}
    _capture(ref.gconv.nn[1], z, "z", output=True)
    y64 = ref(x64, G.ei)
    y = mod(x, G.ei)
    gout = torch.randn(y.shape, generator=torch.Generator().manual_seed(17)).cuda()
    gout[z["z"].abs() < 1e-5] = 0
    y.backward(gout)
    y64.backward(gout.double())
    bu.assert_grads_close("y", y, y64, atol_frac=1e-4, rtol=1e-3)
    bu.assert_grads_close("grad x", x.grad, x64.grad, atol_frac=1e-4, rtol=1e-3)
    _assert_param_grads(mod, ref, 1e-4)


def _assert_param_grads(mod, ref, rel):
    """Every parameter's gradient within `rel` of its fp64 counterpart in relative Frobenius norm.  A Linear bias
    ahead of train-mode BatchNorm has gradient 0 (the normalisation removes it), which fp32 meets only up to rounding
    noise: it is held to `rel` of its Linear weight's gradient instead."""
    params = dict(mod.named_parameters())
    for (n, p), p64 in zip(params.items(), ref.parameters()):
        g, g64 = p.grad.double(), p64.grad
        scale = g64.norm()
        if n.endswith("bias") and n[:-4] + "weight" in params and float(scale) < 1e-9:
            scale = params[n[:-4] + "weight"].grad.double().norm()
        assert float((g - g64).norm()) <= rel * float(scale), (n, float((g - g64).norm() / g64.norm().clamp_min(1e-300)))


# ---- e. past the kernels' widest launch --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_graphs():
    gs = {pow2: _Graph(mu.mr_graph(601, torch.Generator().manual_seed(7 + pow2),
                                   mu.POW2_LENGTHS if pow2 else mu.ROW_LENGTHS,
                                   mu.POW2_BACKGROUND if pow2 else mu.BACKGROUND).cuda(), 601)
          for pow2 in (False, True)}
    yield gs
    gs.clear()
    clear_csr_cache()
    torch.cuda.empty_cache()


@pytest.mark.parametrize("C", PAST_LIMITS)
def test_past_the_kernel_limits_exact(small_graphs, C):
    """Forward (with and without the hub list; float4 and misaligned rows) and backward at C up to 1792, all four
    aggregators, bit for bit against fp64."""
    for aggr in AGGRS:
        G = small_graphs[aggr == "mean"]
        _check_exact(G, aggr, C, 3000 + C, "past limits")
        if C % 4 == 0:
            _check_exact(G, aggr, C, 4000 + C, "past limits", misaligned=True, backward=False)


def test_forced_split_gives_the_bits_of_one_launch(small_graphs):
    """A channel's edge order does not depend on its channel block: C = 1024 forward (one launch) on randn rows equals
    the same channels run as slices of 512 / 256 / 260 + 764, and C = 512 backward (exact data) its 256-wide slices."""
    G = small_graphs[False]
    x = torch.randn(G.N, 1024, generator=torch.Generator().manual_seed(1)).cuda()
    for aggr in AGGRS:
        for csr in (G.csr, G.csr[:3]):
            one = raw_forward(x, csr, aggr)
            for cuts in ((0, 512, 1024), (0, 256, 512, 768, 1024), (0, 260, 1024)):
                split = torch.cat([raw_forward(x[:, a:b].contiguous(), csr, aggr) for a, b in zip(cuts, cuts[1:])], 1)
                _assert_bits("split %s %s" % (aggr, cuts), split, one, G.deg)
    x, gout = _x(G.N, 512, 3), _gout(G.N, 512, 4)
    for aggr in AGGRS:
        G = small_graphs[aggr == "mean"]              # exact gradients: no order of the atomics changes a bit
        one = raw_backward(x, G.csr, aggr, gout)
        split = torch.cat([raw_backward(x[:, a:a + 256].contiguous(), G.csr, aggr, gout[:, a:a + 256].contiguous())
                           for a in (0, 256)], 1)
        _assert_bits("split backward %s" % aggr, split, one, G.deg)


def test_genconv_keeps_its_limits(small_graphs):
    """Non-raw GENConv (MsgNorm couples a row's channels) is not split: past its limits it still raises."""
    G = small_graphs[False]
    x = torch.randn(G.N, 1028, device="cuda")
    prm, _ = _native.genconv_params("softmax", msg_scale=1.0)
    with pytest.raises(NotImplementedError):
        _native.genconv_aggregate(x, x, G.csr, prm)
    with pytest.raises(NotImplementedError):
        _native.genconv_aggregate_backward(x[:, :516].contiguous(), x[:, :516].contiguous(), G.csr, prm,
                                           x[:, :516].contiguous())


@pytest.mark.parametrize("aggr", ("max", "add"))
def test_dense_block_stack_crossing_512_and_1024(aggr):
    """Four DenseGraphBlock(C, 256, 'mr', 'relu', 'batch') in train mode from C = 320: the blocks see C = 320, 576,
    832 and 1088 (backward past 512 from the second, forward past 1024 in the last), against fp64 autograd."""
    N = 1500
    g = torch.Generator().manual_seed(21)
    ei = torch.stack((torch.randint(0, N, (12 * N,), generator=g), torch.randint(0, N, (12 * N,), generator=g))).cuda()
    torch.manual_seed(22)
    blocks = torch.nn.ModuleList([S.DenseGraphBlock(320 + 256 * i, 256, "mr", "relu", "batch", True)
                                  for i in range(4)]).cuda().train()
    for b in blocks:
        b.body.gconv.aggr = aggr
    ref = mu.use_reference_mrconv(copy.deepcopy(blocks).double())
    x = torch.randn(N, 320, generator=g).cuda().requires_grad_(True)
    x64 = x.detach().double().requires_grad_(True)
    h, h64 = x, x64
    for b, b64 in zip(blocks, ref):
        h, h64 = b(h, ei)[0], b64(h64, ei)[0]
    assert h.shape == (N, 1344)
    gout = torch.randn(h.shape, generator=g).cuda()
    h.backward(gout)
    h64.backward(gout.double())
    bu.assert_grads_close("stack output", h, h64, atol_frac=1e-4, rtol=1e-3)
    bu.assert_grads_close("stack grad x", x.grad, x64.grad, atol_frac=1e-3, rtol=1e-3)
    _assert_param_grads(blocks, ref, 1e-3)
    clear_csr_cache()


# ---- f. autocast -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def autocast_graph():
    N = 2000
    g = torch.Generator().manual_seed(8)
    ei = mu.mr_graph(N, g, (0, 257, 2049, 5000), mu.BACKGROUND)
    yield _Graph(ei.cuda(), N)
    clear_csr_cache()


@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float16))
@pytest.mark.parametrize("aggr", AGGRS)
def test_autocast_matches_upcast_input(autocast_graph, aggr, dtype):
    """MRConv(C, 16, aggr) under autocast on half x equals the module fed x.float() bit for bit (C = 64: half rows read
    as they are; C = 33: the fp32 copy), and the aggregate's gradient comes back in x's dtype, the fp32 gradient
    rounded once."""
    G = autocast_graph
    for C in (64, 33):
        torch.manual_seed(C)
        mod = S.MRConv(C, 16, "relu", None, True, aggr).cuda()
        xh = (torch.randn(G.N, C, generator=torch.Generator().manual_seed(C)) * 4).to(dtype).cuda()
        with torch.autocast("cuda", dtype=dtype):
            y_h = mod(xh, G.ei)
            y_f = mod(xh.float(), G.ei)
        _assert_bits("autocast %s %s C=%d" % (dtype, aggr, C), y_h.float(), y_f.float(), G.deg)
        gout = torch.randn(G.N, C, generator=torch.Generator().manual_seed(1)).cuda()
        xl, xf = xh.clone().requires_grad_(True), xh.float().requires_grad_(True)
        raw = "max" if aggr == "min" else aggr
        _aggregate_rows(raw, xl, G.ei)[0].backward(gout)
        _aggregate_rows(raw, xf, G.ei)[0].backward(gout)
        assert xl.grad.dtype == dtype
        # the fp32 backward's atomics may add a source's terms in another order: compare at the rounding's precision
        assert torch.equal(xl.grad, xf.grad.to(dtype)) or \
            (xl.grad.float() - xf.grad.to(dtype).float()).abs().max() <= 2**-7 * xf.grad.abs().max()


# ---- g. PPI --------------------------------------------------------------------------------------------------------
def test_ppi_deepgcn_mr_matches_reference():
    c = gu.load("spconv_ppi_mr")
    model = gsu.ppi_deepgcn(S, c.meta).cuda().eval()
    model.load_state_dict(c.sd, strict=True)
    with torch.no_grad():
        y = model(c.ins["x"].cuda(), c.ins["edge_index"].long().cuda())
    bu.assert_grads_close("PPI DeepGCN mr", y, c.outs["y"], atol_frac=1e-4, rtol=1e-3)


def test_ppi_mr_training_step_against_fp64():
    """examples/ppi/opt.py's model (conv='mr', 256 filters, 14 res blocks, batch norm) on a PPI-sized batch
    (N = 9,716, E = 259,120): one training step's loss and parameter gradients against fp64 autograd of the same
    model with MRConv restated on mrconv_util.MRAggr64."""
    N, E = 9716, 259120
    g = torch.Generator().manual_seed(3)
    ei = torch.stack((torch.randint(0, N, (E,), generator=g), torch.randint(0, N, (E,), generator=g))).cuda()
    x = torch.randn(N, 50, generator=g).cuda()
    target = (torch.rand(N, 121, generator=g) < 0.3).float().cuda()
    opt = dict(n_filters=256, act="relu", norm="batch", bias=True, n_heads=1, block="res", n_blocks=14,
               in_channels=50, n_classes=121, dropout=0.0, conv="mr")
    torch.manual_seed(4)
    model = gsu.ppi_deepgcn(S, opt).cuda().train()
    ref = mu.use_reference_mrconv(copy.deepcopy(model).double())
    loss = torch.nn.functional.binary_cross_entropy_with_logits(model(x, ei), target)
    loss64 = torch.nn.functional.binary_cross_entropy_with_logits(ref(x.double(), ei), target.double())
    loss.backward()
    loss64.backward()
    assert abs(float(loss) - float(loss64)) <= 1e-4 * abs(float(loss64)), (float(loss), float(loss64))
    # 14 blocks of max over ReLU outputs: an fp32 activation a rounding away from the kink, or a near-tie between
    # two sources, routes a few (node, channel) gradients to another source than fp64 does; the head, below all of
    # them, collects those differences (3e-3 of its gradient's norm measured on an H100)
    _assert_param_grads(model, ref, 1e-2)
    clear_csr_cache()
