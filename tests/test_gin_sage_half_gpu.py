"""bf16 / fp16 node features in the sparse GIN / GraphSAGE path on the GPU.  The aggregate reads half rows as they are
and must return exactly the bits of the same call on x.float() (every dispatch, hub segments, fallback copies); the
gradient is the upcast call's fp32 gradient rounded once to x's dtype; the sparse kNN builders give the graph of
x.float(); and the layers, blocks and the reference's example models run under torch.autocast with the outputs of the
same module fed upcast inputs."""
import copy
import re

import pytest
import torch

import backward_util as bu
import gin_sage_util as gsu
from test_sparse_edgeconv_gpu import SparseDeepGCN
from test_sparse_half_gpu import _ulp

pytestmark = pytest.mark.gpu
HALF = [torch.bfloat16, torch.float16]
CONVS = ("gin", "sage", "rsage")
# both sides of every VEC 4 channel-block boundary (NBLK 1 / 2 / 4 / 8 up to 128 / 256 / 512 / 1024 channels)
SWEEP_C = (4, 8, 64, 124, 128, 132, 256, 260, 512, 516, 1020, 1024)
PLANTED = {5: 1023, 6: 1024, 7: 4096, 8: 4097, 9: 8192}     # gin_sage_util.loop_positions' recipes


def _id(v):
    return str(v).replace("torch.", "") if isinstance(v, torch.dtype) else None


def _native():
    from deep_gcns_torch_b200 import _native
    return _native


def _rules():
    """(conv, eps) of every rule: GIN with eps 0 and 0.25, SAGE, relative SAGE."""
    return [("gin", None), ("gin", torch.tensor([0.25], device="cuda")), ("sage", None), ("rsage", None)]


@pytest.fixture(scope="module")
def graph():
    """N = 2003: random edges (duplicates: every 7th repeats its predecessor; every 97th edge a self loop), rows 11 and
    12 with three extra self loops each, the last 40 rows empty, and rows 5..9 of 1023, 1024, 4096, 4097 and 8192 edges
    with self loops planted at the last one-warp row, the first hub row, a full 32-edge ballot chunk, a loop alone in
    its hub segment and loops confined to the second segment."""
    g = torch.Generator().manual_seed(11)
    N, E = 2003, 12000
    src, dst = torch.randint(0, N, (E,), generator=g), torch.randint(10, N - 40, (E,), generator=g)
    src[1::7], dst[1::7] = src[0::7][:len(src[1::7])], dst[0::7][:len(dst[1::7])]
    parts = [torch.stack((src, dst))]
    for r in (11, 12):
        parts.append(torch.full((2, 3), r))
    for r, deg in PLANTED.items():
        parts.append(torch.stack((torch.randint(0, N, (deg,), generator=g), torch.full((deg,), r))))
    ei = torch.cat(parts, 1)
    ei = ei[:, torch.randperm(ei.shape[1], generator=g)]
    gsu.plant_self_loops(ei, PLANTED)
    ei = ei.cuda()
    csr = _native().csr_build(ei, N)
    assert csr[3] is not None
    yield N, ei, csr
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import clear_csr_cache
    clear_csr_cache()


def _x(N, C, dtype, seed):
    return torch.randn(N, C, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda").to(dtype)


def _assert_upcast_bits(x, csr, conv, eps, what):
    nat = _native()
    got = nat.gin_sage_aggregate(conv, x, csr, eps)
    want = nat.gin_sage_aggregate(conv, x.float(), csr, eps)
    assert got.dtype == torch.float32
    assert torch.equal(got, want), "%s %s eps=%s: %d values differ" % (what, conv, eps, int((got != want).sum()))


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_forward_bits_per_dispatch(graph, dtype):
    """Every rule at every C, with the hub list (MODE 0 / 1 / 2) and without it: the bits of the call on x.float()."""
    N, _ei, csr = graph
    for C in SWEEP_C:
        x = _x(N, C, dtype, C)
        for conv, eps in _rules():
            for name, c in (("hub list", csr), ("one warp per row", csr[:3])):
                _assert_upcast_bits(x, c, conv, eps, "C=%d %s" % (C, name))


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_fallbacks_give_the_upcast_bits(graph, dtype):
    """The rows the kernels cannot read as half (C % 4 != 0, a row base off 8 bytes) take the fp32 copy; an 8-byte
    aligned base that is not 16-byte aligned and non-contiguous rows are read as half.  All give the upcast bits."""
    N, _ei, csr = graph
    for C in (3, 6, 130, 1022):                                      # C % 4 != 0
        x = _x(N, C, dtype, C)
        for conv, eps in _rules():
            _assert_upcast_bits(x, csr, conv, eps, "C=%d" % C)
    for C in (64, 256):
        x = _x(N, C, dtype, C)
        for off in (1, 4):                                           # 2 bytes (fp32 copy), 8 bytes (half rows)
            y = torch.empty(N * C + off, dtype=dtype, device="cuda")[off:].view(N, C)
            y.copy_(x)
            assert y.data_ptr() % 16 == 2 * off and y.is_contiguous()
            wide = _x(N, 2 * C, dtype, C + 1)
            wide[:, 1::2] = x
            nc = wide[:, 1::2]
            assert not nc.is_contiguous()
            for conv, eps in _rules():
                _assert_upcast_bits(y, csr, conv, eps, "C=%d base offset %d B" % (C, 2 * off))
                _assert_upcast_bits(nc, csr, conv, eps, "C=%d non-contiguous" % C)
    with pytest.raises(NotImplementedError):                          # C > 1024: refused as in fp32
        _native().gin_sage_aggregate("sage", _x(N, 1028, dtype, 0), csr)


_KERNEL = re.compile(r"genconv_aggregate_kernel<(float|__nv_bfloat16|__half), (?:\(int\))?(\d+), (?:\(int\))?(\d+), "
                     r"(?:\(int\))?\d+, (?:\(int\))?(\d+)")


def _profile(fn):
    """(kernel widths {(type, VEC, NBLK, MODE)}, names of every CPU op and GPU kernel) of fn() on the GPU; a capture
    without the aggregate's kernels is taken again (CUPTI can drop a session's kernel records)."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.key for e in prof.key_averages()}
        widths = {m.groups() for m in map(_KERNEL.search, names) if m}
        if widths:
            break
    return widths, names


@pytest.mark.parametrize("C", (64, 128, 132, 256, 516, 1024))
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_half_call_launches_the_fp32_widths_without_a_copy(graph, dtype, C):
    N, _ei, csr = graph
    nat = _native()
    tname = {torch.bfloat16: "__nv_bfloat16", torch.float16: "__half"}[dtype]
    x = _x(N, C, dtype, C)
    xf = x.float()
    for conv in ("gin", "sage"):
        want, _ = _profile(lambda: nat.gin_sage_aggregate(conv, xf, csr))
        got, names = _profile(lambda: nat.gin_sage_aggregate(conv, x, csr))
        assert want and {w[0] for w in want} == {"float"}, sorted(names)
        assert {g[0] for g in got} == {tname}, sorted(names)
        assert {g[1:] for g in got} == {w[1:] for w in want}, (sorted(got), sorted(want))
        assert {g[3] for g in got} == {"0", "1", "2"}                  # row kernel and both hub kernels
        copies = sorted(n for n in names if n in ("aten::copy_", "aten::to", "aten::_to_copy"))
        assert not copies, copies


def test_no_fp32_copy_of_x():
    """N = 2^20, C = 128, bf16 x: the peak rise over one aggregate call is the fp32 output and the hub partials; an
    fp32 copy of x would add 512 MiB."""
    nat = _native()
    N, C, E = 1 << 20, 128, 8 << 20
    g = torch.Generator(device="cuda").manual_seed(0)
    ei = torch.randint(0, N, (2, E), generator=g, device="cuda")
    ei[1, :4096] = 7                                                  # one hub row
    csr = nat.csr_build(ei, N)
    del ei
    assert csr[3] is not None
    x = torch.randn(N, C, generator=g, device="cuda").to(torch.bfloat16)
    hub = csr[3][3] * 3 * C * 4
    for conv in CONVS:
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = nat.gin_sage_aggregate(conv, x, csr)
        torch.cuda.synchronize()
        rise = torch.cuda.max_memory_allocated() - base
        assert rise <= out.numel() * 4 + hub + (2 << 20), (conv, rise)
        del out


def _grads(conv, csr, x, eps, gout):
    """x.grad of the aggregate on half x, and the fp32 gradient of the call on x.float()."""
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import _GinSageFn
    xh = x.detach().clone().requires_grad_(True)
    _GinSageFn.apply(conv, csr, xh, eps).backward(gout)
    xf = x.detach().float().requires_grad_(True)
    _GinSageFn.apply(conv, csr, xf, eps).backward(gout)
    return xh.grad, xf.grad


@pytest.mark.parametrize("hub", [0, 1024])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_backward_is_the_rounded_upcast_gradient(dtype, hub):
    """Exact fixtures (integer features, c_i a power of two, upstream gradients in sixteenths: every fp32 sum exact in
    any order): bit-equal to the upcast gradient rounded once.  Random data: within one ulp of the dtype."""
    g = torch.Generator().manual_seed(hub + 1)
    N, C = 203, 64
    ei = gsu.exact_graph(N, g, hub).cuda()
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    csr = csr_of(ei, N)
    x = gsu.exact_features(N, C, g).cuda().to(dtype)
    gout = gsu.sixteenths((N, C), g).cuda()
    for conv, eps in _rules():
        gh, gf = _grads(conv, csr, x, eps, gout)
        assert gh.dtype == dtype and gf.dtype == torch.float32
        assert torch.equal(gh, gf.to(dtype)), (conv, eps)
    xr = torch.randn(N, C, generator=g).cuda().to(dtype)
    gr = torch.randn(N, C, generator=g).cuda()
    for conv, eps in _rules():
        gh, gf = _grads(conv, csr, xr, eps, gr)
        assert gh.dtype == dtype
        bound = _ulp(gf, dtype) + 1e-6 * gf.abs().max()             # (+ fp32 noise under cancellation)
        assert bool(((gh.float() - gf).abs() <= bound).all()), (conv, eps)


# ---- layers and models under autocast ------------------------------------------------------------------------------
def _upcast_inputs(_mod, args):
    return tuple(a.float() if torch.is_tensor(a) and a.is_floating_point() else a for a in args)


def _hook_upcast(model):
    """model with a forward pre-hook that upcasts the input of each sparse layer that reads half rows."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    for m in model.modules():
        if isinstance(m, (S.GinConv, S.SAGEConv, S.MRConv, S.DilatedKnnGraph)):
            m.register_forward_pre_hook(_upcast_inputs)
    return model


def _close_grads(what, got, ref, dtype, ulps=2):
    """Gradients of the half run and the upcast run: they differ by the order of the backward's fp32 atomics, i.e. by
    an ulp of the half-precision activation gradients, which may pass through one more half-precision addition."""
    eps = torch.finfo(dtype).eps if got.dtype == dtype else torch.finfo(torch.bfloat16).eps
    scale = float(ref.float().abs().max())
    torch.testing.assert_close(got.float(), ref.float(), rtol=ulps * eps, atol=ulps * eps * scale, msg=what)


def _bn_stats(model):
    return [t for m in model.modules() if isinstance(m, torch.nn.modules.batchnorm._BatchNorm)
            for t in (m.running_mean, m.running_var)]


def _layers(C):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    mods = [("GraphConv %s" % c, S.GraphConv(C, C, c, "relu", "batch")) for c in ("gin", "sage", "rsage", "mr")]
    for c in CONVS:
        mods += [("ResGraphBlock %s" % c, S.ResGraphBlock(C, c, "relu", "batch")),
                 ("DenseGraphBlock %s" % c, S.DenseGraphBlock(C, 16, c, "relu", "batch")),
                 ("DynConv %s" % c, S.DynConv(C, C, 9, 2, c, "relu", "batch"))]
    mods.append(("DynConv mr", S.DynConv(C, C, 9, 1, "mr", "relu", "batch")))
    return mods


@pytest.mark.parametrize("train", [False, True], ids=["eval", "train"])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_layers_under_autocast_match_upcast_inputs(dtype, train):
    B, n, C = 2, 128, 32
    g = torch.Generator().manual_seed(4)
    batch = torch.arange(B).repeat_interleave(n).cuda()
    x0 = torch.randn(B * n, C, generator=g).cuda().to(dtype)
    ei = torch.randint(0, B * n, (2, 3000), generator=g).cuda()
    ei[0, ::50] = ei[1, ::50]
    wgt = torch.randn(B * n, 2 * C, generator=g).cuda()
    for name, mod in _layers(C):
        torch.manual_seed(0)
        mod = mod.cuda().train(train)
        ref = _hook_upcast(copy.deepcopy(mod))
        outs = []
        for m in (mod, ref):
            x = x0.clone().requires_grad_(True)
            with torch.autocast("cuda", dtype=dtype):
                if name.startswith("DynConv"):
                    y = m(x, batch)
                    if m is mod:
                        graph = m.dilated_knn_graph(x, batch)
                        assert torch.equal(graph, m.dilated_knn_graph(x.float(), batch)), name
                else:
                    y = m(x, ei)
                y = y[0] if isinstance(y, tuple) else y
            (y.float() * wgt[:, :y.shape[1]]).sum().backward()
            outs.append((y, x.grad))
        (y, gx), (y_ref, gx_ref) = outs
        assert torch.equal(y, y_ref), name
        for a, b in zip(_bn_stats(mod), _bn_stats(ref)):
            assert torch.equal(a, b), name
        assert gx.dtype == dtype
        _close_grads(name + " grad x", gx, gx_ref, dtype)
        for (pn, p), q in zip(mod.named_parameters(), ref.parameters()):
            assert (p.grad is None) == (q.grad is None), (name, pn)
            if p.grad is not None:
                _close_grads("%s grad %s" % (name, pn), p.grad, q.grad, dtype)


def _step(model, inputs, dtype, seed=9):
    torch.manual_seed(seed)                                         # the same dropout masks on both runs
    with torch.autocast("cuda", dtype=dtype):
        out = model(*inputs)
    out.float().square().mean().backward()
    return out


def _compare_models(what, model, ref, out, out_ref):
    """Logits equal; gradients finite and, since the two backward passes differ only by the order of the fp32
    atomics (an ulp of the half activation gradients that every layer below propagates), close normwise: each weight
    matrix within 10 %, the whole model within 2 % (test_sparse_half_gpu.py's bound)."""
    assert torch.equal(out, out_ref), what
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))
    got, want = [], []
    for (name, p), q in zip(model.named_parameters(), ref.parameters()):
        assert (p.grad is None) == (q.grad is None), (what, name)
        if p.grad is None:
            continue
        assert bool(torch.isfinite(p.grad).all()), (what, name)
        got.append(p.grad.reshape(-1))
        want.append(q.grad.reshape(-1))
        if p.dim() >= 2:
            assert rel(p.grad, q.grad) <= 0.1, (what, name, rel(p.grad, q.grad))
    assert rel(torch.cat(got), torch.cat(want)) <= 0.02, (what, rel(torch.cat(got), torch.cat(want)))


PPI_CASES = [("mr", True), ("edge", True), ("gin", True), ("sage", True), ("rsage", True), ("sage", False)]


@pytest.mark.parametrize("conv,bias", PPI_CASES, ids=["%s-bias%d" % (c, b) for c, b in PPI_CASES])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_ppi_deepgcn_trains_under_autocast(dtype, conv, bias):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    opt = dict(n_filters=32, act="relu", norm="batch", bias=bias, n_heads=1, block="res", n_blocks=4,
               in_channels=50, n_classes=121, dropout=0.2, conv=conv)
    torch.manual_seed(1)
    model = gsu.ppi_deepgcn(S, opt).cuda().train()
    ref = _hook_upcast(copy.deepcopy(model))
    g = torch.Generator().manual_seed(2)
    N = 1500
    ei = torch.randint(0, N, (2, 24000), generator=g).cuda()
    ei[1, :1500] = 3                                                  # a hub row
    inputs = (torch.randn(N, 50, generator=g).cuda(), ei)
    out = _step(model, inputs, dtype)
    out_ref = _step(ref, inputs, dtype)
    _compare_models("PPI DeepGCN %s bias=%s" % (conv, bias), model, ref, out, out_ref)


@pytest.mark.parametrize("conv", ["edge", "mr", "gin", "sage", "rsage"])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_sparse_deepgcn_trains_under_autocast(dtype, conv):
    import types
    opt = types.SimpleNamespace(n_filters=32, k=9, n_blocks=4, stochastic=False, epsilon=0.0, in_channels=6,
                                conv=conv, act="relu", norm="batch", bias=True, dropout=0.3, n_classes=13)
    torch.manual_seed(1)
    model = SparseDeepGCN(opt).cuda().train()
    ref = _hook_upcast(copy.deepcopy(model))
    g = torch.Generator().manual_seed(3)
    B, n = 2, 512
    batch = torch.arange(B).repeat_interleave(n).cuda()
    inputs = (torch.rand(B * n, 3, generator=g).cuda(), torch.rand(B * n, 3, generator=g).cuda(), batch, B)
    out = _step(model, inputs, dtype)
    out_ref = _step(ref, inputs, dtype)
    _compare_models("SparseDeepGCN %s" % conv, model, ref, out, out_ref)
