"""The sparse MRConv, host side (no GPU needed): the channel slices the binding runs the raw aggregate on where the
kernels refuse C, with the library replaced by a recorder that refuses what the kernels refuse; the premises of the
exact fixtures of tests/test_mrconv_sparse_gpu.py; and the random-data error bound, restated in the kernel's order."""
import contextlib

import pytest
import torch

import mrconv_util as mu
from deep_gcns_torch_b200 import _native


def _fwd_accepts(dtype, C, x, out):
    """dgcn_genconv_aggregate's dispatch (no fusion): half rows C % 4 == 0 up to 1024; fp32 float4 rows (C % 4 == 0,
    16-byte aligned x and out) up to 1024, other rows up to 256."""
    if dtype != _native.DTYPE_F32:
        return C % 4 == 0 and C <= 1024
    aligned = (x.value | out.value) % 16 == 0
    return C <= 256 or (C % 4 == 0 and aligned and C <= 1024)


class _Recorder:
    """Stands in for the loaded library: records each aggregate call and refuses (DGCN_ERR_UNSUPPORTED) what the
    kernels refuse."""

    def __init__(self):
        self.calls = []

    def dgcn_genconv_aggregate(self, dtype, x_src, x_dst, N, C, rowptr, src, eid, edge_attr, prm, hubs, fus, keep,
                               out, stream):
        ok = _fwd_accepts(dtype, C, x_src, out)
        self.calls.append(("fwd", dtype, x_src.value, C, out.value, ok))
        return 0 if ok else _native.ERR_UNSUPPORTED

    def dgcn_genconv_aggregate_backward(self, dtype, x_src, x_dst, N, N_src, C, *rest):
        ok = C <= 512
        self.calls.append(("bwd", dtype, x_src.value, C, None, ok))
        return 0 if ok else _native.ERR_UNSUPPORTED

    def dgcn_status_string(self, rc):
        return b"unsupported"

    def dgcn_last_cuda_error(self):
        return b""


@pytest.fixture
def recorder(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: rec)
    monkeypatch.setattr(_native, "_require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "_stream", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return rec


def _csr(N):
    return (torch.zeros(N + 1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32),
            torch.zeros(1, dtype=torch.int32), None)


def _raw(aggr="max"):
    prm, _ = _native.genconv_params(aggr, add_residual=False)
    prm.raw_message = 1
    return prm


def _misaligned(N, C, dtype=torch.float32):
    flat = torch.zeros(N * C + 4, dtype=dtype)
    base = (16 - flat.data_ptr() % 16) % 16 // flat.element_size()
    return flat[base + 1:base + 1 + N * C].view(N, C)


def test_shapes_that_run_today_make_one_unchanged_call(recorder):
    """Every C the kernels take: exactly one call, on x itself (fp32) and the full C, forward and backward."""
    for C in (1, 4, 31, 33, 128, 255, 256, 260, 512, 516, 1024):
        x = torch.randn(5, C)
        recorder.calls.clear()
        _native.genconv_aggregate(x, None, _csr(5), _raw())
        assert [c[:4] for c in recorder.calls] == [("fwd", _native.DTYPE_F32, x.data_ptr(), C)], C
        if C <= 512:
            recorder.calls.clear()
            _native.genconv_aggregate_backward(x, None, _csr(5), _raw(), torch.randn(5, C))
            assert [c[:4] for c in recorder.calls] == [("bwd", _native.DTYPE_F32, x.data_ptr(), C)], C
    for C in (1, 33, 256):
        x = _misaligned(5, C)
        recorder.calls.clear()
        _native.genconv_aggregate(x, None, _csr(5), _raw())
        assert [c[:4] for c in recorder.calls] == [("fwd", _native.DTYPE_F32, x.data_ptr(), C)], C
    xh = torch.randn(5, 1024).to(torch.bfloat16)
    recorder.calls.clear()
    _native.genconv_aggregate(xh, None, _csr(5), _raw())
    assert [c[:4] for c in recorder.calls] == [("fwd", _native.DTYPE_BF16, xh.data_ptr(), 1024)]


@pytest.mark.parametrize("C,misaligned", [(257, False), (258, False), (260, True), (513, False), (1025, False),
                                          (1028, False), (1790, False), (1792, True), (3000, False)])
def test_refused_raw_forward_runs_on_channel_slices(recorder, C, misaligned):
    """A refused raw forward is followed by one accepted call per raw_channel_slices slice, each on its own contiguous
    rows, and the slices tile the channels."""
    x = _misaligned(5, C) if misaligned else torch.randn(5, C)
    out = _native.genconv_aggregate(x, None, _csr(5), _raw("add"))
    assert out.shape == (5, C)
    first, rest = recorder.calls[0], recorder.calls[1:]
    assert first[3] == C and not first[5]
    slices = _native.raw_channel_slices(C)
    assert [c[3] for c in rest] == [b - a for a, b in slices] and all(c[5] for c in rest)
    assert slices[0][0] == 0 and slices[-1][1] == C and all(a[1] == b[0] for a, b in zip(slices, slices[1:]))
    widths = [b - a for a, b in slices]
    assert all(w <= 1024 and (w % 4 == 0 or w <= 256) for w in widths)
    assert sum(w > 256 or w % 4 == 0 for w in widths) >= len(widths) - 1      # at most one narrow ragged tail


@pytest.mark.parametrize("C", (513, 640, 1024, 1025, 1792))
def test_refused_raw_backward_runs_on_channel_slices(recorder, C):
    for dtype in (torch.float32, torch.bfloat16):
        recorder.calls.clear()
        x = torch.randn(5, C).to(dtype)
        gx = _native.genconv_aggregate_backward(x, None, _csr(5), _raw(), torch.randn(5, C))[0]
        assert gx.shape == (5, C) and gx.dtype == torch.float32
        widths = [c[3] for c in recorder.calls[1:]]
        assert not recorder.calls[0][5] and widths == [b - a for a, b in _native.raw_channel_slices(C, True)]
        assert all(w <= 512 for w in widths) and sum(widths) == C
        if dtype == torch.bfloat16:       # 512-wide half slices are read as they are
            assert recorder.calls[1][1] == _native.DTYPE_BF16


def test_genconv_is_not_split(recorder):
    """MsgNorm / residual GENConv couples a row's channels: a refused call raises NotImplementedError, nothing more."""
    x = torch.randn(5, 1028)
    prm, _ = _native.genconv_params("softmax", msg_scale=1.0)
    with pytest.raises(NotImplementedError):
        _native.genconv_aggregate(x, x, _csr(5), prm)
    assert len(recorder.calls) == 1
    recorder.calls.clear()
    with pytest.raises(NotImplementedError):
        _native.genconv_aggregate_backward(x, x, _csr(5), prm, x)
    assert len(recorder.calls) == 1


# ---- fixture premises ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pow2", (False, True))
def test_exact_fixture_premises(pow2):
    """The GPU file's exact graphs: planted lengths at rows 0 and N - 1, partial sums below 2^24 (the layer's too, for
    MRConv(8, 8)), and in the mean graph power-of-two degrees, so S / deg and g / deg are exact."""
    N = 3001
    lengths = mu.POW2_LENGTHS if pow2 else mu.ROW_LENGTHS
    ei = mu.mr_graph(N, torch.Generator().manual_seed(1 + pow2), lengths,
                     mu.POW2_BACKGROUND if pow2 else mu.BACKGROUND, reverse=pow2)
    deg = torch.bincount(ei[1], minlength=N)
    plant = mu.planted_rows(N, lengths, pow2)
    assert 0 in plant and N - 1 in plant
    assert all(int(deg[r]) == L for r, L in plant.items())
    fwd, bwd, lin = mu.exact_bounds(ei, N, 8, 8, g_max=16.0)
    assert fwd < 2**24 and bwd * 8 < 2**24 and lin < 2**24
    if pow2:
        d = deg[deg > 0]
        assert bool(((d & (d - 1)) == 0).all())
        x = mu.mr_features(N, 4, torch.Generator().manual_seed(2)).double()
        s = mu.raw_aggr_chunked(x, ei, "add")
        mean = s / deg.clamp(min=1).double().unsqueeze(1)
        assert torch.equal(mean.float().double(), mean)                       # exact in fp32
        assert torch.equal((mean.float() - x.float()).double(), mean - x)   # and so is m - x


def test_first_winner_picks_the_first_tied_edge():
    """Ties from the twins, repeated sources and the all-equal channel go to the first edge in edge_index order."""
    ei = torch.tensor([[4, 3, 5, 3, 1], [0, 0, 0, 0, 2]])
    x = torch.tensor([[0.], [7.], [0.], [2.], [1.], [2.]])
    assert mu.first_winner(x, ei, "max")[:, 0].tolist() == [1, 5, 0, 5, 5, 5][:0] + [1, 5, 4, 5, 5, 5]
    assert mu.first_winner(x, ei, "min")[0, 0] == 0
    g = torch.ones(6, 1)
    assert mu.raw_grad_chunked(x, ei, "max", g)[:, 0].tolist() == [0, 1, 0, 1, 0, 0]
    assert mu.mr_grad_chunked(x, ei, "add", g)[:, 0].tolist() == [-4, 1, -1, 2, 1, 1]


# ---- the random-data bound, in the kernel's order ----------------------------------------------------------------------
@pytest.mark.parametrize("aggr", mu.AGGRS)
def test_error_bound_holds_in_the_kernel_order(aggr):
    """fp32 in the one-warp kernel's order - one running sum (or max) per channel over the row's edges in CSR order,
    then / deg for mean, then - deg * x_i or - x_i - stays within mr_error_bound of fp64 on randn rows with
    channels at mean +-100, on rows up to 1100 edges."""
    N, C = 300, 4
    g = torch.Generator().manual_seed(9)
    ei = mu.mr_graph(N, g, (0, 1, 33, 1100), mu.BACKGROUND)
    x = torch.randn(N, C, generator=g)
    x[:, 1] += 100.0
    x[:, 2] -= 100.0
    order = torch.sort(ei[1], stable=True).indices
    src, dst = ei[0, order], ei[1, order]
    deg = torch.bincount(dst, minlength=N)
    rowptr = torch.cat((torch.zeros(1, dtype=torch.long), deg.cumsum(0)))
    pos = torch.arange(src.numel()) - rowptr[dst]
    acc = torch.zeros(N, C) if aggr in ("add", "mean") else torch.full((N, C), -float("inf"))
    v = x if aggr != "min" else -x
    for k in range(int(deg.max())):
        sel = pos == k
        rows, vals = dst[sel], v[src[sel]]
        acc[rows] = acc[rows] + vals if aggr in ("add", "mean") else torch.maximum(acc[rows], vals)
    d = deg.float().unsqueeze(1)
    if aggr == "add":
        xj = acc - d * x
    else:
        m = acc / d.clamp(min=1) if aggr == "mean" else (acc if aggr == "max" else -acc)
        m = torch.where(d > 0, m, torch.zeros_like(m))
        xj = torch.where(d > 0, m - x, torch.zeros_like(m))
    err = (xj.double() - mu.mr_aggr_chunked(x, ei, aggr)).abs()
    bound = mu.mr_error_bound(x, ei, aggr)
    assert bool((err <= bound).all())
    if aggr in ("add", "mean"):
        assert float(err.max()) > 0                     # the bound is exercised, not vacuous
