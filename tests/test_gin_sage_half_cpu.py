"""bf16 / fp16 node features in the sparse GIN / GraphSAGE path, host side (no GPU needed): which rows
gin_sage_aggregate hands the kernels as they are and which it copies to fp32, with the library replaced by a recorder,
and the dtypes that still raise."""
import contextlib

import pytest
import torch

from deep_gcns_torch_b200 import _native
from deep_gcns_torch_b200.gcn_lib import sparse as S
from deep_gcns_torch_b200.gcn_lib.sparse import torch_edge


class _Recorder:
    """Stands in for the loaded library: records each dgcn_gin_sage_aggregate call's dtype code and x pointer."""

    def __init__(self):
        self.calls = []

    def dgcn_gin_sage_aggregate(self, dtype, rule, x, N, C, *rest):
        self.calls.append((dtype, x.value, N, C))
        return 0


@pytest.fixture
def recorder(monkeypatch):
    rec = _Recorder()
    monkeypatch.setattr(_native, "lib", lambda: rec)
    monkeypatch.setattr(_native, "_require_cuda", lambda *t: None)
    monkeypatch.setattr(_native, "_stream", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: contextlib.nullcontext())
    return rec


def _csr(N):
    return (torch.zeros(N + 1, dtype=torch.int32), torch.zeros(1, dtype=torch.int32), None, None)


def _call(rec, x):
    rec.calls.clear()
    out = _native.gin_sage_aggregate("sage", x, _csr(x.shape[0]))
    assert out.dtype == torch.float32 and out.shape == x.shape
    (call,) = rec.calls
    return call


@pytest.mark.parametrize("dtype,code", [(torch.bfloat16, _native.DTYPE_BF16), (torch.float16, _native.DTYPE_F16)])
def test_eligible_half_rows_go_as_they_are(recorder, dtype, code):
    for C in (4, 64, 1024):
        x = torch.randn(6, C).to(dtype)
        assert _call(recorder, x) == (code, x.data_ptr(), 6, C)           # no copy at all
    wide = torch.randn(6, 128).to(dtype)
    nc = wide[:, 32:96]                                                   # made contiguous in its own dtype
    got = _call(recorder, nc)
    assert got[0] == code and got[1] != nc.data_ptr()
    flat = torch.randn(6 * 64 + 4).to(dtype)
    off8 = flat[4:].view(6, 64)                                           # 8-byte aligned base
    if off8.data_ptr() % 8 == 0:
        assert _call(recorder, off8) == (code, off8.data_ptr(), 6, 64)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_other_half_rows_get_the_fp32_copy(recorder, dtype):
    for C in (3, 6, 130, 1028):                                           # C % 4 != 0, C > 1024
        x = torch.randn(6, C).to(dtype)
        got = _call(recorder, x)
        assert got[0] == _native.DTYPE_F32 and got[1] != x.data_ptr()
    flat = torch.randn(6 * 64 + 1).to(dtype)
    mis = flat[1:].view(6, 64)                                            # 2-byte offset base
    assert mis.is_contiguous() and mis.data_ptr() % 8 != 0
    assert _call(recorder, mis)[0] == _native.DTYPE_F32


def test_fp32_rows_are_unchanged(recorder):
    x = torch.randn(6, 64)
    assert _call(recorder, x) == (_native.DTYPE_F32, x.data_ptr(), 6, 64)
    x3 = torch.randn(6, 3)
    assert _call(recorder, x3) == (_native.DTYPE_F32, x3.data_ptr(), 6, 3)


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32, torch.int64])
def test_other_dtypes_still_raise(recorder, dtype):
    x = torch.ones(6, 8, dtype=dtype)
    with pytest.raises(RuntimeError, match="fp32"):
        _native.gin_sage_aggregate("gin", x, _csr(6))
    with pytest.raises(RuntimeError, match="fp32"):
        _native.gin_sage_aggregate_backward("gin", x, _csr(6))
    with pytest.raises(RuntimeError, match="fp32"):                       # the backward's gradient stays fp32
        _native.gin_sage_aggregate_backward("gin", x.to(torch.bfloat16), _csr(6))
    assert not recorder.calls


@pytest.mark.parametrize("dtype", [torch.float64, torch.int64])
def test_layers_refuse_other_dtypes(monkeypatch, dtype):
    """GinConv / SAGEConv take fp32, bf16 and fp16 features and refuse the rest before anything is launched."""
    monkeypatch.setattr(_native, "_require_cuda", lambda *t: None)
    ei = torch.tensor([[0, 1], [1, 0]])
    for conv in ("gin", "sage", "rsage"):
        with pytest.raises(RuntimeError, match="fp32, bf16 or fp16"):
            S.GraphConv(4, 4, conv)(torch.ones(2, 4, dtype=dtype), ei)


def test_knn_builder_widens_half_features_in_its_copy(monkeypatch):
    """The kNN builder hands the selection kernels one fp32 (B, C, n, 1) contiguous copy of bf16 / fp16 features, equal
    to the copy it makes of x.float(); fp64 still reaches them as fp64 (and is refused there)."""
    seen = []

    def fake_knn_graph(xb, k, dilation=1, cols=None, **kw):
        seen.append(xb)
        B, _C, n, _ = xb.shape
        return torch.zeros((2, B, n, k), dtype=torch.int64), None
    monkeypatch.setattr(_native, "knn_graph", fake_knn_graph)
    x = torch.randn(2 * 16, 5)
    for dtype in (torch.bfloat16, torch.float16):
        xh = x.to(dtype)
        torch_edge.knn_matrix(xh, 4, torch.tensor([0, 1]))
        torch_edge.knn_matrix(xh.float(), 4, torch.tensor([0, 1]))
        half, up = seen[-2:]
        assert half.dtype == torch.float32 and half.shape == (2, 5, 16, 1) and half.is_contiguous()
        assert torch.equal(half, up)
    torch_edge.knn_matrix(x.double(), 4, torch.tensor([0, 1]))
    assert seen[-1].dtype == torch.float64
