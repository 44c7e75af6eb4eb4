"""bf16 / fp16 rows in the sparse GENConv path, host side: the dgcn_dtype enum against include/dgcn.h, and the rule
that decides which rows the kernels read as they are (no GPU needed)."""
import re

import pytest
import torch

from deep_gcns_torch_b200 import _native
from test_abi_cpu import header


def test_dtype_enum_matches_header():
    m = re.search(r"enum dgcn_dtype \{([^}]*)\}", header())
    vals = dict((k.strip(), int(v)) for k, v in (e.split("=") for e in m.group(1).split(",")))
    assert vals == {"DGCN_F32": _native.DTYPE_F32, "DGCN_BF16": _native.DTYPE_BF16, "DGCN_F16": _native.DTYPE_F16}


def _rows(dtype, n=6, c=8):
    return torch.randn(n, c).to(dtype)


@pytest.mark.parametrize("dtype,code", [(torch.bfloat16, _native.DTYPE_BF16), (torch.float16, _native.DTYPE_F16)])
def test_half_rows_are_read_as_they_are(dtype, code):
    x, ea = _rows(dtype), _rows(dtype, n=10)
    got = _native.aggregate_rows(x, x, ea)
    assert got[0] == code
    same = lambda a, b: a.dtype == b.dtype and a.data_ptr() == b.data_ptr()
    assert same(got[1], x) and same(got[2], x) and same(got[3], ea)            # no copy at all
    got = _native.aggregate_rows(x, None, None)                    # raw aggregation: no x_dst, no edge_attr
    assert got[0] == code and same(got[1], x) and got[2] is None and got[3] is None
    wide = _rows(dtype, c=1024)
    assert _native.aggregate_rows(wide, wide)[0] == code
    assert _native.aggregate_rows(wide, wide, backward=True)[0] == _native.DTYPE_F32   # backward: C <= 512
    assert _native.aggregate_rows(_rows(dtype, c=512), None, backward=True)[0] == code


def test_non_contiguous_half_rows_stay_half():
    """RevGNN's channel chunks: made contiguous in their own dtype, not in fp32."""
    x = _rows(torch.bfloat16, c=16)[:, 4:12]
    assert not x.is_contiguous()
    code, xs, xd, ea = _native.aggregate_rows(x, x)
    assert code == _native.DTYPE_BF16 and xs.dtype == torch.bfloat16 and xs.is_contiguous() and xd is xs
    assert torch.equal(xs, x)


def _upcast(got, *want):
    assert got[0] == _native.DTYPE_F32
    for t, w in zip(got[1:], want):
        if w is None:
            assert t is None
        else:
            assert t.dtype == torch.float32 and t.is_contiguous() and torch.equal(t, w.float())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_everything_else_keeps_the_fp32_copies(dtype):
    x = _rows(dtype)
    other = torch.float16 if dtype == torch.bfloat16 else torch.bfloat16
    ea_other = _rows(other, n=10)
    _upcast(_native.aggregate_rows(x, x, ea_other), x, x, ea_other)               # mixed dtypes
    ea32 = _rows(torch.float32, n=10)
    _upcast(_native.aggregate_rows(x, x, ea32), x, x, ea32)
    x30 = _rows(dtype, c=30)
    _upcast(_native.aggregate_rows(x30, x30), x30, x30)                          # C % 4 != 0
    x1028 = _rows(dtype, c=1028)
    _upcast(_native.aggregate_rows(x1028, x1028), x1028, x1028)                  # C > 1024
    flat = torch.randn(6 * 8 + 1).to(dtype)
    mis = flat[1:].view(6, 8)                                                    # contiguous, 2-byte offset
    assert mis.is_contiguous() and mis.data_ptr() % 8 != 0
    _upcast(_native.aggregate_rows(mis, mis), mis, mis)
    scale, shift = torch.ones(8), torch.zeros(8)
    _upcast(_native.aggregate_rows(x, x, pre=(scale, shift, True)), x, x)        # fused pre-activation
    x64 = torch.randn(6, 8, dtype=torch.float64)
    _upcast(_native.aggregate_rows(x64, x64), x64, x64)                          # fp64
    x32 = _rows(torch.float32)
    got = _native.aggregate_rows(x32, x32)
    assert got[0] == _native.DTYPE_F32 and got[1].data_ptr() == x32.data_ptr()  # fp32: unchanged
