"""The fused res+ block in training, host side (no GPU needed): the C ABI declarations of the keep-mask entry points
against include/dgcn.h, the routing rule (which calls take the fused training path and which run the four lines),
the keep-bit layout and the BatchNorm1d running-statistics bookkeeping against nn.BatchNorm1d itself."""
import os
import re
import types

import pytest
import torch
from torch import nn

from deep_gcns_torch_b200 import _native
from deep_gcns_torch_b200.gcn_lib import sparse as S
from deep_gcns_torch_b200.gcn_lib.sparse import fused

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header():
    with open(os.path.join(ROOT, "include", "dgcn.h")) as fh:
        return fh.read()


def _params(name):
    m = re.search(r"int %s\(([^;]*)\);" % name, _header())
    assert m, name
    return [re.sub(r"\s+", " ", p.strip()) for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",")]


class _FakeLib:
    class _Fn:
        pass

    def __getattr__(self, name):
        fn = self._Fn()
        object.__setattr__(self, name, fn)
        return fn


def test_keep_mask_struct_matches_header():
    m = re.search(r"typedef struct dgcn_keep_mask \{([^}]*)\}", _header())
    fields = [f.split()[-1].lstrip("*") for f in m.group(1).split(";") if f.strip()]
    assert fields == [f[0] for f in _native.KeepMaskC._fields_]


def test_keep_entry_points_extend_the_typed_ones():
    lib = _FakeLib()
    _native._declare(lib)
    fwd, fwd_old = _params("dgcn_genconv_aggregate_fused_keep"), _params("dgcn_genconv_aggregate_fused_rows")
    assert fwd == fwd_old[:-2] + ["const dgcn_keep_mask* keep"] + fwd_old[-2:]
    a, b = lib.dgcn_genconv_aggregate_fused_keep, lib.dgcn_genconv_aggregate_fused_rows
    assert a.restype is b.restype
    assert list(a.argtypes) == list(b.argtypes[:-2]) + [ctypes_ptr(_native.KeepMaskC)] + list(b.argtypes[-2:])
    bwd, bwd_old = _params("dgcn_genconv_aggregate_backward_keep"), _params("dgcn_genconv_aggregate_backward_rows")
    pre = ["const float* pre_scale", "const float* pre_shift", "int32_t pre_relu", "const dgcn_keep_mask* keep"]
    assert bwd == bwd_old[:12] + pre + bwd_old[12:]
    a, b = lib.dgcn_genconv_aggregate_backward_keep, lib.dgcn_genconv_aggregate_backward_rows
    assert a.restype is b.restype
    assert list(a.argtypes) == (list(b.argtypes[:12]) + [b.argtypes[1], b.argtypes[1], _native.c_i32,
                                                          ctypes_ptr(_native.KeepMaskC)] + list(b.argtypes[12:]))
    for name in ("dgcn_keep_bits_pack", "dgcn_res_plus_backward_gy", "dgcn_res_plus_backward_dh"):
        assert len(getattr(lib, name).argtypes) == len(_params(name)), name


def ctypes_ptr(t):
    import ctypes
    return ctypes.POINTER(t)


# ---- routing ------------------------------------------------------------------------------------------------------

class _Rows:
    """Stands for h: a CUDA fp32 (N, C) tensor as far as `trainable` looks (no GPU needed)."""

    def __init__(self, N=16, C=128, dtype=torch.float32, cuda=True, contiguous=True):
        self.shape, self.dtype, self.is_cuda, self._contig = (N, C), dtype, cuda, contiguous

    def dim(self):
        return len(self.shape)

    def is_contiguous(self):
        return self._contig


def _block(C=128, **kw):
    conv = S.GENConv(C, C, aggr="softmax_sg", t=0.1, mlp_layers=kw.pop("mlp_layers", 1), norm="batch", **kw)
    return conv, nn.BatchNorm1d(C)


def test_supported_block_is_trainable():
    conv, norm = _block()
    assert fused.trainable(conv, norm, _Rows(), 0.5)
    assert fused.trainable(conv, norm, _Rows(), 0.0)
    with torch.no_grad():
        assert fused.trainable(conv, norm.train(), _Rows(), 0.1)         # train-mode norm without autograd
        assert not fused.trainable(conv, norm.eval(), _Rows(), 0.1)      # inference: the inference fusion's case
    norm.eval()
    assert fused.trainable(conv, norm, _Rows(), 0.1)                     # frozen norm, autograd on
    assert fused.trainable(conv, nn.BatchNorm1d(128, affine=False), _Rows(), 0.1)
    assert fused.trainable(conv, nn.BatchNorm1d(128, track_running_stats=False), _Rows(), 0.1)
    assert fused.trainable(conv, nn.SyncBatchNorm(128), _Rows(), 0.1)  # no process group: does not sync
    for C in (4, 512):
        c, n = _block(C)
        assert fused.trainable(c, n, _Rows(C=C), 0.5)


@pytest.mark.parametrize("case", ["layernorm", "mlp_layers_2", "encode_edge", "C30", "C516", "fp64", "bf16",
                                  "dropout_1", "dropout_neg", "cpu", "strided", "single_row_batch_stats"])
def test_exclusions_run_the_four_lines(case):
    C = {"C30": 30, "C516": 516}.get(case, 128)
    kw = {"mlp_layers_2": dict(mlp_layers=2), "encode_edge": dict(encode_edge=True, edge_feat_dim=8)}.get(case, {})
    conv, norm = _block(C, **kw)
    h = _Rows(C=C)
    dropout = {"dropout_1": 1.0, "dropout_neg": -0.1}.get(case, 0.5)
    if case == "layernorm":
        norm = nn.LayerNorm(C)
    elif case == "fp64":
        h = _Rows(dtype=torch.float64)
    elif case == "bf16":
        h = _Rows(dtype=torch.bfloat16)
    elif case == "cpu":
        h = _Rows(cuda=False)
    elif case == "strided":
        h = _Rows(contiguous=False)
    elif case == "single_row_batch_stats":
        h = _Rows(N=1)                                                   # nn.BatchNorm1d raises here: keep its error
    assert not fused.trainable(conv, norm, h, dropout)


def test_syncing_sync_batchnorm_runs_the_four_lines(monkeypatch):
    conv, _ = _block()
    norm = nn.SyncBatchNorm(128)
    monkeypatch.setattr(_native, "sync_group", lambda bn: object())      # a group with more than one rank
    assert not fused.trainable(conv, norm, _Rows(), 0.5)


def test_fused_training_false_never_takes_the_training_path(monkeypatch):
    """The default keeps today's behaviour: the training path is not even asked; with fused_training=True and a
    trainable block it is."""
    taken = []
    monkeypatch.setattr(fused, "trainable", lambda *a: True)
    monkeypatch.setattr(fused, "_res_plus_train", lambda *a: taken.append(a) or "fused")
    conv, norm = _block(8)
    conv.forward = types.MethodType(lambda self, x, ei: x * 2, conv)     # a CPU stand-in for the aggregate + MLP
    h = torch.randn(6, 8)
    out = fused.res_plus_block(conv, norm, h, None, dropout=0.0)
    assert not taken and torch.allclose(out, torch.relu(norm(h)) * 2 + h)
    assert fused.res_plus_block(conv, norm, h, None, dropout=0.0, fused_training=True) == "fused" and len(taken) == 1


# ---- keep bits ----------------------------------------------------------------------------------------------------

def pack_reference(keep):
    """The dgcn_keep_mask layout restated: (N, C) -> (N, ceil(C/32)) int32, bit c % 32 of word c / 32 = keep[:, c]."""
    N, C = keep.shape
    W = (C + 31) // 32
    words = torch.zeros((N, W), dtype=torch.int64)
    for c in range(C):
        words[:, c // 32] |= (keep[:, c] != 0).long() << (c % 32)
    words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
    return words.to(torch.int32)


def test_pack_reference_layout():
    keep = torch.zeros(2, 40)
    keep[0, 0] = keep[0, 31] = keep[0, 32] = keep[1, 39] = 1
    got = pack_reference(keep)
    assert got.tolist() == [[1 | -2 ** 31, 1], [0, 1 << 7]]


# ---- running statistics -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kw", [dict(), dict(momentum=0.3), dict(momentum=None), dict(affine=False),
                                dict(track_running_stats=False)], ids=str)
def test_running_statistics_bookkeeping_matches_batchnorm1d(kw):
    g = torch.Generator().manual_seed(0)
    ref = nn.BatchNorm1d(12, **kw).double()
    if ref.weight is not None:
        with torch.no_grad():
            ref.weight.uniform_(0.5, 1.5, generator=g)
            ref.bias.normal_(generator=g)
    got = __import__("copy").deepcopy(ref)
    for step in range(3):
        h = torch.randn(50, 12, generator=g, dtype=torch.float64) * (step + 1) + step
        want = ref(h)
        scale, shift, mean, invstd = fused.bn_batch_affine(got, h)
        torch.testing.assert_close(scale * h + shift, want, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(mean, h.mean(0))
        torch.testing.assert_close(invstd, torch.rsqrt(h.var(0, unbiased=False) + ref.eps))
        for name in ("running_mean", "running_var", "num_batches_tracked"):
            a, b = getattr(got, name), getattr(ref, name)
            assert (a is None) == (b is None), name
            if a is not None:
                torch.testing.assert_close(a, b, rtol=1e-12, atol=1e-12)
