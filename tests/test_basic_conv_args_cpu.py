"""The dgcn_basic_conv / dgcn_bn_sync checks of the five BasicConv entry points (dgcn_graph_conv_forward,
dgcn_dyn_conv_forward, dgcn_graph_conv_backward, dgcn_sparse_edge_conv_forward / _backward), host side: each invalid
configuration gives the same status from every entry point.

Nothing is launched.  The workspace is null with ws_bytes = 0, so a call that gets past the checks stops at its
workspace carve with DGCN_ERR_WORKSPACE, which every path takes before its first launch.  Without CUDA the device
pointers are stand-ins that the host never dereferences; with CUDA they are device tensors of the right shapes."""
import ctypes

import pytest
import torch

B, C, N, K, CO = 2, 4, 8, 3, 6
BAD_ARG, UNSUPPORTED, WORKSPACE = -1, -2, -3
ACT_RELU, ACT_LEAKYRELU, ACT_PRELU = 1, 2, 3
NORM_NONE, NORM_BATCH_EVAL, NORM_BATCH_TRAIN = 0, 1, 2


class _Device:
    """Device pointers: of zero-filled CUDA tensors when there is a device, else a non-null stand-in."""

    def __init__(self):
        self.tensors = []

    def __call__(self, *shape, dtype=torch.float32, fill=None):
        if not torch.cuda.is_available():
            return 0x1000
        t = (torch.zeros(shape, dtype=dtype) if fill is None else fill.to(dtype)).cuda()
        self.tensors.append(t)
        return t.data_ptr()


@pytest.fixture(scope="module")
def setup():
    from deep_gcns_torch_b200 import _native, build
    build.build()
    lib, dev = _native.lib(), _Device()
    x, ei, out = dev(B, C, N), dev(2, B, N, K, dtype=torch.int64), dev(B, CO, N)
    xs, outs = dev(N, C), dev(N, CO)
    rowptr = dev(N + 1, dtype=torch.int32, fill=torch.arange(N + 1) * K)
    src = dev(N * K, dtype=torch.int32)
    grads = [dev(CO, 2 * C), dev(CO), dev(CO), dev(CO), dev(1)]      # weight, bias, bn_weight, bn_bias, prelu
    dil = _native.DilationC(K, 1, None, 0, 0)
    tail = (None, 0, None)                                             # workspace, ws_bytes, stream
    calls = {}
    for conv, name in ((0, "edge"), (1, "mr")):
        calls[name + " forward"] = lambda p, s, conv=conv: lib.dgcn_graph_conv_forward(
            conv, x, B, C, N, C * N, N, ei, None, K, p, CO, out, s, *tail)
        calls[name + " dyn forward"] = lambda p, s, conv=conv: lib.dgcn_dyn_conv_forward(
            conv, x, B, C, N, C * N, N, ctypes.byref(dil), p, CO, out, None, None, s, *tail)
        calls[name + " backward"] = lambda p, s, conv=conv: lib.dgcn_graph_conv_backward(
            conv, x, B, C, N, C * N, N, ei, None, K, p, CO, out, dev(B, C, N), *grads, s, *tail)
    calls["sparse forward"] = lambda p, s: lib.dgcn_sparse_edge_conv_forward(
        xs, N, C, rowptr, src, N * K, p, CO, outs, s, *tail)
    calls["sparse backward"] = lambda p, s: lib.dgcn_sparse_edge_conv_backward(
        xs, N, C, rowptr, src, N * K, p, CO, outs, dev(N, C), *grads, s, *tail)

    def basic_conv(**change):
        p = _native.BasicConvC(weight=dev(CO, 2 * C), bias=dev(CO), act=ACT_PRELU, slope=0.2, prelu_weight=dev(1),
                               norm=NORM_BATCH_EVAL, bn_weight=dev(CO), bn_bias=dev(CO), bn_mean=dev(CO),
                               bn_var=dev(CO), bn_eps=1e-5)
        for k, v in change.items():
            setattr(p, k, v)
        return p

    reduced = []
    reduce = _native.REDUCE_FN(lambda user: reduced.append(user) or 0)
    moments = dev(2 * CO + 1, dtype=torch.float64)
    syncs = {None: None, "ok": _native.BnSyncC(moments, reduce, None),
             "no reduce": _native.BnSyncC(moments, _native.REDUCE_FN(), None),
             "no moments": _native.BnSyncC(None, reduce, None)}
    yield calls, basic_conv, syncs, reduced
    del dev.tensors[:]


def _statuses(setup, change, sync):
    calls, basic_conv, syncs, reduced = setup
    p, s = basic_conv(**change), syncs[sync]
    got = {name: call(ctypes.byref(p), None if s is None else ctypes.byref(s)) for name, call in calls.items()}
    assert not reduced, "a reduce callback ran"
    return got


INVALID = {
    "act 4": (dict(act=4), None, UNSUPPORTED),
    "norm 3": (dict(norm=3), None, UNSUPPORTED),
    "prelu without weight": (dict(prelu_weight=None), None, BAD_ARG),
    "eval without statistics": (dict(bn_mean=None, bn_var=None), None, BAD_ARG),
    "sync without reduce": (dict(norm=NORM_BATCH_TRAIN), "no reduce", BAD_ARG),
    "sync without moments": (dict(norm=NORM_BATCH_TRAIN), "no moments", BAD_ARG),
    "null weight": (dict(weight=None), None, BAD_ARG),
}

VALID = {
    "relu, no norm": (dict(act=ACT_RELU, prelu_weight=None, norm=NORM_NONE, bn_mean=None, bn_var=None), None),
    "prelu, eval": ({}, None),
    "leakyrelu, train, synced": (dict(act=ACT_LEAKYRELU, prelu_weight=None, norm=NORM_BATCH_TRAIN), "ok"),
}


@pytest.mark.parametrize("case", sorted(INVALID))
def test_invalid_basic_conv_same_status_everywhere(setup, case):
    change, sync, want = INVALID[case]
    got = _statuses(setup, change, sync)
    assert got == {name: want for name in got}


@pytest.mark.parametrize("case", sorted(VALID))
def test_valid_basic_conv_reaches_the_workspace(setup, case):
    change, sync = VALID[case]
    got = _statuses(setup, change, sync)
    assert got == {name: WORKSPACE for name in got}
