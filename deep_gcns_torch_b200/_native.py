"""ctypes binding of the C ABI in include/dgcn.h (libdgcn.so, sm_90a kernels).

PyTorch is only the carrier here: it owns device memory (inputs, outputs and the
scratch workspace handed to the library) and the stream the kernels are put on.
There is NO CPU or eager fallback: every wrapper raises if the library is not
built or a tensor is not on a CUDA device.
"""
import ctypes
import os
import threading

import torch
import torch.distributed as dist
from torch import nn

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libdgcn.so")

c_f32p = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_i32 = ctypes.c_int32

ACT = {None: 0, "none": 0, "relu": 1, "leakyrelu": 2, "prelu": 3}
NORM_NONE, NORM_BATCH_EVAL, NORM_BATCH_TRAIN = 0, 1, 2
CONV = {"edge": 0, "mr": 1}
AGGR = {"softmax": 0, "softmax_sg": 0, "softmax_sum": 1, "power": 2, "power_sum": 3,
        "add": 4, "sum": 4, "mean": 5, "max": 6}


class BasicConvC(ctypes.Structure):
    _fields_ = [("weight", c_f32p), ("bias", c_f32p), ("act", c_i32), ("slope", ctypes.c_float),
                ("prelu_weight", c_f32p), ("norm", c_i32), ("bn_weight", c_f32p), ("bn_bias", c_f32p),
                ("bn_mean", c_f32p), ("bn_var", c_f32p), ("bn_eps", ctypes.c_float),
                ("batch_mean_out", c_f32p), ("batch_var_out", c_f32p)]


class DilationC(ctypes.Structure):
    _fields_ = [("k", c_i64), ("dilation", c_i64), ("cols_host", ctypes.POINTER(c_i32)), ("flags", c_i32),
                ("reserved", c_i32)]


KNN_EXACT_FP32 = 1         # dgcn_knn_flags
KNN_TC_TILE_PER_CTA = 2
_knn_flags = threading.local()


class CsrHubsC(ctypes.Structure):
    _fields_ = [("items", ctypes.c_void_p), ("rows", ctypes.c_void_p), ("counts", ctypes.c_void_p),
                ("min_degree", c_i32), ("seg_edges", c_i32), ("partial", ctypes.c_void_p)]


DTYPE_F32, DTYPE_BF16, DTYPE_F16 = 0, 1, 2     # dgcn_dtype: element type of the rows the sparse kernels read
_ROW_DTYPE = {torch.float32: DTYPE_F32, torch.bfloat16: DTYPE_BF16, torch.float16: DTYPE_F16}
HALF_ROWS_MAX_C = 1024     # half rows: the forward's widest channel block; the backward's is ...
HALF_ROWS_MAX_C_BWD = 512  # ... the fp32 backward's own limit

GIN_SAGE = {"gin": 0, "sage": 1, "rsage": 2}   # dgcn_gin_sage

HUB_MIN_DEGREE = 1024      # rows at least this long are aggregated by CTAs instead of one warp
HUB_SEG_EDGES = 4096       # ... one CTA per segment of this many edges


class GenconvParamsC(ctypes.Structure):
    _fields_ = [("aggr", c_i32), ("t", ctypes.c_float), ("t_dev", c_f32p), ("p", ctypes.c_float),
                ("p_dev", c_f32p), ("y", ctypes.c_float), ("y_dev", c_f32p), ("eps", ctypes.c_float),
                ("msg_norm", c_i32), ("msg_scale", ctypes.c_float), ("msg_scale_dev", c_f32p),
                ("add_residual", c_i32), ("raw_message", c_i32)]


class BlockFusionC(ctypes.Structure):
    _fields_ = [("residual", c_f32p), ("res_stride_b", c_i64), ("res_stride_c", c_i64), ("res_scale", ctypes.c_float),
                ("out_stride_b", c_i64)]


class GenconvFusionC(ctypes.Structure):
    _fields_ = [("pre_scale", c_f32p), ("pre_shift", c_f32p), ("pre_relu", c_i32), ("skip_hubs", c_i32),
                ("row_list", ctypes.c_void_p), ("n_rows", c_i64)]


class KeepMaskC(ctypes.Structure):
    _fields_ = [("keep_bits", ctypes.c_void_p), ("words_per_row", c_i64), ("keep_scale", ctypes.c_float)]


ERR_REDUCE = -5            # dgcn_status: the dgcn_bn_sync reduce callback failed
REDUCE_FN = ctypes.CFUNCTYPE(c_i32, ctypes.c_void_p)


class BnSyncC(ctypes.Structure):
    _fields_ = [("moments", ctypes.c_void_p), ("reduce", REDUCE_FN), ("user", ctypes.c_void_p)]


def sync_group(bn):
    """The process group whose ranks share `bn`'s batch statistics, or None for local statistics: the rule of
    torch.nn.SyncBatchNorm.forward (batch statistics in training mode, torch.distributed initialised, more than
    one rank in bn.process_group or, when that is None, in WORLD).  A plain BatchNorm2d never syncs."""
    if not isinstance(bn, nn.SyncBatchNorm):
        return None
    bn_training = bn.training or (bn.running_mean is None and bn.running_var is None)
    if not (bn_training and bn.training and dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group or dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


class _BnSync:
    """dgcn_bn_sync of one call: an fp64 moments buffer (2*C_out + 1) and a reduce callback that all-reduces it over
    `group` on the current stream.  The callback object lives as long as this instance; no exception crosses the C
    ABI: the callback stores it and returns 1, and check() raises it as the cause."""

    def __init__(self, group, c_out, dev):
        self.moments = torch.empty(2 * c_out + 1, dtype=torch.float64, device=dev)
        self.error = None

        def reduce(_user):
            try:
                dist.all_reduce(self.moments, group=group)
                return 0
            except BaseException as e:     # noqa: B036 - nothing may unwind through the C frames
                self.error = e
                return 1
        self._fn = REDUCE_FN(reduce)
        self.c = BnSyncC(_ptr(self.moments), self._fn, None)

    def check(self, rc, what):
        if rc == ERR_REDUCE:
            raise RuntimeError("%s failed: all-reduce of the BatchNorm statistics raised %r" % (what, self.error)) \
                from self.error
        _check(rc, what)


_lib = None
_lock = threading.Lock()


def _declare(lib):
    vp, sz = ctypes.c_void_p, ctypes.c_size_t
    lib.dgcn_version.restype = ctypes.c_int
    lib.dgcn_version.argtypes = []
    lib.dgcn_status_string.restype = ctypes.c_char_p
    lib.dgcn_status_string.argtypes = [ctypes.c_int]
    lib.dgcn_last_cuda_error.restype = ctypes.c_char_p
    lib.dgcn_last_cuda_error.argtypes = []
    lib.dgcn_knn_graph_workspace_bytes.restype = sz
    lib.dgcn_knn_graph_workspace_bytes.argtypes = [c_i64] * 4
    lib.dgcn_knn_graph.restype = ctypes.c_int
    lib.dgcn_knn_graph.argtypes = [vp, c_i64, c_i64, c_i64, c_i64, c_i64, ctypes.POINTER(DilationC), c_i32,
                                   vp, vp, vp, sz, vp]
    lib.dgcn_graph_conv_workspace_bytes.restype = sz
    lib.dgcn_graph_conv_workspace_bytes.argtypes = [c_i32] + [c_i64] * 5
    lib.dgcn_graph_conv_forward.restype = ctypes.c_int
    lib.dgcn_graph_conv_forward.argtypes = [c_i32, vp, c_i64, c_i64, c_i64, c_i64, c_i64, vp, vp, c_i64,
                                            ctypes.POINTER(BasicConvC), c_i64, vp, ctypes.POINTER(BnSyncC), vp, sz, vp]
    lib.dgcn_dyn_conv_workspace_bytes.restype = sz
    lib.dgcn_dyn_conv_workspace_bytes.argtypes = [c_i32] + [c_i64] * 5
    lib.dgcn_dyn_conv_forward.restype = ctypes.c_int
    lib.dgcn_dyn_conv_forward.argtypes = [c_i32, vp, c_i64, c_i64, c_i64, c_i64, c_i64, ctypes.POINTER(DilationC),
                                          ctypes.POINTER(BasicConvC), c_i64, vp, vp, ctypes.POINTER(BlockFusionC),
                                          ctypes.POINTER(BnSyncC), vp, sz, vp]
    lib.dgcn_graph_conv_backward_workspace_bytes.restype = sz
    lib.dgcn_graph_conv_backward_workspace_bytes.argtypes = [c_i32] + [c_i64] * 5
    lib.dgcn_graph_conv_backward.restype = ctypes.c_int
    lib.dgcn_graph_conv_backward.argtypes = [c_i32, vp, c_i64, c_i64, c_i64, c_i64, c_i64, vp, vp, c_i64,
                                             ctypes.POINTER(BasicConvC), c_i64, vp, vp, vp, vp, vp, vp, vp,
                                             ctypes.POINTER(BnSyncC), vp, sz, vp]
    lib.dgcn_csr_build_workspace_bytes.restype = sz
    lib.dgcn_csr_build_workspace_bytes.argtypes = [c_i64, c_i64]
    lib.dgcn_csr_build.restype = ctypes.c_int
    lib.dgcn_csr_build.argtypes = [vp, c_i64, c_i64, vp, vp, vp, vp, sz, vp]
    lib.dgcn_genconv_aggregate.restype = ctypes.c_int
    lib.dgcn_genconv_aggregate.argtypes = [c_i32, vp, vp, c_i64, c_i64, vp, vp, vp, vp, ctypes.POINTER(GenconvParamsC),
                                           ctypes.POINTER(CsrHubsC), ctypes.POINTER(GenconvFusionC),
                                           ctypes.POINTER(KeepMaskC), vp, vp]
    lib.dgcn_linear_residual_workspace_bytes.restype = sz
    lib.dgcn_linear_residual_workspace_bytes.argtypes = [c_i64, c_i64]
    lib.dgcn_linear_residual.restype = ctypes.c_int
    lib.dgcn_linear_residual.argtypes = [vp, c_i64, c_i64, vp, vp, c_i64, vp, vp, vp, sz, vp]
    lib.dgcn_csr_hub_rows.restype = ctypes.c_int
    lib.dgcn_csr_hub_rows.argtypes = [vp, c_i64, c_i64, c_i32, c_i32, vp, vp, vp, vp]
    lib.dgcn_genconv_aggregate_backward.restype = ctypes.c_int
    lib.dgcn_genconv_aggregate_backward.argtypes = [c_i32, vp, vp, c_i64, c_i64, c_i64, vp, vp, vp, vp,
                                                    ctypes.POINTER(GenconvParamsC), c_i32, vp, vp, c_i32,
                                                    ctypes.POINTER(KeepMaskC), vp, vp, vp, vp, vp, vp]
    lib.dgcn_gin_sage_aggregate.restype = ctypes.c_int
    lib.dgcn_gin_sage_aggregate.argtypes = [c_i32, c_i32, vp, c_i64, c_i64, vp, vp, ctypes.POINTER(CsrHubsC), vp, vp,
                                            vp]
    lib.dgcn_gin_sage_aggregate_backward.restype = ctypes.c_int
    lib.dgcn_gin_sage_aggregate_backward.argtypes = [c_i32, c_i64, c_i64, vp, vp, vp, vp, vp, vp]
    lib.dgcn_debug_kernel_timing.restype = ctypes.c_int
    lib.dgcn_debug_kernel_timing.argtypes = [c_i32]
    lib.dgcn_debug_kernel_timing_read.restype = ctypes.c_int
    lib.dgcn_debug_kernel_timing_read.argtypes = [ctypes.c_char_p, ctypes.POINTER(ctypes.c_double),
                                                  ctypes.POINTER(c_i64)]
    lib.dgcn_debug_tc_certification.restype = ctypes.c_int
    lib.dgcn_debug_tc_certification.argtypes = [c_i32]
    lib.dgcn_debug_tc_certification_read.restype = ctypes.c_int
    lib.dgcn_debug_tc_certification_read.argtypes = [ctypes.POINTER(c_i64), ctypes.POINTER(c_i64)]
    lib.dgcn_sparse_edge_conv_workspace_bytes.restype = sz
    lib.dgcn_sparse_edge_conv_workspace_bytes.argtypes = [c_i64] * 3
    lib.dgcn_sparse_edge_conv_forward.restype = ctypes.c_int
    lib.dgcn_sparse_edge_conv_forward.argtypes = [vp, c_i64, c_i64, vp, vp, c_i64, ctypes.POINTER(BasicConvC), c_i64,
                                                  vp, ctypes.POINTER(BnSyncC), vp, sz, vp]
    lib.dgcn_sparse_edge_conv_backward_workspace_bytes.restype = sz
    lib.dgcn_sparse_edge_conv_backward_workspace_bytes.argtypes = [c_i64] * 3
    lib.dgcn_sparse_edge_conv_backward.restype = ctypes.c_int
    lib.dgcn_sparse_edge_conv_backward.argtypes = [vp, c_i64, c_i64, vp, vp, c_i64, ctypes.POINTER(BasicConvC), c_i64,
                                                   vp, vp, vp, vp, vp, vp, vp, ctypes.POINTER(BnSyncC), vp, sz, vp]
    lib.dgcn_gather_rows.restype = ctypes.c_int
    lib.dgcn_gather_rows.argtypes = [c_i32, vp, c_i64, vp, c_i64, vp, vp]
    lib.dgcn_keep_bits_pack.restype = ctypes.c_int
    lib.dgcn_keep_bits_pack.argtypes = [vp, c_i64, c_i64, vp, vp]
    lib.dgcn_res_plus_backward_gy.restype = ctypes.c_int
    lib.dgcn_res_plus_backward_gy.argtypes = [vp, c_i64, c_i64, vp, vp, ctypes.POINTER(KeepMaskC), vp, vp, vp, vp, vp,
                                              vp]
    lib.dgcn_res_plus_backward_dh.restype = ctypes.c_int
    lib.dgcn_res_plus_backward_dh.argtypes = [vp, vp, c_i64, c_i64, vp, vp, vp, vp, vp, vp]


def lib():
    """The loaded library; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        "deep_gcns_torch_b200: %s is missing - build it with "
                        "`python -m deep_gcns_torch_b200.build` (there is no CPU/eager fallback)" % LIB_PATH)
                handle = ctypes.CDLL(LIB_PATH)
                _declare(handle)
                _lib = handle
    return _lib


def _check(rc, what):
    if rc != 0:
        l = lib()
        msg = l.dgcn_status_string(rc).decode()
        extra = l.dgcn_last_cuda_error().decode() if rc == -4 else ""
        # DGCN_ERR_UNSUPPORTED: a valid request the kernels do not cover (NotImplementedError is a RuntimeError)
        raise (NotImplementedError if rc == ERR_UNSUPPORTED else RuntimeError)("%s failed: %s %s" % (what, msg, extra))


def _ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("deep_gcns_torch_b200 runs on CUDA tensors only (sm_90a kernels, no CPU fallback); "
                               "got a tensor on %s" % t.device)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _workspace(nbytes, dev):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=dev)


def _dense_view(x):
    """(B,C,N,1) or (B,C,N) fp32 with unit point stride -> tensor, B, C, N, stride_b, stride_c."""
    if x.dim() == 4:
        if x.size(3) != 1:
            raise RuntimeError("dense input must be (B, C, N, 1), got %s" % (tuple(x.shape),))
        x = x.squeeze(-1)
    if x.dtype != torch.float32:
        raise RuntimeError("dense path computes in fp32, got %s" % x.dtype)
    B, C, N = x.shape
    if N > 1 and x.stride(2) != 1:
        x = x.contiguous()
    return x, B, C, N, x.stride(0), x.stride(1)


def _dilation(k, dilation, cols):
    d = DilationC()
    d.k, d.dilation = int(k), int(dilation)
    d.flags, d.reserved = getattr(_knn_flags, "value", 0), 0
    keep = None
    if cols is not None:
        arr = (c_i32 * int(k))(*[int(c) for c in cols])
        d.cols_host = ctypes.cast(arr, ctypes.POINTER(c_i32))
        keep = arr
    return d, keep


def _f32(t):
    if t is None:
        return None
    t = t.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


def aggregate_rows(x_src, x_dst=None, edge_attr=None, pre=None, backward=False):
    """(dgcn_dtype, x_src, x_dst, edge_attr) as the GENConv and GIN / GraphSAGE aggregate kernels read them.

    bf16 / fp16 rows are read as they are (widened to fp32 in registers: bit for bit the result of the fp32 copy)
    when x_src is bf16 or fp16, x_dst and edge_attr (where given) have the same dtype, C % 4 == 0,
    C <= HALF_ROWS_MAX_C (HALF_ROWS_MAX_C_BWD for the backward), no pre-activation is fused and every row base is
    8-byte aligned.  Non-contiguous half rows are made contiguous in their own dtype.  Everything else gets the
    fp32 copies it always got."""
    code = _ROW_DTYPE.get(x_src.dtype)
    C = x_src.shape[-1]
    if code not in (None, DTYPE_F32) and pre is None and C % 4 == 0 and \
            C <= (HALF_ROWS_MAX_C_BWD if backward else HALF_ROWS_MAX_C) and \
            all(t is None or t.dtype == x_src.dtype for t in (x_dst, edge_attr)):
        xs = x_src.detach().contiguous()
        xd = xs if x_dst is x_src else (None if x_dst is None else x_dst.detach().contiguous())
        ea = None if edge_attr is None else edge_attr.detach().contiguous()
        if all(t is None or t.data_ptr() % 8 == 0 for t in (xs, xd, ea)):
            return code, xs, xd, ea
    return DTYPE_F32, _f32(x_src), _f32(x_dst), _f32(edge_attr)


class ConvParams:
    """Tensors of one BasicConv([2*C_in, C_out]) (gcn_lib/dense/torch_nn.py:48-58).

    sync_group: process group over which train-mode statistics are shared (SyncBatchNorm), None for local ones.
    After a synced forward, `moments` holds the cross-rank [sum | sum of squares | count] (fp64, on the device)."""

    def __init__(self, weight, bias=None, act="relu", prelu_weight=None, norm=NORM_NONE, bn_weight=None,
                 bn_bias=None, bn_mean=None, bn_var=None, bn_eps=1e-5, sync_group=None):
        self.weight = _f32(weight).reshape(weight.shape[0], -1)
        self.bias = _f32(bias)
        self.act = ACT[act.lower() if isinstance(act, str) else act]
        self.prelu_weight = _f32(prelu_weight)
        self.norm = norm
        self.bn_weight, self.bn_bias = _f32(bn_weight), _f32(bn_bias)
        self.bn_mean, self.bn_var = _f32(bn_mean), _f32(bn_var)
        self.bn_eps = float(bn_eps)
        self.batch_mean = self.batch_var = None
        self.sync_group = sync_group if norm == NORM_BATCH_TRAIN else None
        self.moments = None

    def backward_stats(self):
        """(mean, var) the backward normalises with: the forward's batch statistics in train mode, else the running
        ones."""
        return (self.batch_mean, self.batch_var) if self.norm == NORM_BATCH_TRAIN else (self.bn_mean, self.bn_var)

    def grad_buffers(self, x_shape, dev, need_x=True):
        """The gradients a backward writes, in the order of the C ABI's gradient arguments: x (of shape x_shape,
        when need_x), weight, and bias, BatchNorm affine and PReLU weight where the layer has them."""
        f = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        c_out, bn = self.weight.shape[0], self.norm != NORM_NONE
        return {"x": f(*x_shape) if need_x else None, "weight": f(*self.weight.shape),
                "bias": f(c_out) if self.bias is not None else None,
                "bn_weight": f(c_out) if bn else None, "bn_bias": f(c_out) if bn else None,
                "prelu": f(1) if self.prelu_weight is not None else None}

    def tensors(self):
        return (self.weight, self.bias, self.prelu_weight, self.bn_weight, self.bn_bias, self.bn_mean, self.bn_var)

    def c_struct(self, dev, stats=None):
        """dgcn_basic_conv of these tensors.  stats None (forward): bn_mean / bn_var are the running statistics, and
        in train mode new batch_mean / batch_var tensors receive the batch statistics.  stats = (mean, var)
        (backward): the statistics the forward normalised with; nothing is allocated."""
        c_out = self.weight.shape[0]
        s = BasicConvC()
        s.weight, s.bias = _ptr(self.weight), _ptr(self.bias)
        s.act, s.slope, s.prelu_weight = self.act, 0.2, _ptr(self.prelu_weight)
        s.norm = self.norm
        s.bn_weight, s.bn_bias = _ptr(self.bn_weight), _ptr(self.bn_bias)
        mean, var = (self.bn_mean, self.bn_var) if stats is None else stats
        s.bn_mean, s.bn_var, s.bn_eps = _ptr(mean), _ptr(var), self.bn_eps
        if stats is None and self.norm == NORM_BATCH_TRAIN:
            self.batch_mean = torch.empty(c_out, dtype=torch.float32, device=dev)
            self.batch_var = torch.empty(c_out, dtype=torch.float32, device=dev)
            s.batch_mean_out, s.batch_var_out = _ptr(self.batch_mean), _ptr(self.batch_var)
        return s


def _basic_conv_call(fn, prm, nbytes, dev, *args):
    """fn(*args, sync, ws, ws_bytes, stream), the call every BasicConv entry point ends with, in a workspace of nbytes.
    With prm.sync_group the call gets a dgcn_bn_sync, and a failed reduce is raised with the all-reduce's exception as
    its cause.  Returns the cross-rank moments of a synced call, else None."""
    bs = None if prm.sync_group is None else _BnSync(prm.sync_group, prm.weight.shape[0], dev)
    ws = _workspace(nbytes, dev)
    rc = fn(*args, None if bs is None else ctypes.byref(bs.c), _ptr(ws), ws.numel(), _stream(dev))
    (_check if bs is None else bs.check)(rc, fn.__name__)
    return None if bs is None else bs.moments


def knn_graph(x, k, dilation=1, cols=None, exclude_self=False, want_edge_index=True, want_nbr=False):
    """dgcn_knn_graph: returns (edge_index (2,B,N,k) int64 | None, nbr (B,N,k) int32 | None)."""
    _require_cuda(x)
    x3, B, C, N, sb, sc = _dense_view(x)
    K = int(k) * int(dilation)
    if K > N - (1 if exclude_self else 0):
        raise RuntimeError("selected index k out of range")      # what torch.topk says in the reference
    dev = x3.device
    with torch.cuda.device(dev):
        l = lib()
        dil, keep = _dilation(k, dilation, cols)
        ei = torch.empty((2, B, N, k), dtype=torch.int64, device=dev) if want_edge_index else None
        nbr = torch.empty((B, N, k), dtype=torch.int32, device=dev) if want_nbr else None
        ws = _workspace(l.dgcn_knn_graph_workspace_bytes(B, C, N, K), dev)
        rc = l.dgcn_knn_graph(_ptr(x3), B, C, N, sb, sc, ctypes.byref(dil), int(bool(exclude_self)), _ptr(ei),
                              _ptr(nbr), _ptr(ws), ws.numel(), _stream(dev))
        _check(rc, "dgcn_knn_graph")
    return ei, nbr


def graph_conv_forward(conv, x, prm, edge_index=None, nbr=None):
    """dgcn_graph_conv_forward: out (B, C_out, N, 1)."""
    _require_cuda(x, edge_index, nbr, *prm.tensors())
    x3, B, C, N, sb, sc = _dense_view(x)
    dev = x3.device
    c_out = prm.weight.shape[0]
    if edge_index is not None:
        if edge_index.dtype != torch.int64:
            edge_index = edge_index.long()
        edge_index = edge_index.contiguous()
        k = edge_index.shape[-1]
    else:
        nbr = nbr.contiguous()
        k = nbr.shape[-1]
    with torch.cuda.device(dev):
        l = lib()
        cs = prm.c_struct(dev)
        out = torch.empty((B, c_out, N, 1), dtype=torch.float32, device=dev)
        prm.moments = _basic_conv_call(l.dgcn_graph_conv_forward, prm,
                                       l.dgcn_graph_conv_workspace_bytes(CONV[conv], B, C, c_out, N, k), dev,
                                       CONV[conv], _ptr(x3), B, C, N, sb, sc, _ptr(edge_index), _ptr(nbr), k,
                                       ctypes.byref(cs), c_out, _ptr(out))
    return out


def dyn_conv_forward(conv, x, prm, k, dilation=1, cols=None, want_nbr=False, residual=None, res_scale=1.0, out=None):
    """dgcn_dyn_conv_forward: (out (B, C_out, N, 1), nbr (B,N,k) int32 | None).

    residual (B, C_out, N[, 1]): out = conv + residual * res_scale (ResDynBlock2d); out: write into this tensor, which
    may be a channel slice of a wider (B, C_total, N, 1) buffer (inference only, no train-mode BatchNorm)."""
    _require_cuda(x, residual, out, *prm.tensors())
    x3, B, C, N, sb, sc = _dense_view(x)
    K = int(k) * int(dilation)
    if K > N:
        raise RuntimeError("selected index k out of range")
    dev = x3.device
    c_out = prm.weight.shape[0]
    with torch.cuda.device(dev):
        l = lib()
        cs = prm.c_struct(dev)
        dil, keep = _dilation(k, dilation, cols)
        fus = None
        if residual is not None or out is not None:
            fus = BlockFusionC()
            if residual is not None:
                r3, rB, rC, rN, rsb, rsc = _dense_view(residual)
                if (rB, rC, rN) != (B, c_out, N):
                    raise RuntimeError("dyn_conv_forward: residual must be (B, C_out, N, 1)")
                fus.residual, fus.res_stride_b, fus.res_stride_c, fus.res_scale = _ptr(r3), rsb, rsc, float(res_scale)
            if out is not None:
                if tuple(out.shape[:3]) != (B, c_out, N) or out.dtype != torch.float32 or out.stride(2) != 1 or \
                        out.stride(1) != N:
                    raise RuntimeError("dyn_conv_forward: out must be a (B, C_out, N, 1) fp32 channel slice")
                fus.out_stride_b = out.stride(0)
        if out is None:
            out = torch.empty((B, c_out, N, 1), dtype=torch.float32, device=dev)
        nbr = torch.empty((B, N, k), dtype=torch.int32, device=dev) if want_nbr else None
        if prm.sync_group is not None and fus is not None:
            raise RuntimeError("dyn_conv_forward: the block epilogue does not run with train-mode BatchNorm")
        prm.moments = _basic_conv_call(l.dgcn_dyn_conv_forward, prm,
                                       l.dgcn_dyn_conv_workspace_bytes(CONV[conv], B, C, c_out, N, K), dev,
                                       CONV[conv], _ptr(x3), B, C, N, sb, sc, ctypes.byref(dil), ctypes.byref(cs),
                                       c_out, _ptr(out), _ptr(nbr), None if fus is None else ctypes.byref(fus))
    return out, nbr


def graph_conv_backward(conv, x, prm, grad_out, edge_index=None, nbr=None, need_x=True):
    """dgcn_graph_conv_backward: dict of gradients (x, weight, bias, bn_weight, bn_bias, prelu)."""
    _require_cuda(x, grad_out, edge_index, nbr)
    x3, B, C, N, sb, sc = _dense_view(x)
    dev = x3.device
    c_out = prm.weight.shape[0]
    go = _f32(grad_out).reshape(B, c_out, N)
    if edge_index is not None:
        edge_index = edge_index.long().contiguous()
        k = edge_index.shape[-1]
    else:
        nbr = nbr.contiguous()
        k = nbr.shape[-1]
    with torch.cuda.device(dev):
        l = lib()
        cs = prm.c_struct(dev, prm.backward_stats())
        g = prm.grad_buffers((B, C, N), dev, need_x)
        # synced: dx from the cross-rank sums; the parameter gradients stay local (SyncBatchNorm)
        _basic_conv_call(l.dgcn_graph_conv_backward, prm,
                         l.dgcn_graph_conv_backward_workspace_bytes(CONV[conv], B, C, c_out, N, k), dev,
                         CONV[conv], _ptr(x3), B, C, N, sb, sc, _ptr(edge_index), _ptr(nbr), k, ctypes.byref(cs),
                         c_out, _ptr(go), *map(_ptr, g.values()))
    return g


def csr_build(edge_index, num_nodes):
    """dgcn_csr_build: (rowptr (N+1), src (E), eid (E)) int32, rows = destinations, stable."""
    _require_cuda(edge_index)
    if edge_index.dtype != torch.int64:
        edge_index = edge_index.long()
    edge_index = edge_index.contiguous()
    E = edge_index.shape[1]
    dev = edge_index.device
    with torch.cuda.device(dev):
        l = lib()
        rowptr = torch.empty(num_nodes + 1, dtype=torch.int32, device=dev)
        src = torch.empty(max(E, 1), dtype=torch.int32, device=dev)
        eid = torch.empty(max(E, 1), dtype=torch.int32, device=dev)
        ws = _workspace(l.dgcn_csr_build_workspace_bytes(num_nodes, E), dev)
        rc = l.dgcn_csr_build(_ptr(edge_index), E, num_nodes, _ptr(rowptr), _ptr(src), _ptr(eid), _ptr(ws),
                              ws.numel(), _stream(dev))
        _check(rc, "dgcn_csr_build")
        # long rows (hubs of power-law graphs): (row, segment) work items, listed once, on the device
        hubs = None
        if E >= HUB_MIN_DEGREE:
            max_items = E // HUB_SEG_EDGES + E // HUB_MIN_DEGREE + 2
            max_rows = E // HUB_MIN_DEGREE + 2
            items = torch.empty(2 * max_items, dtype=torch.int32, device=dev)
            rows = torch.empty(3 * max_rows, dtype=torch.int32, device=dev)
            counts = torch.zeros(2, dtype=torch.int32, device=dev)
            _check(l.dgcn_csr_hub_rows(_ptr(rowptr), num_nodes, E, HUB_MIN_DEGREE, HUB_SEG_EDGES, _ptr(items),
                                       _ptr(rows), _ptr(counts), _stream(dev)), "dgcn_csr_hub_rows")
            n_items = int(counts[0])            # one-time host read at graph-build time
            if n_items > 0:
                hubs = (items, rows, counts, n_items)
    # (src / eid keep >= 1 element: a 0-element tensor has a null data_ptr)
    return rowptr, src, eid, hubs


def _sparse_rows(x, csr):
    """x (N, C_in) as the sparse EdgeConv reads it (fp32, contiguous) and the CSR's rowptr / src."""
    rowptr, src = csr[0], csr[1]
    _require_cuda(x, rowptr, src)
    if x.dim() != 2 or x.dtype != torch.float32:
        raise RuntimeError("sparse EdgeConv takes fp32 (N, C) node features, got %s %s" % (x.dtype, tuple(x.shape)))
    return x.detach().contiguous(), rowptr, src


def sparse_edge_conv_forward(x, csr, E, prm):
    """dgcn_sparse_edge_conv_forward: out (N, C_out) over the CSR graph (csr_build) of E edges; in train mode
    prm.batch_mean / prm.batch_var receive the batch statistics of the E edge rows (with prm.sync_group, of every
    rank's edge rows, and prm.moments their cross-rank moments)."""
    x, rowptr, src = _sparse_rows(x, csr)
    _require_cuda(*prm.tensors())
    N, C = x.shape
    c_out = prm.weight.shape[0]
    dev = x.device
    with torch.cuda.device(dev):
        l = lib()
        cs = prm.c_struct(dev)
        out = torch.empty((N, c_out), dtype=torch.float32, device=dev)
        prm.moments = _basic_conv_call(l.dgcn_sparse_edge_conv_forward, prm,
                                       l.dgcn_sparse_edge_conv_workspace_bytes(N, C, c_out), dev,
                                       _ptr(x), N, C, _ptr(rowptr), _ptr(src), int(E), ctypes.byref(cs), c_out,
                                       _ptr(out))
    return out


def sparse_edge_conv_backward(x, csr, E, prm, grad_out, need_x=True):
    """dgcn_sparse_edge_conv_backward: dict of gradients (x, weight, bias, bn_weight, bn_bias, prelu)."""
    x, rowptr, src = _sparse_rows(x, csr)
    _require_cuda(grad_out)
    N, C = x.shape
    c_out = prm.weight.shape[0]
    dev = x.device
    go = _f32(grad_out)
    with torch.cuda.device(dev):
        l = lib()
        cs = prm.c_struct(dev, prm.backward_stats())
        g = prm.grad_buffers((N, C), dev, need_x)
        # synced: dx from the cross-rank sums; the parameter gradients stay local (SyncBatchNorm)
        _basic_conv_call(l.dgcn_sparse_edge_conv_backward, prm,
                         l.dgcn_sparse_edge_conv_backward_workspace_bytes(N, C, c_out), dev,
                         _ptr(x), N, C, _ptr(rowptr), _ptr(src), int(E), ctypes.byref(cs), c_out, _ptr(go),
                         *map(_ptr, g.values()))
    return g


def _scalar(prm, name, value):
    """python float -> host field; tensor (nn.Parameter) -> device pointer (no host sync)."""
    if torch.is_tensor(value):
        v = _f32(value)
        setattr(prm, name + "_dev", _ptr(v))
        setattr(prm, name, 0.0)
        return v
    setattr(prm, name, float(value))
    setattr(prm, name + "_dev", None)
    return None


def genconv_params(aggr, t=1.0, p=1.0, y=0.0, eps=1e-7, msg_scale=None, add_residual=True):
    if aggr not in AGGR:
        raise NotImplementedError("To be implemented")           # torch_message.py:84-85
    prm = GenconvParamsC()
    prm.aggr = AGGR[aggr]
    keep = [_scalar(prm, "t", t), _scalar(prm, "p", p), _scalar(prm, "y", y)]
    prm.eps = float(eps)
    prm.msg_norm = 0 if msg_scale is None else 1
    keep.append(_scalar(prm, "msg_scale", 1.0 if msg_scale is None else msg_scale))
    prm.add_residual = int(bool(add_residual))
    prm.raw_message = 0
    return prm, keep


def _keep_mask(keep):
    """keep = (bits (N, W) int32 from keep_bits, keep_scale) -> (dgcn_keep_mask, bits) | (None, None)."""
    if keep is None:
        return None, None
    bits = keep[0]
    if bits.dtype != torch.int32 or bits.dim() != 2 or not bits.is_contiguous():
        raise RuntimeError("keep bits must be a contiguous (N, W) int32 tensor (keep_bits)")
    return KeepMaskC(_ptr(bits), bits.shape[1], float(keep[1])), bits


ERR_UNSUPPORTED = -2       # dgcn_status: a valid request the kernels do not cover
RAW_MAX_C = 1024           # raw aggregate, forward: the widest launch on float4 rows (C % 4 == 0, 16-byte aligned) ...
RAW_MAX_C_VEC1 = 256       # ... and on any other rows (one channel per lane)
RAW_MAX_C_BWD = 512        # ... backward: the widest launch


def raw_channel_slices(C, backward=False):
    """[(c0, c1)]: contiguous channel slices covering 0 .. C, each a launch the raw aggregate kernels accept on a fresh
    contiguous (so 16-byte aligned) copy of its rows.  Backward: RAW_MAX_C_BWD channels at a time.  Forward: RAW_MAX_C
    at a time, and a last slice that is wider than RAW_MAX_C_VEC1 with C % 4 != 0 becomes its multiple-of-4 part plus
    the last C % 4 channels."""
    step = RAW_MAX_C_BWD if backward else RAW_MAX_C
    cuts = list(range(0, C, step)) + [C]
    if not backward and C % 4 and C - cuts[-2] > RAW_MAX_C_VEC1:
        cuts.insert(-1, C - C % 4)
    return list(zip(cuts[:-1], cuts[1:]))


def _fresh(t):
    """A contiguous copy of t in a new (so 16-byte aligned) allocation, even when t is contiguous already."""
    return t.clone(memory_format=torch.contiguous_format)


def _channel_separable(prm, x_dst, edge_attr, pre, keep, rows=None, skip_hubs=False):
    """Raw messages without MsgNorm, residual, edge rows or block fusion: every output channel depends on its own input
    channel only, so the aggregate may run on channel slices.  (MsgNorm couples the channels of a row.)"""
    return bool(prm.raw_message) and not prm.msg_norm and not prm.add_residual and x_dst is None and \
        edge_attr is None and pre is None and keep is None and rows is None and not skip_hubs


def genconv_aggregate(x_src, x_dst, csr, prm, edge_attr=None, out=None, pre=None, rows=None, skip_hubs=False,
                      keep=None):
    """dgcn_genconv_aggregate: out (N, C) = x_dst + MsgNorm(aggregate(message)).

    out: write into this (N, C) tensor (e.g. a view of a persistent buffer) instead of a new one.
    pre = (scale (C), shift (C), relu): rows of x_src / x_dst are read as act(scale * x + shift).
    keep = (bits, keep_scale) (dgcn_keep_mask, with pre and relu): rows are read as
    keep ? relu(scale * x + shift) * keep_scale : 0 (dropout in training).
    rows (int32) / skip_hubs: destination rows of this launch (dgcn_genconv_fusion).
    Raw messages (prm.raw_message, x_dst None, nothing fused) at a C the kernels refuse - C > RAW_MAX_C, or
    C > RAW_MAX_C_VEC1 on rows that are not float4-able - run as one launch per raw_channel_slices slice, each on a
    contiguous copy of its channels, written into one (N, C) output.  Each channel sums or compares the same edges in
    the same order in any channel block, so the bits are those a single launch would give."""
    rc, out = _genconv_aggregate(x_src, x_dst, csr, prm, edge_attr, out, pre, rows, skip_hubs, keep)
    if rc == ERR_UNSUPPORTED and _channel_separable(prm, x_dst, edge_attr, pre, keep, rows, skip_hubs):
        x_src = x_src.detach()
        for c0, c1 in raw_channel_slices(x_src.shape[1]):
            rc, part = _genconv_aggregate(_fresh(x_src[:, c0:c1]), None, csr, prm)
            _check(rc, "dgcn_genconv_aggregate")
            out[:, c0:c1] = part
        return out
    _check(rc, "dgcn_genconv_aggregate")
    return out


def _genconv_aggregate(x_src, x_dst, csr, prm, edge_attr=None, out=None, pre=None, rows=None, skip_hubs=False,
                       keep=None):
    """One dgcn_genconv_aggregate call: (status, out)."""
    rowptr, src, eid = csr[:3]
    _require_cuda(x_src, x_dst, rowptr, src, eid, edge_attr, out, rows, None if keep is None else keep[0])
    dtype, x_src, x_dst, edge_attr = aggregate_rows(x_src, x_dst, edge_attr, pre=pre)
    km, _bits = _keep_mask(keep)
    N, C = rowptr.numel() - 1, x_src.shape[1]
    dev = x_src.device
    hubs = None
    with torch.cuda.device(dev):
        if len(csr) > 3 and csr[3] is not None:
            items, hrows, counts, n_items = csr[3]
            partial = torch.empty(n_items * 3 * C, dtype=torch.float32, device=dev)
            hubs = CsrHubsC(_ptr(items), _ptr(hrows), _ptr(counts), HUB_MIN_DEGREE, HUB_SEG_EDGES, _ptr(partial))
        if out is None:
            out = torch.empty((N, C), dtype=torch.float32, device=dev)
        elif out.shape != (N, C) or out.dtype != torch.float32 or not out.is_contiguous():
            raise RuntimeError("genconv_aggregate: out must be a contiguous fp32 (N, C) tensor")
        elif dtype != DTYPE_F32 and out.data_ptr() % 16 != 0:       # half rows store out as float4
            dtype, x_src, x_dst, edge_attr = DTYPE_F32, _f32(x_src), _f32(x_dst), _f32(edge_attr)
        fus, keep = None, None
        if pre is not None or rows is not None or skip_hubs:
            fus = GenconvFusionC()
            if pre is not None:
                keep = (_f32(pre[0]), _f32(pre[1]))
                fus.pre_scale, fus.pre_shift, fus.pre_relu = _ptr(keep[0]), _ptr(keep[1]), int(bool(pre[2]))
            fus.skip_hubs = int(bool(skip_hubs))
            if rows is not None:
                if rows.dtype != torch.int32 or not rows.is_contiguous():
                    raise RuntimeError("genconv_aggregate: rows must be a contiguous int32 tensor")
                fus.row_list, fus.n_rows = (rows.data_ptr() or None), rows.numel()
                if rows.numel() == 0 and skip_hubs:
                    return 0, out
        rc = lib().dgcn_genconv_aggregate(dtype, _ptr(x_src), _ptr(x_dst), N, C, _ptr(rowptr), _ptr(src), _ptr(eid),
                                          _ptr(edge_attr), ctypes.byref(prm),
                                          ctypes.byref(hubs) if hubs is not None else None,
                                          ctypes.byref(fus) if fus is not None else None,
                                          ctypes.byref(km) if km is not None else None, _ptr(out), _stream(dev))
    return rc, out


def genconv_aggregate_backward(x_src, x_dst, csr, prm, grad_out, edge_attr=None, softmax_grad=False,
                               need_edge_attr=False, pre=None, keep=None):
    """dgcn_genconv_aggregate_backward: (grad_x_src (N_src,C) fp32, grad_x_dst (N,C) fp32 | None,
    grad_edge_attr in edge_attr's row dtype | None, grad_scalars (4) = d/dt, d/dp, d/dy, d/dmsg_scale).
    pre / keep: the forward's (genconv_aggregate); the row gradients are then w.r.t. the activated rows.
    Raw messages past RAW_MAX_C_BWD channels (x_dst None, nothing fused) run as one launch per raw_channel_slices
    slice, as in genconv_aggregate; the scalar gradients are summed over the slices."""
    rc, res = _genconv_aggregate_backward(x_src, x_dst, csr, prm, grad_out, edge_attr, softmax_grad, need_edge_attr,
                                          pre, keep)
    if rc == ERR_UNSUPPORTED and _channel_separable(prm, x_dst, edge_attr, pre, keep):
        gsrc, gsc = res[0], res[3]
        x_src, grad_out = x_src.detach(), grad_out.detach()
        for c0, c1 in raw_channel_slices(x_src.shape[1], backward=True):
            rc, part = _genconv_aggregate_backward(_fresh(x_src[:, c0:c1]), None, csr, prm,
                                                   _fresh(grad_out[:, c0:c1]), softmax_grad=softmax_grad)
            _check(rc, "dgcn_genconv_aggregate_backward")
            gsrc[:, c0:c1] = part[0]
            gsc += part[3]
        return res
    _check(rc, "dgcn_genconv_aggregate_backward")
    return res


def _genconv_aggregate_backward(x_src, x_dst, csr, prm, grad_out, edge_attr=None, softmax_grad=False,
                                need_edge_attr=False, pre=None, keep=None):
    """One dgcn_genconv_aggregate_backward call: (status, (grad_x_src, grad_x_dst, grad_edge_attr, grad_scalars))."""
    rowptr, src, eid = csr[:3]
    _require_cuda(x_src, x_dst, grad_out, edge_attr)
    dtype, x_src, x_dst, edge_attr = aggregate_rows(x_src, x_dst, edge_attr, pre=pre, backward=True)
    km, _bits = _keep_mask(keep)
    ps = ph = None
    if pre is not None:
        ps, ph = _f32(pre[0]), _f32(pre[1])
    grad_out = _f32(grad_out)
    N, C = rowptr.numel() - 1, x_src.shape[1]
    dev = x_src.device
    with torch.cuda.device(dev):
        gsrc = torch.zeros(x_src.shape, dtype=torch.float32, device=dev)
        gdst = torch.empty((N, C), dtype=torch.float32, device=dev) if x_dst is not None else None
        gea = None
        if need_edge_attr and edge_attr is not None:
            # half rows: every CSR edge writes its row once (rounded like Tensor.to), so when edge_attr has one row
            # per edge nothing needs clearing (src keeps >= 1 element; an edgeless graph takes the zeros)
            full = dtype != DTYPE_F32 and edge_attr.shape[0] == src.numel() and edge_attr.shape[0] > 1
            gea = torch.empty_like(edge_attr) if full else torch.zeros_like(edge_attr)
        gsc = torch.zeros(4, dtype=torch.float32, device=dev)
        rc = lib().dgcn_genconv_aggregate_backward(dtype, _ptr(x_src), _ptr(x_dst), N, x_src.shape[0], C,
                                                   _ptr(rowptr), _ptr(src), _ptr(eid), _ptr(edge_attr),
                                                   ctypes.byref(prm), int(bool(softmax_grad)), _ptr(ps), _ptr(ph),
                                                   int(bool(pre[2])) if pre is not None else 0,
                                                   ctypes.byref(km) if km is not None else None, _ptr(grad_out),
                                                   _ptr(gsrc), _ptr(gdst), _ptr(gea), _ptr(gsc), _stream(dev))
    return rc, (gsrc, gdst, gea, gsc)


def _gin_sage_args(rule, x, csr, eps, half_rows=False):
    """half_rows: x may also be bf16 / fp16 (the forward's node features; the backward's gradient is fp32)."""
    if rule not in GIN_SAGE:
        raise ValueError("gin_sage_aggregate: rule must be one of %s, got %r" % (sorted(GIN_SAGE), rule))
    rowptr, src = csr[0], csr[1]
    _require_cuda(x, rowptr, src, eps)
    if x.dim() != 2 or x.dtype not in (_ROW_DTYPE if half_rows else (torch.float32,)):
        raise RuntimeError("the GIN / SAGE aggregation takes %s (N, C) node features, got %s %s"
                           % ("fp32, bf16 or fp16" if half_rows else "fp32", x.dtype, tuple(x.shape)))
    if rowptr.numel() - 1 != x.shape[0]:
        raise RuntimeError("gin_sage_aggregate: the CSR graph has %d rows, x has %d" % (rowptr.numel() - 1, x.shape[0]))
    return rowptr, src, None if (eps is None or rule != "gin") else _f32(eps).reshape(1)


def gin_sage_aggregate(rule, x, csr, eps=None):
    """dgcn_gin_sage_aggregate: (N, C) fp32 = sum_j x_j + (1 + eps) x_i ('gin', eps a (1,) tensor or None for 0), or
    the mean over {j -> i, j != i} + {i} of x_j ('sage') / of x_j - x_i ('rsage'), over the CSR graph (csr_of).
    x fp32, bf16 or fp16: half rows are read as they are where aggregate_rows allows, else as an fp32 copy; either
    way the result is bit for bit that of the call on x.float()."""
    rowptr, src, eps = _gin_sage_args(rule, x, csr, eps, half_rows=True)
    dtype, x, _, _ = aggregate_rows(x)
    N, C = x.shape
    dev = x.device
    with torch.cuda.device(dev):
        hubs = None
        if len(csr) > 3 and csr[3] is not None:
            items, hrows, counts, n_items = csr[3]
            partial = torch.empty(n_items * 3 * C, dtype=torch.float32, device=dev)
            hubs = CsrHubsC(_ptr(items), _ptr(hrows), _ptr(counts), HUB_MIN_DEGREE, HUB_SEG_EDGES, _ptr(partial))
        out = torch.empty((N, C), dtype=torch.float32, device=dev)
        rc = lib().dgcn_gin_sage_aggregate(dtype, GIN_SAGE[rule], _ptr(x), N, C, _ptr(rowptr), _ptr(src),
                                           ctypes.byref(hubs) if hubs is not None else None, _ptr(eps), _ptr(out),
                                           _stream(dev))
        _check(rc, "dgcn_gin_sage_aggregate")
    return out


def gin_sage_aggregate_backward(rule, grad_out, csr, eps=None):
    """dgcn_gin_sage_aggregate_backward: grad_x (N, C) fp32 of gin_sage_aggregate for the upstream grad_out."""
    rowptr, src, eps = _gin_sage_args(rule, grad_out, csr, eps)
    go = _f32(grad_out)
    N, C = go.shape
    dev = go.device
    with torch.cuda.device(dev):
        gx = torch.zeros((N, C), dtype=torch.float32, device=dev)
        rc = lib().dgcn_gin_sage_aggregate_backward(GIN_SAGE[rule], N, C, _ptr(rowptr), _ptr(src), _ptr(eps), _ptr(go),
                                                    _ptr(gx), _stream(dev))
        _check(rc, "dgcn_gin_sage_aggregate_backward")
    return gx


def keep_bits(keep):
    """dgcn_keep_bits_pack: keep (N, C) fp32 (non-zero = kept) -> (N, ceil(C / 32)) int32, bit c % 32 of word c / 32."""
    _require_cuda(keep)
    keep = _f32(keep)
    N, C = keep.shape
    with torch.cuda.device(keep.device):
        bits = torch.empty((N, (C + 31) // 32), dtype=torch.int32, device=keep.device)
        _check(lib().dgcn_keep_bits_pack(_ptr(keep), N, C, _ptr(bits), _stream(keep.device)), "dgcn_keep_bits_pack")
    return bits


def res_plus_backward_gy(h, scale, shift, keep, grad_src, grad_dst, mean=None, invstd=None):
    """dgcn_res_plus_backward_gy: grad_src <- g_y (in place); returns the fp64 (2, C) [sum g_y | sum g_y * xhat]
    when mean / invstd are given, else None."""
    _require_cuda(h, grad_src, grad_dst)
    N, C = h.shape
    km, _bits = _keep_mask(keep)
    with torch.cuda.device(h.device):
        sums = torch.zeros((2, C), dtype=torch.float64, device=h.device) if mean is not None else None
        _check(lib().dgcn_res_plus_backward_gy(_ptr(h), N, C, _ptr(scale), _ptr(shift),
                                               ctypes.byref(km) if km is not None else None, _ptr(mean), _ptr(invstd),
                                               _ptr(grad_src), _ptr(grad_dst), _ptr(sums), _stream(h.device)),
               "dgcn_res_plus_backward_gy")
    return sums


def res_plus_backward_dh(g_y, h, a, b=None, d=None, grad_skip=None, out=None):
    """dgcn_res_plus_backward_dh: a * g_y + b * h + d + grad_skip per channel (out may be grad_skip)."""
    _require_cuda(g_y, h, grad_skip)
    N, C = g_y.shape
    with torch.cuda.device(g_y.device):
        out = torch.empty_like(g_y) if out is None else out
        _check(lib().dgcn_res_plus_backward_dh(_ptr(g_y), _ptr(h), N, C, _ptr(a), _ptr(b), _ptr(d), _ptr(grad_skip),
                                               _ptr(out), _stream(g_y.device)), "dgcn_res_plus_backward_dh")
    return out


def linear_residual_supported(K, M):
    return lib().dgcn_linear_residual_workspace_bytes(int(K), int(M)) > 0


def linear_residual(a, weight, bias=None, res=None, out=None):
    """dgcn_linear_residual: out (N, M) = a @ weight^T (+ bias) (+ res) on the tensor cores (wgmma)."""
    _require_cuda(a, weight, bias, res, out)
    a, weight, bias, res = _f32(a), _f32(weight), _f32(bias), _f32(res)
    N, K = a.shape
    M = weight.shape[0]
    dev = a.device
    with torch.cuda.device(dev):
        l = lib()
        nbytes = l.dgcn_linear_residual_workspace_bytes(K, M)
        if nbytes == 0:
            raise RuntimeError("dgcn_linear_residual: unsupported shape K=%d M=%d" % (K, M))
        if out is None:
            out = torch.empty((N, M), dtype=torch.float32, device=dev)
        elif out.shape != (N, M) or out.dtype != torch.float32 or not out.is_contiguous():
            raise RuntimeError("linear_residual: out must be a contiguous fp32 (N, M) tensor")
        ws = _workspace(nbytes, dev)
        _check(l.dgcn_linear_residual(_ptr(a), N, K, _ptr(weight), _ptr(bias), M, _ptr(res), _ptr(out), _ptr(ws),
                                      ws.numel(), _stream(dev)), "dgcn_linear_residual")
    return out


def gather_rows(x, rows, out=None):
    """out[r] = x[rows[r]] in x's dtype (fp32, bf16 or fp16; other dtypes are copied as fp32)."""
    _require_cuda(x, rows, out)
    dtype = _ROW_DTYPE.get(x.dtype)
    x = x.detach().contiguous() if dtype is not None else _f32(x)
    dtype = DTYPE_F32 if dtype is None else dtype
    rows = rows.to(torch.int32).contiguous()
    R, C = rows.numel(), x.shape[1]
    with torch.cuda.device(x.device):
        if out is None:
            out = torch.empty((R, C), dtype=x.dtype, device=x.device)
        elif out.dtype != x.dtype or out.shape != (R, C) or not out.is_contiguous():
            raise RuntimeError("gather_rows: out must be a contiguous (R, C) tensor of x's dtype")
        _check(lib().dgcn_gather_rows(dtype, _ptr(x), C, _ptr(rows), R, _ptr(out), _stream(x.device)),
               "dgcn_gather_rows")
    return out


def kernel_timing(enable):
    """Switch the event bracket around each path's dominant kernel on/off (bench.py)."""
    return lib().dgcn_debug_kernel_timing(int(bool(enable)))


def kernel_timing_read(tag):
    """(total_ms, launches) of the bracketed kernel `tag` since the last read."""
    ms, n = ctypes.c_double(0.0), c_i64(0)
    _check(lib().dgcn_debug_kernel_timing_read(tag.encode(), ctypes.byref(ms), ctypes.byref(n)),
           "dgcn_debug_kernel_timing_read")
    return ms.value, n.value


def tc_certification(enable):
    """Count the queries the tensor-core pre-filter leaves uncertified (dgcn_debug_tc_certification; synchronises
    after every selection while enabled)."""
    return lib().dgcn_debug_tc_certification(int(bool(enable)))


def tc_certification_read():
    """(uncertified queries, queries) since the last read."""
    failed, total = c_i64(0), c_i64(0)
    _check(lib().dgcn_debug_tc_certification_read(ctypes.byref(failed), ctypes.byref(total)),
           "dgcn_debug_tc_certification_read")
    return failed.value, total.value


def set_knn_path(path):
    """A/B switch for tests and measurements: 'ffma' makes the calls of THIS thread pass
    DGCN_KNN_EXACT_FP32 (fp32 FMA selection kernels only); 'tc1' passes DGCN_KNN_TC_TILE_PER_CTA (tensor-core
    pre-filter, always the one-tile-per-CTA kernel); 'tc' / 'auto' = the default routing (tensor-core pre-filter +
    exact re-rank where the shape allows, several query tiles per CTA where that kernel applies).  The library
    holds no state."""
    _knn_flags.value = {"ffma": KNN_EXACT_FP32, "tc1": KNN_TC_TILE_PER_CTA, "tc": 0, "auto": 0}[path]
