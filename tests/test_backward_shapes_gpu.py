"""Gradients of the dense graph convolutions (dgcn_graph_conv_backward) at the shapes training runs, against fp64
torch autograd through oracle.dense on the graph the kernel used (tests/backward_util.py).

Every case checks the forward output and every gradient the layer has, elementwise.  EdgeConv cases zero the
upstream gradient at the near-ties of the max (at most 1e-3 of the entries); MRConv cases use seeds without
near-ties.  Each case prints its worst |got - ref| / max|ref| per gradient and the masked fraction.

Paths of dgcn_graph_conv_backward (dense_bwd.cu, its GEMMs in basic_conv.cu), and the case that reaches each:
  wgrad_kernel over several KCH = 512 chunks with a partial last one     a (2 chunks), c (8), d (3, 6-point tail)
  tile_gemm_kernel / wgrad_kernel over several 128-wide tiles              d (C_in 130 / 160, 2 C_out = 192)
  unaligned operands (ci % 4 != 0, vec = 0, N % 4 != 0)                   b (C_in 3, N 1030, misaligned x), d
  strided x (stride_b != C N) in wgrad_kernel and MRConv's kmajor2         b
  nbr of the fused slab path (K > 48) and of stochastic columns          a (K 60, 540), c (K 100), f
  edge_of with arbitrary centres (edge_index[1] != arange)               e
  grad_x == nullptr (need_x False)                                        b
"""
import copy

import pytest
import torch

import backward_util as bu
from oracle import dense as od

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4


def _init_params(mod, g, slope=None):
    """Random BN affine parameters and running statistics, every third gamma negative (the max becomes a min);
    PReLU slope `slope`."""
    for m in mod.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            c = m.num_features
            m.weight.data = torch.randn(c, generator=g) * 0.5 + 0.8
            m.weight.data[::3] *= -1
            m.bias.data = torch.randn(c, generator=g) * 0.2
            m.running_mean.data = torch.randn(c, generator=g) * 0.3
            m.running_var.data = torch.rand(c, generator=g) + 0.4
        if isinstance(m, torch.nn.PReLU) and slope is not None:
            m.weight.data.fill_(slope)
    return mod


def _fused_graph(dyn, xc, cols=None):
    """The graph DynConv2d's fused forward hands to the backward (its int32 nbr list) must be the one
    dilated_knn_graph builds; returns that (2,B,N,k) graph."""
    from deep_gcns_torch_b200 import _native
    gc = dyn.gconv
    with torch.no_grad():
        if cols is None:
            ei = dyn.dilated_knn_graph(xc)
        else:
            ei = _native.knn_graph(xc, dyn.k, dyn.d, cols=cols)[0]
            full = _native.knn_graph(xc, dyn.k * dyn.d, 1)[0]
            assert torch.equal(ei, full[:, :, :, torch.as_tensor(cols, device=xc.device)])
        _, nbr = _native.dyn_conv_forward(gc._conv, xc, gc._conv_params(), dyn.k, dyn.d, cols, want_nbr=True)
    assert torch.equal(nbr.long(), ei[0])
    return ei


def _check(tag, run, x, ei, gconv, conv, act, norm, train, grad_x, knn=None, skip=None, seed=0):
    """run() -> the layer's output on the GPU, computed from an input whose values are x (CPU fp32) and whose
    gradient grad_x() returns (None: the input does not require grad).  ei: the graph the kernel used."""
    nn_cpu = copy.deepcopy(gconv.nn).cpu()
    B, C, N = x.shape[:3]
    co = gconv.nn[0].out_channels + (C if skip == "cat" else 0)
    wgt = torch.randn(B, co, N, 1, generator=torch.Generator().manual_seed(seed))
    frac = None
    if conv == "edge":
        mask = bu.edge_tie_mask(x, ei, nn_cpu, act, norm, train)
        body = wgt[:, C:] if skip == "cat" else wgt
        body[mask] = 0
        frac = mask.double().mean().item()
    else:
        bu.assert_no_mr_ties(x, ei, nn_cpu, act)
    y_ref, ref = bu.oracle_grads(x, ei, nn_cpu, conv, act, norm, train, wgt, knn=knn, skip=skip)

    for p in gconv.parameters():
        p.grad = None
    y = run()
    torch.testing.assert_close(y.detach().cpu(), y_ref.float(), rtol=RTOL, atol=ATOL)
    (y * wgt.cuda()).sum().backward()
    nn_ = gconv.nn
    got = {"x": grad_x() if grad_x is not None else None, "weight": nn_[0].weight.grad, "bias": nn_[0].bias.grad}
    for m in nn_:
        if isinstance(m, torch.nn.PReLU):
            got["slope"] = m.weight.grad
        if isinstance(m, torch.nn.BatchNorm2d):
            got["bn_w"], got["bn_b"] = m.weight.grad, m.bias.grad
    ratios = {}
    for name, r in ref.items():
        if name == "x" and grad_x is None:
            continue
        assert got[name] is not None, "%s: no gradient" % name
        ratios[name] = bu.assert_grads_close("%s/%s" % (tag, name), got[name], r)
    print("backward case %s: worst |got - ref| / max|ref| %s; masked fraction %s" % (
        tag, " ".join("%s=%.2e" % kv for kv in ratios.items()), "-" if frac is None else "%.2e" % frac))
    return ratios


# -- a. MRGCN-28 (bench_models c4) backbone layer in training ---------------------------------------------------
def _case_a(d):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(100 + d)
    torch.manual_seed(d)
    mod = _init_params(D.DynConv2d(64, 64, 20, d, "mr", "relu", "batch"), g)
    return mod, torch.randn(2, 64, 1024, 1, generator=g)


@pytest.mark.parametrize("d", [1, 3, 27])
def test_c4_backbone_layer_training(d):
    """d = 1 (K 20): fused tensor-core kNN path; d = 3, 27 (K 60, 540): slab path with dist_rows_tc.  The
    backward runs on the nbr list of either; N = 1024 gives wgrad_kernel two KCH chunks."""
    mod, x = _case_a(d)
    mod = mod.cuda().train()
    xc = x.cuda().requires_grad_(True)
    ei = _fused_graph(mod, xc.detach())
    _check("a-d%d" % d, lambda: mod(xc), x, ei, mod.gconv, "mr", "relu", "batch", True, lambda: xc.grad,
           knn=dict(K=20 * d, dilation=d), seed=d)


# -- b. MRGCN-28 head: the 3 position channels of the inputs ----------------------------------------------------
def _case_b():
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(11)
    torch.manual_seed(11)
    mod = _init_params(D.GraphConv2d(3, 64, "mr", "relu", "batch"), g)
    return mod, torch.rand(2, 9, 1024, 1, generator=g), torch.rand(2, 6, 1030, 1, generator=g)


def test_c4_head_strided_and_misaligned_input():
    """x = inputs[:, 0:3] (stride_b = 9 N: strided x in wgrad_kernel and kmajor2) without requires_grad
    (need_x False, grad_x == nullptr: weight and BN gradients only); then a requires-grad slice wide[:, 1:4]
    at N = 1030 (x not 16-byte aligned, N % 4 != 0: vec = 0; ci = 3: ci % 4 != 0), whose gradient must land
    in `wide` and nowhere else."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    mod, inputs, wide = _case_b()
    mod = mod.cuda().train()
    graph = D.DilatedKnnGraph(20, 1)
    x = inputs.cuda()[:, 0:3]
    assert x.stride(0) == 9 * 1024
    ei = graph(x)
    _check("b-head", lambda: mod(x, ei), inputs[:, 0:3], ei, mod.gconv, "mr", "relu", "batch", True, None,
           knn=dict(K=20, exclude_self=True), seed=1)

    wc = wide.cuda().requires_grad_(True)
    xs = wc[:, 1:4]
    assert xs.data_ptr() % 16 != 0
    ei = graph(xs)
    _check("b-slice", lambda: mod(xs, ei), wide[:, 1:4], ei, mod.gconv, "mr", "relu", "batch", True,
           lambda: wc.grad[:, 1:4], knn=dict(K=20, exclude_self=True), seed=2)
    assert not wc.grad[:, [0, 4, 5]].any()


# -- c. ResGCN-28 layer: EdgeConv at N = 4096 ---------------------------------------------------------------------
def _case_c(d):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(200 + d)
    torch.manual_seed(d)
    mod = _init_params(D.DynConv2d(64, 64, 20, d, "edge", "relu", "batch"), g)
    return mod, torch.randn(2, 64, 4096, 1, generator=g)


@pytest.mark.parametrize("d,train", [(1, True), (1, False), (5, True)])
def test_resgcn_layer(d, train):
    """Train (d = 1): the tile-per-CTA tensor-core kNN kernel builds nbr.  Eval runs under both kNN routings:
    'tc' (knn_tc4, the several-tiles-per-CTA kernel, which the fused forward admits in eval) and 'tc1' (one
    tile per CTA).  d = 5 (K 100): slab path.  N = 4096: eight KCH chunks; the near-tie mask is exercised."""
    from deep_gcns_torch_b200 import _native
    mod, x = _case_c(d)
    mod = mod.cuda().train(train)
    xc = x.cuda().requires_grad_(True)
    for path in (("auto",) if train else ("tc", "tc1")):
        _native.set_knn_path(path)
        try:
            ei = _fused_graph(mod, xc.detach())
            xc.grad = None
            _check("c-d%d-%s-%s" % (d, "train" if train else "eval", path), lambda: mod(xc), x, ei, mod.gconv,
                   "edge", "relu", "batch", train, lambda: xc.grad, knn=dict(K=20 * d, dilation=d), seed=d)
        finally:
            _native.set_knn_path("auto")


# -- d. tiling and alignment ------------------------------------------------------------------------------------
def _case_d(conv):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(300 if conv == "edge" else 301)
    torch.manual_seed(3)
    if conv == "edge":
        mod = _init_params(D.DynConv2d(130, 96, 9, 1, "edge", "prelu", "batch"), g, slope=-0.3)
        return mod, torch.randn(2, 130, 1030, 1, generator=g)
    mod = _init_params(D.DynConv2d(160, 72, 9, 1, "mr", "relu", "batch"), g)
    return mod, torch.randn(2, 160, 600, 1, generator=g)


@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_tiling_and_alignment(conv):
    """EdgeConv C_in 130 -> 96 (M = 2 C_out = 192 and C_in > 128: two tiles in both GEMMs; ci % 4 != 0),
    N = 1030 (three KCH chunks, the last one 6 points), PReLU slope -0.3, eval BN with negative gammas (the
    min branch of the arg-max).  MRConv C_in 160 -> 72 at N = 600 in training (2 C_in = 320: three tiles)."""
    train = conv == "mr"
    act = "prelu" if conv == "edge" else "relu"
    mod, x = _case_d(conv)
    mod = mod.cuda().train(train)
    xc = x.cuda().requires_grad_(True)
    ei = _fused_graph(mod, xc.detach())
    _check("d-" + conv, lambda: mod(xc), x, ei, mod.gconv, conv, act, "batch", train, lambda: xc.grad,
           knn=dict(K=9), seed=4)


# -- e. static graph with arbitrary centres ---------------------------------------------------------------------
def _case_e(conv):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(400 if conv == "edge" else 401)
    torch.manual_seed(4)
    mod = _init_params(D.GraphConv2d(16, 24, conv, "leakyrelu", "batch"), g)
    x = torch.randn(2, 16, 700, 1, generator=g)
    ei = torch.randint(0, 700, (2, 2, 700, 9), generator=g)      # edge_index[1] random, not arange
    return mod, x, ei


@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_arbitrary_centres(conv):
    """edge_index[1] != arange: the centre branch of edge_of (EdgeConv, train BN) and mr_gather_arg_kernel
    (MRConv, eval BN)."""
    train = conv == "edge"
    mod, x, ei = _case_e(conv)
    mod = mod.cuda().train(train)
    xc = x.cuda().requires_grad_(True)
    eic = ei.cuda()
    _check("e-" + conv, lambda: mod(xc, eic), x, ei, mod.gconv, conv, "leakyrelu", "batch", train,
           lambda: xc.grad, seed=5)


# -- f. stochastic dilation in training ---------------------------------------------------------------------------
def test_stochastic_dilation_training():
    """K = 72 slab path with an explicit column list written into nbr.  The columns are reproduced with
    torch.manual_seed, as the module draws them (one rand(1), then randperm(K)); the oracle graph is the full
    sorted K list at those columns."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(500)
    torch.manual_seed(5)
    mod = D.DynConv2d(32, 32, 9, 8, "edge", stochastic=True, epsilon=1.0).cuda().train()
    x = torch.randn(2, 32, 512, 1, generator=g)
    xc = x.cuda().requires_grad_(True)
    torch.manual_seed(11)
    cols = od.dilation_columns(9, 8, True, 1.0, True).tolist()
    assert cols != list(range(0, 72, 8))
    ei = _fused_graph(mod, xc.detach(), cols=cols)

    def run():
        torch.manual_seed(11)
        return mod(xc)
    _check("f-stochastic", run, x, ei, mod.gconv, "edge", "relu", None, True, lambda: xc.grad,
           knn=dict(K=72, cols=cols), seed=6)


# -- g. blocks in training ----------------------------------------------------------------------------------------
def _case_g(kind):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    g = torch.Generator().manual_seed(600 if kind == "res" else 601)
    torch.manual_seed(6)
    if kind == "res":
        blk = D.ResDynBlock2d(64, 20, 2, "edge", "relu", "batch", res_scale=0.7)
    else:
        blk = D.DenseDynBlock2d(64, 32, 20, 1, "mr", "relu", "batch")
    return _init_params(blk, g), torch.randn(2, 64, 1024, 1, generator=g)


@pytest.mark.parametrize("kind", ["res", "dense"])
def test_blocks_training(kind):
    """grad x through the body plus the skip connection: body(x) + x * 0.7 (ResDynBlock2d, EdgeConv, d = 2) and
    cat(x, body(x)) (DenseDynBlock2d, MRConv)."""
    blk, x = _case_g(kind)
    blk = blk.cuda().train()
    xc = x.cuda().requires_grad_(True)
    ei = _fused_graph(blk.body, xc.detach())
    conv, d = ("edge", 2) if kind == "res" else ("mr", 1)
    _check("g-" + kind, lambda: blk(xc), x, ei, blk.body.gconv, conv, "relu", "batch", True, lambda: xc.grad,
           knn=dict(K=20 * d, dilation=d), skip=0.7 if kind == "res" else "cat", seed=7)
