"""Sparse-layout EdgeConv (csrc/sparse_edge.cu, EdgConv) against fp64 autograd of sparse_edge_util.edge_conv on the
same edge_index, at the shapes where its kernels change behaviour, at the sem_seg_sparse layer's full size, and for
the module variants.

Every case checks the output and every gradient the layer has (x, W, b, the PReLU weight, gamma, beta), and in
batch-statistics mode also the batch mean / variance the kernel normalised with and the running statistics after
the step.  Each case prints its worst |got - ref| / max|ref| per tensor and, where there is one, the masked fraction.

a. Exact-arithmetic grid (sparse_edge_util.exact_fixture / EXACT_SHAPES): integer features with OFFSET channels,
   weights in sixteenths, explicit graphs.  No mask: eval outputs bit-equal, gradients at 1e-6 (leaky relu 1e-5);
   train at the default bounds, with batch statistics to 1e-6 (|mean| + std) and 1e-5 var.
b. The sem_seg_sparse layers at N = 16 x 4096 (E = 1,048,576), and a ResDynBlock on the slab kNN route.
c. Module variants at N = 1030.
b and c draw random inputs and zero the upstream gradient at the near-ties of the max (edge_tie_mask).

sparse_edge.cu paths (SPE_ROWS = 32 rows per CTA, channels and source slots in chunks of 32; common.cuh: TILE = 128,
KCH = 512), and the case that reaches each:
  wgrad_kernel split-K over KCH chunks, partial last one     n543-co64 (2, last 31 nodes), n1313-co65 (3, last 289),
                                                             n1030-ci130-co129 (3, last 6), c (3, last 6); full
                                                             chunks only: n2048-ci128 (4), b (128)
  M = 2 C_out > TILE: a second column tile of node_pq_kernel   n1313-co65 (M 130), n1030-ci130-co129 (M 258: three),
  and wgrad_kernel                                           b (M 128: exactly one)
  C_in > TILE: a second grad_x output tile (tile_gemm_kernel)  n1030-ci130-co129 (C_in 130)
  vec = 0 (N % 4 != 0: scalar loads of xt and dpqt)          n33-co2, n97-co1, n159-co32, n543-co64, n1313-co65,
                                                             n1030-ci130-co129, c
  C_in % 4 != 0                                              n33-co2 (3), n97-co1 (5), n159-co32 (7), n543-co64 (9),
                                                             n1030-ci130-co129 (130), b head (9), c slice (3)
  N % 32 in {1, 31}: a last CTA of 1 / 31 rows               n33-co2, n97-co1, n1313-co65 (1); n159-co32, n543-co64 (31)
  rows of 0 / 1 / 31 / 32 / 33 / 63 / 64 / 65 edges           every exact shape (sparse_edge_util.ROW_LENGTHS)
  rows of > 1024 edges (32-edge source chunks: 35)           n159-co32, n1313-co65, n1030-ci130-co129 (HUB = 1100)
  C_out (lanes over 32-channel chunks)                       1: n97-co1; 2: n33-co2; 32: n159-co32; 33: n256-co33;
                                                             64: n543-co64; 65: n1313-co65; 129: n1030-ci130-co129
  grad_x == nullptr (need_x False)                           b head, c no-grad
  bias=False / BatchNorm1d(affine=False) / no running stats  c
The exact grid runs relu in eval and train on every shape, and leaky relu and PReLU (+0.25, -0.5) on the two largest.
"""
import gc

import pytest
import torch
from torch import nn

import backward_util as bu
import sparse_edge_util as seu

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
TIE_REL, KINK_REL = 1e-4, 1e-5      # near-tie / kink mask of the random cases, as test_sparse_edgeconv_gpu.py
MAX_MASKED = 2e-3
MEAN_REL, VAR_REL = 1e-6, 1e-5      # batch statistics: |dmean| <= MEAN_REL (|mean| + std), |dvar| <= VAR_REL var


def _bn(mod):
    return next((m for m in mod.nn if isinstance(m, nn.BatchNorm1d)), None)


def _oracle(mod, x, ei, gout, batch_stats):
    """fp64 autograd of the restatement on x's device: (y, {gradient name: tensor}, (batch mean, biased var))."""
    dev = x.device
    p = seu.edge_conv_params(mod.nn, torch.float64, dev)
    leaves = {"x": x.detach().double().requires_grad_(True), "weight": p["weight"].requires_grad_(True)}
    if "bias" in p:
        leaves["bias"] = p["bias"].requires_grad_(True)
    if "slope" in p:
        leaves["prelu"] = p["slope"].requires_grad_(True)
    if "norm" in p and p["norm"]["weight"] is not None:
        leaves["bn_weight"] = p["norm"]["weight"].requires_grad_(True)
        leaves["bn_bias"] = p["norm"]["bias"].requires_grad_(True)
    zs = []
    y, stats = seu.edge_conv(leaves["x"], ei, p, seu.mlp_act(mod.nn), batch_stats, return_stats=True, retain_z=zs)
    (y * gout.double()).sum().backward()
    grads = {k: v.grad for k, v in leaves.items()}
    if batch_stats:
        grads["weight_terms"] = _weight_terms(zs[0].grad, x.detach().double(), ei)
    return y.detach(), grads, stats


def _weight_terms(dz, x, ei):
    """(C_out, 2 C_in): the size of the terms the kernel sums into each weight gradient, sum_n |dP_n| |x_n| for W1
    and that plus sum_n |dQ_n| |x_n| for W2 (dW1 = dA, dW2 = dB - dA with dA = dP^T x, dB = dQ^T x; dP_n, dQ_n: dz
    summed over the edges into / out of node n)."""
    n = x.shape[0]
    dp = torch.zeros(n, dz.shape[1], dtype=dz.dtype, device=dz.device).index_add_(0, ei[1].long(), dz)
    dq = torch.zeros_like(dp).index_add_(0, ei[0].long(), dz)
    a, b = dp.abs().T @ x.abs(), dq.abs().T @ x.abs()
    return torch.cat((a, a + b), 1)


def _module_grads(mod, grad_x):
    lin = mod.nn[0]
    g = {"x": grad_x() if grad_x is not None else None, "weight": lin.weight.grad,
         "bias": None if lin.bias is None else lin.bias.grad}
    for m in list(mod.nn)[1:]:
        if isinstance(m, nn.PReLU):
            g["prelu"] = m.weight.grad
        if isinstance(m, nn.BatchNorm1d) and m.weight is not None:
            g["bn_weight"], g["bn_bias"] = m.weight.grad, m.bias.grad
    return g


def _check(tag, mod, x, ei, gout, exact=False, mask=None, x_in=None, grad_x=None, steps=1):
    """Forward and backward of sum(y * gout) through `mod` on the GPU, against _oracle.  x: the values of the input;
    x_in: the tensor given to the module (default: a requires-grad copy of x) and grad_x() its gradient (None: x_in
    does not require grad).  exact: a sparse_edge_util.exact_fixture case (no mask; eval outputs bit-equal and
    gradients at 1e-6).  mask: (N, C_out) entries whose upstream gradient is zeroed on both sides.  steps: forward /
    backward steps, with the running statistics checked after each."""
    bn = _bn(mod)
    batch_stats = bn is not None and (mod.training or bn.running_mean is None)
    act = seu.mlp_act(mod.nn)
    if mask is not None:
        gout = gout.masked_fill(mask, 0.0)
    E = ei.shape[1]
    for step in range(steps):
        tracks = batch_stats and bn.track_running_stats
        if tracks:
            old = (bn.running_mean.double().clone(), bn.running_var.double().clone())
        ref_y, ref, stats = _oracle(mod, x, ei, gout, batch_stats)
        terms = ref.pop("weight_terms", None)
        mod.zero_grad(set_to_none=True)
        xi, gx = x_in, grad_x
        if xi is None:
            xi = x.clone().requires_grad_(True)
            gx = lambda: xi.grad
        y = mod(xi, ei)
        prm = y.grad_fn.prm
        (y * gout).sum().backward()
        got = _module_grads(mod, gx)
        name = "%s step %d" % (tag, step) if steps > 1 else tag
        ratios = {}
        if exact and not batch_stats and act != "leakyrelu":
            assert torch.equal(y.detach(), ref_y.float()), name + ": output not bit-equal to fp64"
            ratios["y"] = 0.0
        elif exact and not batch_stats:    # leaky relu's slope 0.2 is not dyadic: u * 0.2 rounds in fp32
            torch.testing.assert_close(y.detach().double(), ref_y, rtol=1e-6, atol=0.0)
            ratios["y"] = float((y.detach().double() - ref_y).abs().max() / ref_y.abs().max().clamp_min(1e-30))
        elif exact:
            ratios["y"] = bu.assert_grads_close(name + " y", y, ref_y)
        else:
            torch.testing.assert_close(y.detach().double(), ref_y, rtol=RTOL, atol=ATOL, msg=lambda s: name + ": " + s)
            ratios["y"] = float((y.detach().double() - ref_y).abs().max() / ref_y.abs().max().clamp_min(1e-30))
        need_x = x_in is None or grad_x is not None
        assert set(k for k, v in got.items() if v is not None) == set(ref) - (set() if need_x else {"x"})
        tol = (1e-5 if act == "leakyrelu" else 1e-6) if exact and not batch_stats else None
        for key in ref:
            if got.get(key) is None:
                continue
            # BatchNorm on batch statistics removes the Linear's bias: its gradient is a sum of terms that cancel to
            # 0, and gets an absolute tolerance on the scale of the weight's gradient
            floor = float(ref["weight"].abs().max()) if batch_stats and key == "bias" else 0.0
            kw = dict(atol_frac=tol, rtol=tol) if tol is not None else {}
            if key == "weight" and exact and batch_stats:
                # likewise the part OFFSET * sum_n dP_n of an offset input channel's weight gradient: those columns
                # also get 2^-20 of the size of the terms being summed (the fp32 sum's rounding), as the dense tests
                # give the cancelling bias gradient
                ci = x.shape[1]
                cols = seu.offset_channels(ci) + [ci + c for c in seu.offset_channels(ci)]
                slack = torch.zeros_like(terms)
                slack[:, cols] = 2.0 ** -20 * terms[:, cols]
                kw["slack"] = slack
            ratios[key] = bu.assert_grads_close("%s %s" % (name, key), got[key], ref[key], floor=floor, **kw)
        extra = ""
        if batch_stats:
            mean, var = stats
            std = var.sqrt()
            dm = (prm.batch_mean.double() - mean).abs()
            dv = (prm.batch_var.double() - var).abs()
            assert bool((dm <= MEAN_REL * (mean.abs() + std)).all()), (name, float((dm / (mean.abs() + std)).max()))
            assert bool((dv <= VAR_REL * var).all()), (name, float((dv / var.clamp_min(1e-300)).max()),
                                                       int((dv / var.clamp_min(1e-300)).argmax()))
            extra = " batch mean %.2e var %.2e (|mean|/std up to %.0f)" % (
                float((dm / (mean.abs() + std).clamp_min(1e-300)).max()), float((dv / var.clamp_min(1e-300)).max()),
                float((mean.abs() / std.clamp_min(1e-300)).masked_fill(var == 0, 0).max()))
            if exact and mod.nn[0].weight.shape[0] >= 2:
                assert float(prm.batch_var[1]) == 0.0, name + ": the dead channel's batch variance is not 0"
            if tracks:
                mom = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked)
                rm = (1 - mom) * old[0] + mom * mean
                rv = (1 - mom) * old[1] + mom * var * (E / (E - 1))
                # the batch statistics' own bounds, carried by mom <= 1, plus the update's fp32 rounding
                assert bool(((bn.running_mean.double() - rm).abs() <=
                             MEAN_REL * (mean.abs() + std) + 1e-6 * rm.abs()).all()), name + ": running mean"
                assert bool(((bn.running_var.double() - rv).abs() <= (VAR_REL + 1e-6) * rv).all()), \
                    name + ": running var"
            elif bn.running_mean is None:
                assert bn.running_var is None and bn.num_batches_tracked is None
        print("sparse edgeconv %s: worst |got - ref| / max|ref| %s;%s masked fraction %s" % (
            name, " ".join("%s=%.2e" % kv for kv in ratios.items()), extra,
            "-" if mask is None else "%.2e" % float(mask.double().mean())))
        del ref_y, ref, stats, y
    gc.collect()
    torch.cuda.empty_cache()


# -- a. exact-arithmetic grid -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,act,slope,train", seu.exact_cases(),
                         ids=["%s-%s%s-%s" % (n, a, "" if s is None else s, "train" if t else "eval")
                              for n, a, s, t in seu.exact_cases()])
def test_exact_grid(name, act, slope, train):
    N, ci, co, hub, seed = seu.EXACT_SHAPES[name]
    mod, x, ei, gout = seu.exact_fixture(N, ci, co, act, slope, train, seed, hub)
    mod = mod.cuda()
    x, ei, gout = x.cuda(), ei.cuda(), gout.cuda()
    deg = torch.bincount(ei[1], minlength=N).cpu()
    for n in seu.ROW_LENGTHS + ((seu.HUB,) if hub else ()):
        assert int((deg == n).sum()) >= 1, n
    if train:   # the preconditions (tests/test_sparse_edgeconv_cpu.py checks them without a GPU too)
        assert int(seu.edge_tie_mask(mod.nn, x, ei, TIE_REL, KINK_REL, True, exact=True).sum()) == 0
    _check("a-%s-%s%s-%s" % (name, act, "" if slope is None else slope, "train" if train else "eval"), mod, x, ei,
           gout, exact=True)


# -- b. the sem_seg_sparse layers at full size --------------------------------------------------------------------
def _init_bn(mod, g):
    """Random BN affine parameters and running statistics (those that exist), every third gamma negative."""
    for m in mod.modules():
        if isinstance(m, nn.BatchNorm1d):
            c = m.num_features
            if m.affine:
                m.weight.data = torch.randn(c, generator=g) * 0.5 + 0.8
                m.weight.data[::3] *= -1
                m.bias.data = torch.randn(c, generator=g) * 0.2
            if m.track_running_stats:
                m.running_mean.data = torch.randn(c, generator=g) * 0.3
                m.running_var.data = torch.rand(c, generator=g) + 0.4
    return mod


def _random_case(tag, mod, x, ei, train, seed, **kw):
    mod.train(train)
    g = torch.Generator().manual_seed(seed)
    mask = seu.edge_tie_mask(mod.nn, x, ei, TIE_REL, KINK_REL, train or _bn(mod).running_mean is None)
    frac = float(mask.double().mean())
    gout = torch.randn(x.shape[0], mod.nn[0].out_features, generator=g).cuda()
    _check(tag, mod, x, ei, gout, mask=mask, **kw)
    assert frac <= MAX_MASKED, (tag, frac)


B_CLOUDS, B_POINTS, B_K = 16, 4096, 16


def _cloud_graph(g):
    """(2, B_CLOUDS * B_POINTS * B_K) int64: exactly B_K in-edges per node, sources drawn within the node's cloud,
    grouped by target (the CSR shape of a k = 16 kNN graph)."""
    N = B_CLOUDS * B_POINTS
    dst = torch.arange(N).repeat_interleave(B_K)
    src = torch.randint(0, B_POINTS, (N * B_K,), generator=g) + (dst // B_POINTS) * B_POINTS
    return torch.stack((src, dst))


@pytest.mark.parametrize("train", [True, False])
def test_sem_seg_layer_full_size(train):
    """EdgConv(64, 64, 'relu', 'batch') at N = 16 x 4096, E = 1,048,576: 2048 CTAs of batch-statistic partials,
    split-K over 128 KCH chunks, dQ atomics from every edge in train mode."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(20)
    torch.manual_seed(20)
    mod = _init_bn(S.EdgConv(64, 64, "relu", "batch"), g).cuda()
    ei = _cloud_graph(g).cuda()
    assert ei.shape[1] == 1048576
    x = torch.randn(B_CLOUDS * B_POINTS, 64, generator=g).cuda()
    _random_case("b-layer-%s" % ("train" if train else "eval"), mod, x, ei, train, seed=21)


def test_sem_seg_head_full_size():
    """GraphConv(9, 64, 'edge', 'relu', 'batch') on the kNN graph of the positions, positions and colours in [0, 1]
    (un-centred), train mode, x without requires_grad (grad_x == nullptr)."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(30)
    torch.manual_seed(30)
    head = S.GraphConv(9, 64, "edge", "relu", "batch")
    _init_bn(head, g)
    head = head.cuda()
    x = torch.rand(B_CLOUDS * B_POINTS, 9, generator=g).cuda()
    batch = torch.arange(B_CLOUDS, device="cuda").repeat_interleave(B_POINTS)
    ei = S.DilatedKnnGraph(B_K, 1)(x[:, :3], batch)
    assert ei.shape[1] == 1048576
    _random_case("b-head-train", head.gconv, x, ei, True, seed=31, x_in=x, grad_x=None)


def test_res_dyn_block_slab_route():
    """ResDynBlock(64, 16, 4, 'edge', 'relu', 'batch') on 2 x 4096 points (K = 64: the slab kNN route), train mode:
    the block's graph adjudicated per cloud against the fp64 kNN, body(x) + x * res_scale against fp64."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(40)
    torch.manual_seed(40)
    B, n, k, d = 2, 4096, 16, 4
    blk = _init_bn(S.ResDynBlock(64, k, d, "edge", "relu", "batch", res_scale=0.5), g).cuda().train()
    x = torch.randn(B * n, 64, generator=g).cuda()
    batch = torch.arange(B, device="cuda").repeat_interleave(n)
    with torch.no_grad():
        ei = blk.body.dilated_knn_graph(x, batch)
    nbr = (ei[0].view(B, n, k) - torch.arange(B, device="cuda").view(B, 1, 1) * n).cpu()
    assert torch.equal(ei[1].view(B, n, k).cpu(), torch.arange(B * n).view(B, n, 1).expand(B, n, k))
    bu.check_graph(x.view(B, n, 64).transpose(1, 2).unsqueeze(-1).cpu(), nbr, K=k * d, dilation=d)
    conv = blk.body.gconv
    mask = seu.edge_tie_mask(conv.nn, x, ei, TIE_REL, KINK_REL, True)
    gout = torch.randn(B * n, 64, generator=g).cuda().masked_fill(mask, 0.0)
    ref_y, ref, _ = _oracle(conv, x, ei, gout, True)
    del ref["weight_terms"]
    xg = x.clone().requires_grad_(True)
    blk.zero_grad(set_to_none=True)
    y, _ = blk(xg, batch, ei)
    (y * gout).sum().backward()
    ref_x = ref["x"] + gout.double() * 0.5                   # d/dx of body(x) + x * res_scale
    torch.testing.assert_close(y.detach().double(), ref_y + x.double() * 0.5, rtol=RTOL, atol=ATOL)
    ratios = {"x": bu.assert_grads_close("block x", xg.grad, ref_x)}
    got = _module_grads(conv, None)
    for key in ("weight", "bias", "bn_weight", "bn_bias"):
        floor = float(ref["weight"].abs().max()) if key == "bias" else 0.0
        ratios[key] = bu.assert_grads_close("block " + key, got[key], ref[key], floor=floor)
    frac = float(mask.double().mean())
    print("sparse edgeconv b-resdynblock: worst |got - ref| / max|ref| %s; masked fraction %.2e" % (
        " ".join("%s=%.2e" % kv for kv in ratios.items()), frac))
    assert frac <= MAX_MASKED, frac


# -- c. module variants -------------------------------------------------------------------------------------------
def _variant_inputs(seed, ci=24):
    g = torch.Generator().manual_seed(seed)
    N = 1030
    ei = torch.randint(0, N, (2, 12 * N), generator=g)
    return g, torch.randn(N, ci, generator=g), ei


@pytest.mark.parametrize("variant", ["bias_false", "affine_false", "no_running_stats_eval", "momentum_none",
                                     "x_slice", "x_no_grad"])
def test_module_variants(variant):
    """N = 1030 (three KCH chunks, the last 6 nodes; vec = 0), C 24 -> 40, random graph of 12 N edges."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    torch.manual_seed(50)
    g, x, ei = _variant_inputs(51)
    ei = ei.cuda()
    tag = "c-" + variant
    if variant == "bias_false":
        mod = _init_bn(S.EdgConv(24, 40, "relu", "batch", bias=False), g).cuda()
        assert mod.nn[0].bias is None
        _random_case(tag, mod, x.cuda(), ei, True, seed=52)
    elif variant == "affine_false":
        mod = S.EdgConv(24, 40, "leakyrelu", "batch")
        assert isinstance(mod.nn[1], nn.BatchNorm1d)
        mod.nn[1] = _init_bn(nn.BatchNorm1d(40, affine=False), g)
        _random_case(tag, mod.cuda(), x.cuda(), ei, True, seed=53)
    elif variant == "no_running_stats_eval":
        mod = S.EdgConv(24, 40, "prelu", "batch")
        assert isinstance(mod.nn[1], nn.BatchNorm1d)
        mod.nn[1] = nn.BatchNorm1d(40, track_running_stats=False)
        _init_bn(mod, g)
        _random_case(tag, mod.cuda(), x.cuda(), ei, False, seed=54)      # eval, yet batch statistics
        assert mod.nn[1].running_mean is None and mod.nn[1].running_var is None
    elif variant == "momentum_none":
        mod = _init_bn(S.EdgConv(24, 40, "relu", "batch"), g)
        mod.nn[1].momentum = None
        _random_case(tag, mod.cuda(), x.cuda(), ei, True, seed=55, steps=2)
        assert int(mod.nn[1].num_batches_tracked) == 2
    elif variant == "x_slice":
        mod = _init_bn(S.EdgConv(3, 40, "relu", "batch"), g).cuda()
        wide = torch.randn(1030, 6, generator=g).cuda().requires_grad_(True)
        xs = wide[:, 1:4]
        assert not xs.is_contiguous()
        _random_case(tag, mod, xs.detach(), ei, True, seed=56, x_in=xs, grad_x=lambda: wide.grad[:, 1:4])
        assert not wide.grad[:, [0, 4, 5]].any()
    else:
        mod = _init_bn(S.EdgConv(24, 40, "relu", "batch"), g).cuda()
        xc = x.cuda()
        _random_case(tag, mod, xc, ei, True, seed=57, x_in=xc, grad_x=None)
