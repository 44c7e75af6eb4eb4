"""Train-mode BatchNorm batch statistics of the dense graph convolutions against fp64, on channels whose mean is
large compared with their spread (r = |mean| / std up to 1000), a constant channel and a channel whose variance is
close to eps.  Every writer of the statistics partials is reached (the kernel names are checked with torch.profiler
in each case):

- graph_gather_kernel (static EdgeConv, through edge_index and through nbr; un-centred input coordinates),
- cta_epilogue of knn_small_kernel (fp32 kNN, generic consumer: c_out = 24, N % 8 != 0; c_out = 256, which has no
  tensor-core route in train mode),
- cta_epilogue_wide<..., TRAIN = true> of knn_tc_kernel (c_out 64 / 128, N % 8 == 0; B = 1, N = 128, K = 40, whose
  partial count is 1 CTA + the completion kernel's 132 rows),
- the extra rows of knn_exact_rows_kernel (a cloud of repeated points, whose queries the pre-filter cannot certify),
- row_consume of the slab path (K = 60),
- mr_node_kernel (MRConv, static and dynamic),
- the headline shape B = 16, N = 4096, k = 20, c_out = 64 (statistics only).

The reference is taken in fp64 on the graph the kernel selected: the batch mean and biased variance of the
activations over the B*N*k edges (EdgeConv) or B*N nodes (MRConv) the kernel normalises, with the activations
rounded to fp32 where the kernel rounds them (_activations64); the outputs are checked against oracle.dense in fp64.  The synced-statistics
path (dgcn_bn_sync) runs on one GPU with torch.distributed.all_reduce replaced by the one-rank identity."""
import copy

import pytest
import torch

import backward_util as bu
from oracle import dense as od

pytestmark = pytest.mark.gpu

VAR_REL = 1e-5
MEAN_REL, MEAN_STD = 1e-6, 1e-5
CONST = 3.7


def _params(ci, co, act, seed, offset=False):
    """BasicConv([2 ci, co]) tensors (fp32, CPU).  Channel 0 is constant (weight 0, bias 3.7), channel 1 has
    mean 1.3 and std 3e-3 (variance ~ eps), the others cycle through r = 1, 10, 100, 1000 with means in [1, 4]
    (either sign with act 'none').  About half of the BatchNorm scales are negative (EdgeConv's min routing).
    offset: plain random weights and no bias (the input carries the large mean)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(co, 2 * ci, generator=g)
    w /= w.norm(dim=1, keepdim=True)                  # pre-activation std ~ 1 on centred unit-variance features
    b = torch.zeros(co)
    if not offset:
        r = torch.tensor([1.0, 10.0, 100.0, 1000.0])[torch.arange(co) % 4]
        mu = 1.0 + 3.0 * torch.rand(co, generator=g)
        if act == "none":
            mu *= torch.where(torch.rand(co, generator=g) < 0.5, -1.0, 1.0)
        w *= (mu.abs() / r)[:, None]
        b = mu
        w[1] *= 3e-3 / float(w[1].norm())
        b[1] = 1.3
        w[0] = 0.0
        b[0] = CONST
    gamma = (0.5 + torch.rand(co, generator=g)) * torch.where(torch.rand(co, generator=g) < 0.5, -1.0, 1.0)
    beta = 0.2 * torch.randn(co, generator=g)
    return w, b, gamma, beta


def _conv_params(w, b, gamma, beta, act, sync_group=None):
    from deep_gcns_torch_b200 import _native
    return _native.ConvParams(w.cuda(), b.cuda(), act=act, norm=_native.NORM_BATCH_TRAIN, bn_weight=gamma.cuda(),
                              bn_bias=beta.cuda(), sync_group=sync_group)


def _p64(w, b, gamma, beta, dev):
    d = lambda t: t.to(dev, torch.float64)
    co = w.shape[0]
    return {"weight": d(w).view(co, -1, 1, 1), "bias": d(b),
            "norm": {"weight": d(gamma), "bias": d(beta), "running_mean": None, "running_var": None}}


def _activations64(x, ei, p, conv, act):
    """The activations at the positions the kernel normalises ((B, Co, N, k) EdgeConv, (B, Co, N, 1) MRConv), as
    the kernel rounds them: EdgeConv's per-node rows P = (W1 - W2) x + b and Q = W2 x are exact products rounded
    once to fp32 (the packed W1 - W2 rounded as the kernel packs it), a = act(P_i + Q_j) in fp32; MRConv's
    pre-activation is rounded once to fp32.  The statistics of these values are then taken in fp64.  (Against
    unrounded fp64 activations the batch variance would also carry the sample covariance of the per-node rounding
    with the data, ~ r * 2^-24 / sqrt(nodes) - 1e-5 at r = 1000 on 128 nodes - which no statistics scheme removes.)"""
    xd = x.double()
    w = p["weight"][:, :, 0, 0]
    if conv == "edge":
        C = x.shape[1]
        w1, w2 = w[:, :C].float(), w[:, C:].float()
        wk = (w1 - w2).double()
        P = (torch.einsum("oc,bcn->bon", wk, xd[..., 0]) + p["bias"].view(1, -1, 1)).float()
        Q = torch.einsum("oc,bcn->bon", w2.double(), xd[..., 0]).float()
        Pi = od.batched_index_select(P.unsqueeze(-1), ei[1])
        Qj = od.batched_index_select(Q.unsqueeze(-1), ei[0])
        return od.activation(Pi + Qj, act).double()
    xi = od.batched_index_select(xd, ei[1])
    xj = od.batched_index_select(xd, ei[0])
    feat = torch.cat([xd, (xj - xi).max(-1, keepdim=True)[0]], 1)
    z = torch.einsum("oc,bcnk->bonk", w, feat) + p["bias"].view(1, -1, 1, 1)
    return od.activation(z.float(), act).double()


def _edge_index(nbr):
    B, N, k = nbr.shape
    i = torch.arange(N, device=nbr.device).view(1, N, 1).expand(B, N, k)
    return torch.stack((nbr.long(), i))


def _assert_stats(mean, var, a64, const_channel=True, what=""):
    dims = (0, 2, 3)
    m64 = a64.mean(dims)
    v64 = a64.var(dims, unbiased=False)
    mean, var = mean.double(), var.double()
    lo = 1 if const_channel else 0
    err_v = ((var - v64).abs() / v64.clamp_min(1e-300))[lo:]
    # VAR_REL up to r = |mean| / std = 1000; the conditioning of a channel is set through its weights, so its actual
    # r can come out above 1000, where the bound grows like the fp32 rounding of the partial means (linearly in r)
    r = (m64.abs() / v64.sqrt().clamp_min(1e-300))[lo:]
    bad = (var - v64).abs()[lo:] > VAR_REL * v64[lo:] * (r / 1000).clamp_min(1.0)
    assert not bool(bad.any()), "%s batch variance: %d channels off, worst relative error %.3e at channel %d" % (
        what, int(bad.sum()), float(err_v.max()), int(err_v.argmax()) + lo)
    mbad = (mean - m64).abs() > MEAN_REL * m64.abs() + MEAN_STD * v64.sqrt()
    assert not bool(mbad[lo:].any()), "%s batch mean: %d channels off, worst %s" % (
        what, int(mbad[lo:].sum()), float(((mean - m64).abs() / v64.sqrt().clamp_min(1e-300))[lo:].max()))
    if const_channel:
        assert float(var[0]) == 0.0, "%s constant channel: batch variance %r" % (what, float(var[0]))
        assert float(mean[0]) == float(torch.tensor(CONST, dtype=torch.float32)), \
            "%s constant channel: batch mean %r" % (what, float(mean[0]))
    return float(err_v.max())


def _kernel_names(fn):
    return bu.kernel_names(fn)


# name: conv, kind (static edge_index / static nbr / dyn), knn path, B, C, N, k, dilation, c_out, act, writer kernel
CASES = {
    "gather-edge_index": ("edge", "edge_index", None, 2, 32, 1024, 20, 1, 64, "relu", "graph_gather_kernel"),
    "gather-nbr": ("edge", "nbr", None, 2, 16, 1000, 16, 1, 40, "none", "graph_gather_kernel"),
    "ffma-generic-c24": ("edge", "dyn", "ffma", 2, 16, 1000, 9, 1, 24, "relu", "knn_small_kernel"),
    "tc1-wide-c64": ("edge", "dyn", "tc1", 1, 32, 512, 9, 1, 64, "relu", "knn_tc_kernel"),
    "tc1-wide-c128": ("edge", "dyn", "tc1", 2, 32, 1024, 16, 1, 128, "none", "knn_tc_kernel"),
    "tc1-clustered": ("edge", "dyn", "tc1", 3, 32, 512, 9, 1, 64, "relu", "knn_exact_rows_kernel"),
    "slab-k20-d3": ("edge", "dyn", None, 2, 32, 1024, 20, 3, 32, "relu", "select_rows"),
    "c256-no-tc": ("edge", "dyn", None, 1, 32, 512, 9, 1, 256, "none", "knn_small_kernel"),
    "B1-N128-K40": ("edge", "dyn", None, 1, 32, 128, 40, 1, 64, "relu", "knn_tc_kernel"),
    "mr-static": ("mr", "edge_index", None, 2, 32, 1000, 16, 1, 48, "relu", "mr_node_kernel"),
    "mr-dyn": ("mr", "dyn", None, 2, 32, 1024, 16, 1, 64, "none", "mr_node_kernel"),
    "headline-B16-N4096": ("edge", "dyn", None, 16, 64, 4096, 20, 1, 64, "relu", "knn_tc_kernel"),
}


def _input(name, B, C, N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, N, 1, generator=g)
    if name == "tc1-clustered":       # cloud 0: 64 points, each 8 times - the pre-filter cannot certify exact ties
        x[0] = x[0, :, :64].repeat(1, N // 64, 1)
    return x.cuda()


def _static_graph(B, N, k, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.stack((torch.randint(0, N, (B, N, k), generator=g), torch.randint(0, N, (B, N, k), generator=g)))


def _forward(name, x, prm, sync=False):
    """Runs the case's forward with ConvParams prm; returns (out, edge_index the kernel used, kernel names)."""
    from deep_gcns_torch_b200 import _native
    conv, kind, path, B, C, N, k, d, co, act, writer = CASES[name]
    if kind == "dyn":
        if path:
            _native.set_knn_path(path)
        try:
            (out, nbr), names = _kernel_names(lambda: _native.dyn_conv_forward(conv, x, prm, k, d, want_nbr=True))
        finally:
            _native.set_knn_path("auto")
        return out, _edge_index(nbr), names
    ei = _static_graph(B, N, k, 11).cuda()
    if kind == "edge_index":
        out, names = _kernel_names(lambda: _native.graph_conv_forward(conv, x, prm, edge_index=ei))
        return out, ei, names
    nbr = ei[0].int().contiguous()
    out, names = _kernel_names(lambda: _native.graph_conv_forward(conv, x, prm, nbr=nbr))
    return out, _edge_index(nbr), names


@pytest.mark.parametrize("name", list(CASES))
def test_batch_stats_against_fp64(name):
    from deep_gcns_torch_b200 import _native
    conv, kind, path, B, C, N, k, d, co, act, writer = CASES[name]
    x = _input(name, B, C, N, seed=len(name))
    w, b, gamma, beta = _params(C, co, act, seed=co + N)
    prm = _conv_params(w, b, gamma, beta, act)
    if name == "tc1-clustered":
        _native.tc_certification(True)
        try:
            _native.tc_certification_read()
            out, ei, names = _forward(name, x, prm)
            failed, queries = _native.tc_certification_read()
        finally:
            _native.tc_certification(False)
        assert 0 < failed < queries, (failed, queries)
    else:
        out, ei, names = _forward(name, x, prm)
    assert any(writer in n for n in names), (writer, sorted(names))
    if path == "tc1" or name.startswith("B1") or name.startswith("headline"):
        assert not any("knn_tc4_kernel" in n for n in names)
    p = _p64(w, b, gamma, beta, x.device)
    a64 = _activations64(x, ei, p, conv, act)
    worst = _assert_stats(prm.batch_mean, prm.batch_var, a64, what=name)
    if name.startswith("headline"):
        print("%s: worst relative variance error %.2e" % (name, worst))
        return
    del a64
    ref = od.graph_conv(x.double(), ei, p, conv, act, "batch", training=True)
    bu.assert_grads_close(name + " output", out, ref)
    # the constant channel normalises to beta: fmaf(s, 3.7, t) with t = beta - 3.7 s
    s = abs(float(gamma[0])) / (1e-5 ** 0.5)
    tol = 8 * float(torch.finfo(torch.float32).eps) * s * CONST
    assert float((out[:, 0].double() - float(beta[0])).abs().max()) <= tol
    print("%s: worst relative variance error %.2e" % (name, worst))


def test_uncentred_coordinates_static_graph():
    """The input itself is offset (x + 100 on every other channel) and the graph is the oracle's kNN of the centred
    cloud: EdgeConv's x_i half carries the large mean into every channel."""
    from deep_gcns_torch_b200 import _native
    B, C, N, k, co = 2, 16, 1024, 16, 64
    x0 = torch.randn(B, C, N, 1, generator=torch.Generator().manual_seed(3))
    ei = od.knn_matrix(x0, k)
    x = x0.clone()
    x[:, ::2] += 100.0
    x = x.cuda()
    w, b, gamma, beta = _params(C, co, "none", seed=9, offset=True)
    prm = _conv_params(w, b, gamma, beta, "none")
    ei = ei.cuda()
    out, names = _kernel_names(lambda: _native.graph_conv_forward("edge", x, prm, edge_index=ei))
    assert any("graph_gather_kernel" in n for n in names)
    p = _p64(w, b, gamma, beta, x.device)
    a64 = _activations64(x, ei, p, "edge", "none")
    r = (a64.mean((0, 2, 3)).abs() / a64.std((0, 2, 3))).max()
    assert float(r) > 30, float(r)
    _assert_stats(prm.batch_mean, prm.batch_var, a64, const_channel=False, what="uncentred")
    bu.assert_grads_close("uncentred output", out, od.graph_conv(x.double(), ei, p, "edge", "none", "batch", True))


@pytest.mark.parametrize("name", ["gather-edge_index", "tc1-wide-c64", "slab-k20-d3", "mr-static", "mr-dyn"])
def test_synced_statistics_one_rank(name, monkeypatch):
    """dgcn_bn_sync on one rank: bn_merge_kernel forms [sum a | sum a^2 | count] in fp64, the all-reduce is the
    identity, bn_finalize_moments_kernel recovers the statistics; the backward runs moments_over_count_kernel."""
    import torch.distributed as dist
    from deep_gcns_torch_b200 import _native
    monkeypatch.setattr(dist, "all_reduce", lambda *a, **kw: None)
    conv, kind, path, B, C, N, k, d, co, act, writer = CASES[name]
    x = _input(name, B, C, N, seed=len(name))
    w, b, gamma, beta = _params(C, co, act, seed=co + N)
    prm = _conv_params(w, b, gamma, beta, act, sync_group=object())
    out, ei, _ = _forward(name, x, prm)
    a64 = _activations64(x, ei, _p64(w, b, gamma, beta, x.device), conv, act)
    _assert_stats(prm.batch_mean, prm.batch_var, a64, what=name + " synced")
    n = a64[:, 0].numel()
    m = prm.moments.cpu()
    assert float(m[2 * co]) == n
    # the same statistics as the local path
    loc = _conv_params(w, b, gamma, beta, act)
    out_l, ei_l, _ = _forward(name, x, loc)
    assert torch.equal(ei_l, ei)
    torch.testing.assert_close(prm.batch_mean, loc.batch_mean, rtol=1e-6, atol=0)
    torch.testing.assert_close(prm.batch_var, loc.batch_var, rtol=1e-6, atol=0)
    torch.testing.assert_close(out, out_l, rtol=1e-5, atol=1e-5 * float(out_l.abs().max()))
    go = torch.randn(out.shape, generator=torch.Generator().manual_seed(4)).cuda()
    g_s = _native.graph_conv_backward(conv, x, prm, go, edge_index=ei)
    g_l = _native.graph_conv_backward(conv, x, loc, go, edge_index=ei)
    for key in ("x", "weight", "bn_weight", "bn_bias"):     # (the bias gradient of a batch-normalised conv is 0)
        torch.testing.assert_close(g_s[key], g_l[key], rtol=1e-4, atol=1e-5 * float(g_l[key].abs().max()), msg=key)


@pytest.mark.parametrize("conv", ["edge", "mr"])
def test_module_running_stats(conv):
    """DynConv2d in training mode (momentum 0.1, running statistics from zero): the running mean and the running
    (unbiased) variance against the fp64 update, and the output against fp64."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B, C, N, k, co, act = 2, 32, 1024, 16, 64, "relu"
    torch.manual_seed(0)
    m = D.DynConv2d(C, co, k, 1, conv, act, "batch")
    w, b, gamma, beta = _params(C, co, act, seed=5)
    nn_ = m.gconv.nn
    nn_[0].weight.data = w.view(co, 2 * C, 1, 1).clone()
    nn_[0].bias.data = b.clone()
    nn_[2].weight.data, nn_[2].bias.data = gamma.clone(), beta.clone()
    nn_[2].running_mean.zero_()
    nn_[2].running_var.zero_()
    m = m.cuda().train()
    x = _input("module", B, C, N, seed=21).requires_grad_(True)
    with torch.no_grad():
        ei = copy.deepcopy(m).dilated_knn_graph(x.detach())
    y = m(x)
    a64 = _activations64(x.detach(), ei, _p64(w, b, gamma, beta, x.device), conv, act)
    cnt = a64[:, 0].numel()
    m64, v64 = a64.mean((0, 2, 3)), a64.var((0, 2, 3), unbiased=False)
    rm, rv = nn_[2].running_mean.double(), nn_[2].running_var.double()
    rm_ref, rv_ref = 0.1 * m64, 0.1 * v64 * cnt / (cnt - 1)
    assert bool(((rm - rm_ref).abs() <= MEAN_REL * rm_ref.abs() + 0.1 * MEAN_STD * v64.sqrt()).all())
    assert bool(((rv - rv_ref).abs()[1:] <= 2 * VAR_REL * rv_ref[1:]).all()), float(
        ((rv - rv_ref).abs() / rv_ref.clamp_min(1e-300))[1:].max())
    assert float(rv[0]) == 0.0
    p = od.params_from_module(nn_, dtype=torch.float64)
    bu.assert_grads_close("module output", y, od.graph_conv(x.detach().double(), ei, p, conv, act, "batch", True))
