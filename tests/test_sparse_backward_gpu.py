"""Gradients of the fused GENConv aggregate (dgcn_genconv_aggregate_backward) against torch
autograd through the oracle restatement of the reference forward (fp64)."""
import pytest
import torch

import backward_util as bu
from oracle import sparse as osp

pytestmark = pytest.mark.gpu

CFGS = [
    dict(aggr="softmax_sg", t=0.1),
    dict(aggr="softmax", t=0.6, learn_t=True, msg_norm=True, learn_msg_scale=True),
    dict(aggr="softmax", t=1.0),
    dict(aggr="softmax_sum", t=0.4, learn_t=True, y=0.3, learn_y=True),
    dict(aggr="power", p=2.0, learn_p=True, msg_norm=True),
    dict(aggr="power_sum", p=1.5, learn_p=True, y=-0.2, learn_y=True),
    dict(aggr="add"),
    dict(aggr="mean", msg_norm=True),
    dict(aggr="max"),
]


def _oracle_h(ref, xr, ei, N):
    """x + [MsgNorm](aggregate(message)) of the fp64 copy `ref` of a GENConv, differentiable in xr and the
    learnable scalars as the reference is."""
    scal = lambda name, d: getattr(ref, name, d)
    h = osp.genconv_pre_mlp(xr, ei, None, ref.aggr, scal("t", 1.0), scal("p", 1.0), scal("y", 0.0),
                            ref.msg_norm.msg_scale if ref.msg_norm is not None else None, ref.eps)
    if not getattr(ref, "learn_t", False) and ref.aggr in ("softmax", "softmax_sg", "softmax_sum"):
        # the reference computes the softmax weights under no_grad unless learn_t (torch_message.py:51-55)
        msg = osp.message(xr, ei, None, ref.eps)
        with torch.no_grad():
            z = msg * scal("t", 1.0)
            gmax = osp._seg_max(z, ei[1], N)
            e = (z - gmax.index_select(0, ei[1])).exp()
            w = e / osp._seg_sum(e, ei[1], N).index_select(0, ei[1])
        m = osp._seg_sum(msg * w, ei[1], N)
        if ref.aggr == "softmax_sum":
            m = torch.pow(osp.in_degree(ei[1], N, torch.float64).unsqueeze(1), torch.sigmoid(ref.y)) * m
        h = xr + (osp.msg_norm(xr, m, ref.msg_norm.msg_scale) if ref.msg_norm is not None else m)
    return h


def _grads_vs_oracle(mod, x, ei, wgt, tag):
    """Forward and backward of mod.propagate (residual on) against fp64 autograd of the oracle: output, grad x
    and the grads of the learnable scalars, elementwise (backward_util.assert_grads_close)."""
    N = x.shape[0]
    ref = __import__("copy").deepcopy(mod).double()
    xr = x.double().requires_grad_(True)
    h = _oracle_h(ref, xr, ei, N)
    (h * wgt.double()).sum().backward()
    mod = mod.cuda().train()
    xc = x.cuda().requires_grad_(True)
    scale = mod.msg_norm.msg_scale if mod.msg_norm is not None else None
    hc = mod.propagate(ei.cuda(), x=xc, msg_scale=scale, residual=True)
    torch.testing.assert_close(hc.detach().cpu(), h.detach().float(), rtol=1e-3, atol=1e-4)
    (hc * wgt.cuda()).sum().backward()
    pairs = [("x", xc.grad, xr.grad)]
    for name in ("t", "p", "y"):
        pr = getattr(ref, name, None)
        if torch.is_tensor(pr) and pr.requires_grad:
            pairs.append((name, getattr(mod, name).grad, pr.grad))
    if ref.msg_norm is not None and ref.msg_norm.msg_scale.requires_grad:
        pairs.append(("msg_scale", mod.msg_norm.msg_scale.grad, ref.msg_norm.msg_scale.grad))
    for name, got, want in pairs:
        assert bool(torch.isfinite(want).all()), name
        # a learnable scalar's gradient may be 0 up to rounding (MsgNorm is blind to the scale of the message):
        # its absolute term is then taken from 1, not from the gradient itself
        bu.assert_grads_close("%s/%s" % (tag, name), got, want, floor=0.0 if name == "x" else 1.0)


HUB_CFGS = [
    dict(aggr="softmax", t=0.6, learn_t=True),
    dict(aggr="power", p=2.0, learn_p=True, msg_norm=True),
    dict(aggr="max"),
    dict(aggr="mean", msg_norm=True),
]


def _id(cfg):
    return cfg["aggr"] + ("_lt" if cfg.get("learn_t") else "") + ("_msgnorm" if cfg.get("msg_norm") else "")


@pytest.mark.parametrize("cfg", HUB_CFGS, ids=_id)
def test_hub_row_and_zero_rows_against_oracle(cfg):
    """One destination row with 3000 in-edges (>= HUB_MIN_DEGREE): the forward aggregates it with the
    segmented hub kernels, the backward recomputes it on one warp.  x is zero at two other destination rows
    that have edges: with MsgNorm that is the |x| = 0 branch, whose gradient the reference's x.norm gives as 0."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    g = torch.Generator().manual_seed(17)
    N, C, E_hub, E_rest = 260, 128, 3000, 2000
    dst = torch.cat((torch.full((E_hub,), 5, dtype=torch.int64), torch.randint(6, N - 20, (E_rest,), generator=g)))
    ei = torch.stack((torch.randint(0, N, (E_hub + E_rest,), generator=g), dst))
    deg = torch.bincount(dst, minlength=N)
    assert int(deg[5]) >= _native.HUB_MIN_DEGREE
    hubs = csr_of(ei.cuda(), N, cache=False)[3]
    assert hubs is not None and hubs[3] > 0
    x = torch.randn(N, C, generator=g)
    zero_rows = [int(r) for r in dst[E_hub:E_hub + 2]]
    assert zero_rows[0] != zero_rows[1] and min(int(deg[r]) for r in zero_rows) > 0
    x[zero_rows] = 0
    wgt = torch.randn(N, C, generator=g)
    torch.manual_seed(1)
    mod = S.GENConv(C, C, mlp_layers=1, norm="layer", **cfg)
    if mod.msg_norm is not None:
        mod.msg_norm.msg_scale.data.fill_(0.7)
    _grads_vs_oracle(mod, x, ei, wgt, "hub-" + cfg["aggr"])


@pytest.mark.parametrize("cfg", CFGS + [dict(aggr="power", p=2.0, learn_p=True)], ids=_id)
def test_edgeless_graph_against_oracle(cfg):
    """E = 0: every row is empty.  grad x is grad_out plus the MsgNorm term; for power without MsgNorm the
    empty rows' d_p term (of the clamped 1e-7 ** (1/p)) must match fp64 autograd too."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(50)
    N, C = 50, 40
    ei = torch.zeros((2, 0), dtype=torch.int64)
    x = torch.randn(N, C, generator=g)
    wgt = torch.randn(N, C, generator=g)
    torch.manual_seed(1)
    mod = S.GENConv(C, C, mlp_layers=1, norm="layer", **cfg)
    if mod.msg_norm is not None:
        mod.msg_norm.msg_scale.data.fill_(0.7)
    _grads_vs_oracle(mod, x, ei, wgt, "edgeless-" + cfg["aggr"])


@pytest.mark.parametrize("C",[24, 48, 128, 200, 512])     # every NCH instantiation: 1, 2, 4, 8, 16
@pytest.mark.parametrize("cfg", CFGS, ids=lambda c: c["aggr"] + ("_lt" if c.get("learn_t") else ""))
def test_grads_match_autograd_of_oracle(cfg, C):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(C)
    N, E = 260, 3000
    dst = torch.randint(0, N - 20, (E,), generator=g)
    dst[:700] = 5
    ei = torch.stack((torch.randint(0, N, (E,), generator=g), dst))
    x = torch.randn(N, C, generator=g)
    wgt = torch.randn(N, C, generator=g)
    torch.manual_seed(1)
    mod = S.GENConv(C, C, mlp_layers=1, norm="layer", **cfg)
    if mod.msg_norm is not None:
        mod.msg_norm.msg_scale.data.fill_(0.7)

    # fp64 oracle with autograd
    ref = __import__("copy").deepcopy(mod).double()
    xr = x.double().requires_grad_(True)
    h = _oracle_h(ref, xr, ei, N)
    (h * wgt.double()).sum().backward()

    mod = mod.cuda().train()
    xc = x.cuda().requires_grad_(True)
    scale = mod.msg_norm.msg_scale if mod.msg_norm is not None else None
    hc = mod.propagate(ei.cuda(), x=xc, msg_scale=scale, residual=True)
    torch.testing.assert_close(hc.detach().cpu(), h.detach().float(), rtol=1e-3, atol=1e-4)
    (hc * wgt.cuda()).sum().backward()

    def check(name, got, want):
        scale_ = want.abs().max().clamp_min(1e-6)
        err = (got.cpu().double() - want).abs().max() / scale_
        assert err < 3e-3, (name, float(err))
    check("x", xc.grad, xr.grad)
    for name in ("t", "p", "y"):
        pr = getattr(ref, name, None)
        if torch.is_tensor(pr) and pr.requires_grad:
            check(name, getattr(mod, name).grad, pr.grad)
    if ref.msg_norm is not None and ref.msg_norm.msg_scale.requires_grad:
        check("msg_scale", mod.msg_norm.msg_scale.grad, ref.msg_norm.msg_scale.grad)


def test_edge_attr_gradient_and_full_layer():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(3)
    N, E, C = 120, 900, 32
    ei = torch.randint(0, N, (2, E), generator=g)
    x, ea = torch.randn(N, C, generator=g), torch.randn(E, 7, generator=g)
    torch.manual_seed(2)
    mod = S.GENConv(C, 48, aggr="softmax", t=0.5, learn_t=True, encode_edge=True, edge_feat_dim=7, mlp_layers=2,
                    norm="layer")
    ref = __import__("copy").deepcopy(mod).double()
    xr, ear = x.double().requires_grad_(True), ea.double().requires_grad_(True)
    out_ref = ref.mlp(osp.genconv_pre_mlp(xr, ei, ref.edge_encoder(ear), "softmax", ref.t, 1.0, 0.0, None, ref.eps))
    out_ref.square().sum().backward()
    mod = mod.cuda()
    xc, eac = x.cuda().requires_grad_(True), ea.cuda().requires_grad_(True)
    out = mod(xc, ei.cuda(), eac)
    torch.testing.assert_close(out.detach().cpu(), out_ref.detach().float(), rtol=1e-3, atol=1e-4)
    out.square().sum().backward()
    for got, want in ((xc.grad, xr.grad), (eac.grad, ear.grad), (mod.t.grad, ref.t.grad),
                      (mod.edge_encoder.weight.grad, ref.edge_encoder.weight.grad),
                      (mod.mlp[0].weight.grad, ref.mlp[0].weight.grad)):
        err = (got.cpu().double() - want).abs().max() / want.abs().max().clamp_min(1e-6)
        assert err < 3e-3, float(err)
