"""The gradient comparison of the backward tests (tests/backward_util.py) has teeth: on CPU, at the shapes of
test_backward_shapes_gpu.py, it accepts fp32 rounding and rejects the errors a backward kernel could make -
a dropped chunk of points in the weight gradient, or a max routed to another edge outside the near-tie mask."""
import pytest
import torch

import backward_util as bu
from oracle import dense as od


def _basic_conv(c_in, c_out, act, norm, g, eval_stats=False):
    from deep_gcns_torch_b200.gcn_lib.dense.torch_nn import BasicConv
    torch.manual_seed(int(torch.randint(0, 1 << 30, (1,), generator=g)))
    nn_ = BasicConv([2 * c_in, c_out], act, norm, True)
    for m in nn_:
        if isinstance(m, torch.nn.BatchNorm2d):
            m.weight.data = torch.randn(c_out, generator=g) * 0.5 + 0.8
            m.weight.data[::3] *= -1                   # negative gammas: the max turns into a min
            m.bias.data = torch.randn(c_out, generator=g) * 0.2
            if eval_stats:
                m.running_mean.data = torch.randn(c_out, generator=g) * 0.3
                m.running_var.data = torch.rand(c_out, generator=g) + 0.4
        if isinstance(m, torch.nn.PReLU):
            m.weight.data.fill_(-0.3)
    return nn_


def _case_d_edge():
    """test_backward_shapes_gpu case d, EdgeConv: C_in 130, C_out 96, N 1030, k 9, PReLU -0.3, eval BN."""
    g = torch.Generator().manual_seed(1030)
    nn_ = _basic_conv(130, 96, "prelu", "batch", g, eval_stats=True)
    x = torch.randn(2, 130, 1030, 1, generator=g)
    ei = od.knn_matrix(x, 9)
    wgt = torch.randn(2, 96, 1030, 1, generator=g)
    wgt[bu.edge_tie_mask(x, ei, nn_, "prelu", "batch", False)] = 0
    return nn_, x, ei, wgt


def test_fp32_autograd_passes_against_fp64():
    nn_, x, ei, wgt = _case_d_edge()
    _, ref = bu.oracle_grads(x, ei, nn_, "edge", "prelu", "batch", False, wgt)
    p = od.params_from_module(nn_)
    leaves = {"x": x.clone().requires_grad_(True), "weight": p["weight"].requires_grad_(True),
              "bias": p["bias"].requires_grad_(True), "slope": p["slope"].requires_grad_(True),
              "bn_w": p["norm"]["weight"].requires_grad_(True), "bn_b": p["norm"]["bias"].requires_grad_(True)}
    (od.graph_conv(leaves["x"], ei, p, "edge", "prelu", "batch", False) * wgt).sum().backward()
    for name, leaf in leaves.items():
        bu.assert_grads_close(name, leaf.grad, ref[name])


def test_dropped_partial_chunk_fails():
    """The weight gradient is a sum over points in chunks of 512 (wgrad_kernel).  At N = 1030 the third chunk
    holds points 1024..1029; leaving it out for one cloud must fail the comparison."""
    nn_, x, ei, wgt = _case_d_edge()
    _, ref = bu.oracle_grads(x, ei, nn_, "edge", "prelu", "batch", False, wgt)
    # the kernel's factorisation: z_e = P[i] + Q[j], P = (W1 - W2) x + b, Q = W2 x
    p = od.params_from_module(nn_, dtype=torch.float64)
    C = x.shape[1]
    w = p["weight"]
    xd = x.double()
    P = torch.nn.functional.conv2d(xd, w[:, :C] - w[:, C:], p["bias"]).requires_grad_(True)
    Q = torch.nn.functional.conv2d(xd, w[:, C:]).requires_grad_(True)
    z = od.batched_index_select(P, ei[1]) + od.batched_index_select(Q, ei[0])
    y = od.normalization(od.activation(z, "prelu", p["slope"]), "batch", p["norm"], False)
    (y.max(-1, keepdim=True)[0] * wgt.double()).sum().backward()

    def wgrad(keep):
        dP, dQ, xs = P.grad * keep, Q.grad * keep, xd.squeeze(-1)
        dA = torch.einsum("bmn,bcn->mc", dP.squeeze(-1), xs)
        dW2 = torch.einsum("bmn,bcn->mc", (dQ - dP).squeeze(-1), xs)
        return torch.cat((dA, dW2), 1)

    keep = torch.ones_like(P)
    bu.assert_grads_close("weight", wgrad(keep), ref["weight"])
    keep[0, :, 1024:] = 0
    with pytest.raises(AssertionError, match="weight"):
        bu.assert_grads_close("weight", wgrad(keep), ref["weight"])


def test_max_routed_to_second_edge_fails_unless_masked():
    """test_backward_shapes_gpu case c (EdgeConv, B 2, N 4096, C 64, k 20, eval BN) on the oracle's own graph:
    sending one near-tie entry's gradient to its second edge, as an fp32 kernel may, is an O(1) error at single
    elements of grad x.  The check catches it; with the entry masked on both sides it passes."""
    g = torch.Generator().manual_seed(4096)
    nn_ = _basic_conv(64, 64, "relu", "batch", g, eval_stats=True)
    x = torch.randn(2, 64, 4096, 1, generator=g)
    ei = od.knn_matrix(x, 20)
    wgt = torch.randn(2, 64, 4096, 1, generator=g).double()
    mask = bu.edge_tie_mask(x, ei, nn_, "relu", "batch", False)

    p = od.params_from_module(nn_, dtype=torch.float64)
    xd = x.double()
    xi, xj = od.batched_index_select(xd, ei[1]), od.batched_index_select(xd, ei[0])
    z = torch.nn.functional.conv2d(torch.cat([xi, xj - xi], 1), p["weight"], p["bias"])
    # per edge, the value the max ranks: act(z) with the sign of the BN scale (same order as y = s act(z) + t)
    v = od.activation(z, "relu") * torch.where(p["norm"]["weight"] >= 0, 1.0, -1.0).double().view(1, -1, 1, 1)
    top2 = v.topk(2, -1)
    gap = top2.values[..., 0] - top2.values[..., 1]
    z2 = z.gather(-1, top2.indices[..., 1:2]).squeeze(-1)
    # a true near-tie whose second edge carries gradient (z > 0), with the largest upstream gradient
    cand = (gap < bu.TIE_REL * top2.values[..., 0].abs().clamp_min(1.0)) & (z2 > 0) & mask.squeeze(-1)
    assert int(cand.sum()) > 0
    score = torch.where(cand, wgt.squeeze(-1).abs(), torch.zeros_like(gap))
    b, c, i = torch.unravel_index(score.argmax(), score.shape)
    l1, l2 = int(top2.indices[b, c, i, 0]), int(top2.indices[b, c, i, 1])
    assert int(ei[0, b, i, l1]) != int(ei[0, b, i, l2])

    def grads(w):
        x_ = xd.clone().requires_grad_(True)
        xi_, xj_ = od.batched_index_select(x_, ei[1]), od.batched_index_select(x_, ei[0])
        Y_ = od.basic_conv(torch.cat([xi_, xj_ - xi_], 1), p, "relu", "batch", False)
        ref_loss = (Y_.max(-1, keepdim=True)[0] * w).sum()
        routed = w[b, c, i, 0] * (Y_[b, c, i, l2] - Y_[b, c, i, l1])   # the max picks l2 instead of l1
        gr, = torch.autograd.grad(ref_loss, x_, retain_graph=True)
        gk, = torch.autograd.grad(ref_loss + routed, x_)
        return gk, gr

    got, ref = grads(wgt)
    with pytest.raises(AssertionError, match="x:"):
        bu.assert_grads_close("x", got, ref)
    got, ref = grads(torch.where(mask, torch.zeros_like(wgt), wgt))
    bu.assert_grads_close("x", got, ref)
