"""The premises of the exact tie and kink tests (tests/test_exact_ties_gpu.py), on the CPU:

- on the exact fixtures (exact_util) the pre-activations of EdgeConv and MRConv in fp32 - on the kernels' factorised
  (W1 - W2) x_i + b + W2 x_j and on the reference's W [x_i; x_j - x_i] + b - are bit-equal to fp64, the operands
  survive a round trip through bf16 and fp16, and fp32 squared distances are the exact integers;
- torch's subgradients at the kinks and ties are the ones the kernels must reproduce: relu'(0) = 0,
  leaky_relu'(0) = 0.2, prelu'(0) = slope with a zero slope gradient, torch.max(dim) routes a tie to its first index
  (also when gamma = 0 makes every BatchNorm output equal), clamp passes the gradient at its bounds, and the fp32
  message relu(10) + 1e-7 is exactly 10."""
import pytest
import torch
import torch.nn.functional as F

import exact_util as eu
from oracle import dense as od

KINDS = ["pad1", "pad25", "pad60", "zeros", "dup3", "dups"]


@pytest.mark.parametrize("C", [3, 16, 64])
def test_distances_and_operands_exact(C):
    x = eu.batch(KINDS, C, 96)
    for dt in (torch.bfloat16, torch.float16):
        assert torch.equal(x.to(dt).float(), x)
    xt = x.squeeze(-1).transpose(1, 2)
    sq = (xt * xt).sum(-1)
    d32 = sq.unsqueeze(2) - 2 * xt @ xt.transpose(1, 2) + sq.unsqueeze(1)
    d64 = (xt.double().unsqueeze(2) - xt.double().unsqueeze(1)).pow(2).sum(-1)
    assert torch.equal(d32.double(), d64)
    nbr = eu.lex_knn(x, 20)
    dd = d64.gather(2, nbr)
    assert bool((dd[..., 1:] >= dd[..., :-1]).all())
    tie = dd[..., 1:] == dd[..., :-1]
    assert bool((nbr[..., 1:][tie] > nbr[..., :-1][tie]).all())
    assert int(tie.sum()) > nbr.numel() // 4          # the fixture is mostly ties
    ex = eu.lex_knn(x, 20, exclude_self=True)
    assert not bool((ex == torch.arange(96).view(1, 96, 1)).any())


@pytest.mark.parametrize("conv", ["edge", "mr"])
@pytest.mark.parametrize("C,co", [(16, 24), (64, 64)])
def test_pre_activations_exact_in_fp32(conv, C, co):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    mod = eu.set_params(D.DynConv2d(C, co, 9, 1, conv, "relu", "batch", True), "on", seed=C)
    w = mod.gconv.nn[0].weight.detach()[:, :, 0, 0]
    b = mod.gconv.nn[0].bias.detach()
    for dt in (torch.bfloat16, torch.float16):
        assert torch.equal(w.to(dt).float(), w)
    x = eu.batch(["pad25", "dup3"], C, 128, seed=C)
    ei = eu.edge_index_of(eu.lex_knn(x, 9))
    p64 = od.params_from_module(mod.gconv.nn, dtype=torch.float64)
    xd = x.double()
    xi, xj = od.batched_index_select(xd, ei[1]), od.batched_index_select(xd, ei[0])
    if conv == "edge":
        z64 = F.conv2d(torch.cat([xi, xj - xi], 1), p64["weight"], p64["bias"])
        w1, w2 = w[:, :C], w[:, C:]
        assert torch.equal((w1 - w2).to(torch.bfloat16).float(), w1 - w2)
        P = torch.einsum("oc,bcn->bon", w1 - w2, x[..., 0]) + b.view(1, -1, 1)
        Q = torch.einsum("oc,bcn->bon", w2, x[..., 0])
        z32 = od.batched_index_select(P.unsqueeze(-1), ei[1]) + od.batched_index_select(Q.unsqueeze(-1), ei[0])
    else:
        z64 = F.conv2d(torch.cat([xd, (xj - xi).max(-1, keepdim=True)[0]], 1), p64["weight"], p64["bias"])
        x32i, x32j = od.batched_index_select(x, ei[1]), od.batched_index_select(x, ei[0])
        z32 = F.conv2d(torch.cat([x, (x32j - x32i).max(-1, keepdim=True)[0]], 1), w[:, :, None, None], b)
    assert torch.equal(z32.double(), z64)
    assert bool((z64 == 0).any())                      # zero padding: kinks hit exactly


def test_activation_subgradients_at_zero():
    z = torch.zeros(3, dtype=torch.float64, requires_grad=True)
    F.relu(z).sum().backward()
    assert z.grad.tolist() == [0.0] * 3
    z.grad = None
    F.leaky_relu(z, 0.2).sum().backward()
    assert z.grad.tolist() == [0.2] * 3
    for slope in (0.25, -0.25):
        z.grad = None
        s = torch.tensor([slope], dtype=torch.float64, requires_grad=True)
        F.prelu(z, s).sum().backward()
        assert z.grad.tolist() == [slope] * 3
        assert s.grad.item() == 0.0


def test_max_routes_ties_to_first_index():
    v = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0]], dtype=torch.float64, requires_grad=True)
    torch.max(v, -1, keepdim=True)[0].sum().backward()
    assert v.grad.tolist() == [[0.0, 1.0, 0.0, 0.0, 0.0]]
    # gamma = 0: every BatchNorm output of the row equals beta, eval and train, and the max routes to edge 0
    a = torch.tensor([[[[1.0, 3.0, -2.0, 0.0]]]], dtype=torch.float64, requires_grad=True)
    for training in (False, True):
        a.grad = None
        gamma = torch.zeros(1, dtype=torch.float64, requires_grad=True)
        beta = torch.full((1,), 0.25, dtype=torch.float64)
        y = F.batch_norm(a, torch.zeros(1, dtype=torch.float64), torch.ones(1, dtype=torch.float64), gamma, beta,
                         training, 0.1, 1e-5)
        assert bool((y == 0.25).all())
        torch.max(y, -1, keepdim=True)[0].sum().backward()
        ahat = (a.detach() - (a.detach().mean() if training else 0.0)) / torch.sqrt(
            (a.detach().var(unbiased=False) if training else 1.0) + torch.tensor(1e-5, dtype=torch.float64))
        assert gamma.grad.item() == pytest.approx(float(ahat[0, 0, 0, 0]), rel=1e-12)


def test_clamp_bounds_and_message_at_ten():
    m = torch.tensor([1e-7, 5.0, 10.0, 10.5], dtype=torch.float64, requires_grad=True)
    m.clamp(1e-7, 10.0).sum().backward()
    assert m.grad.tolist() == [1.0, 1.0, 1.0, 0.0]
    ten = F.relu(torch.tensor([10.0, 0.0, 1.0])) + 1e-7
    assert ten[0].item() == 10.0                       # fp32: 10 + 1e-7 rounds back to 10
    assert ten[1].item() == torch.tensor(1e-7).item() and ten[2].item() != 1.0
