"""The fused res+ block in training (res_plus_block(..., fused_training=True)) on the GPU against the four lines in
fp64 with the same keep mask (reproduced by reseeding, applied as keep / (1 - p) by hand): output, running
statistics and the gradients of h, the Linear, the BatchNorm and GENConv's learnable scalars, elementwise
(backward_util.assert_grads_close).  Also an 8-layer DeeperGCN training step, torch.utils.checkpoint and the bytes
the block saves for backward."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import backward_util as bu
import golden_util as gu
from test_res_plus_train_cpu import pack_reference
from test_sparse_backward_gpu import CFGS, _oracle_h

pytestmark = pytest.mark.gpu
SEED = 77


def _id(cfg):
    return cfg["aggr"] + ("_lt" if cfg.get("learn_t") else "") + ("_msgnorm" if cfg.get("msg_norm") else "")


def _graph(kind, N, g):
    if kind == "hub":        # a 3000-edge row (segmented hub kernels forward), empty rows at the end
        dst = torch.cat((torch.full((3000,), 5, dtype=torch.int64), torch.randint(6, N - 20, (2000,), generator=g)))
        return torch.stack((torch.randint(0, N, (5000,), generator=g), dst))
    if kind == "edgeless":
        return torch.zeros((2, 0), dtype=torch.int64)
    dst = torch.randint(0, N - 20, (3000,), generator=g)
    dst[:700] = 5
    return torch.stack((torch.randint(0, N, (3000,), generator=g), dst))


def _modules(cfg, C, mode, g):
    torch.manual_seed(1)
    conv = S().GENConv(C, C, mlp_layers=1, norm="batch", **cfg).train()
    if conv.msg_norm is not None:
        conv.msg_norm.msg_scale.data.fill_(0.7)
    norm = nn.BatchNorm1d(C, affine=mode != "noaffine", track_running_stats=mode != "untracked")
    with torch.no_grad():
        if norm.weight is not None:
            norm.weight.uniform_(0.5, 1.5, generator=g)
            norm.bias.normal_(0.0, 0.3, generator=g)
        if norm.running_mean is not None:   # near the statistics of h (randn * 1.5 + 0.3), as after training: a
            # frozen norm far off would push the power mean's messages onto its clamp at 10, a kink
            norm.running_mean.normal_(0.3, 0.1, generator=g)
            norm.running_var.uniform_(1.5, 3.0, generator=g)
    norm.train(mode != "frozen")
    return conv, norm


def S():
    from deep_gcns_torch_b200.gcn_lib import sparse
    return sparse


def _draw_keep(N, C, p):
    torch.manual_seed(SEED)
    return torch.empty((N, C), device="cuda").bernoulli_(1 - p)


def _check_block(cfg, C, p, mode="train", graph="plain", seed=0):
    from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block
    g = torch.Generator().manual_seed(seed + C)
    N = 260 if graph != "edgeless" else 50
    ei = _graph(graph, N, g)
    h = torch.randn(N, C, generator=g) * 1.5 + 0.3
    wgt = torch.randn(N, C, generator=g)
    conv, norm = _modules(cfg, C, mode, g)
    conv64, norm64 = copy.deepcopy(conv).double(), copy.deepcopy(norm).double()
    # fp64 four lines with the fused block's mask
    h64 = h.double().requires_grad_(True)
    h2 = F.relu(norm64(h64))
    if p > 0:
        h2 = h2 * (_draw_keep(N, C, p).cpu().double() / (1 - p))
    ref = h64 + conv64.mlp[0](_oracle_h(conv64, h2, ei, N))
    (ref * wgt.double()).sum().backward()
    # fused
    conv, norm = conv.cuda(), norm.cuda()
    hc = h.cuda().requires_grad_(True)
    torch.manual_seed(SEED)
    out = res_plus_block(conv, norm, hc, ei.cuda(), dropout=p, fused_training=True)
    assert type(out.grad_fn).__name__ == "_ResPlusTrainFnBackward"
    tag = "%s/C%d/p%g/%s/%s" % (_id(cfg), C, p, mode, graph)
    bu.assert_grads_close(tag + "/out", out, ref)
    for name in ("running_mean", "running_var", "num_batches_tracked"):
        a, b = getattr(norm, name), getattr(norm64, name)
        assert (a is None) == (b is None)
        if a is not None:
            bu.assert_grads_close(tag + "/" + name, a, b)
    (out * wgt.cuda()).sum().backward()
    pairs = [("h", hc.grad, h64.grad), ("W", conv.mlp[0].weight.grad, conv64.mlp[0].weight.grad),
             ("b", conv.mlp[0].bias.grad, conv64.mlp[0].bias.grad)]
    if norm.weight is not None:
        pairs += [("gamma", norm.weight.grad, norm64.weight.grad), ("beta", norm.bias.grad, norm64.bias.grad)]
    for name in ("t", "p", "y"):
        pr = getattr(conv64, name, None)
        if torch.is_tensor(pr) and pr.requires_grad:
            pairs.append((name, getattr(conv, name).grad, pr.grad))
    if conv64.msg_norm is not None and conv64.msg_norm.msg_scale.requires_grad:
        pairs.append(("msg_scale", conv.msg_norm.msg_scale.grad, conv64.msg_norm.msg_scale.grad))
    for name, got, want in pairs:
        assert got is not None, (tag, name)
        bu.assert_grads_close(tag + "/d" + name, got, want, floor=0.0 if name in ("h", "W") else 1.0)


@pytest.mark.parametrize("C", [64, 128, 200, 512])
@pytest.mark.parametrize("p", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("cfg", CFGS, ids=_id)
def test_block_matches_fp64_four_lines(cfg, p, C):
    _check_block(cfg, C, p)


@pytest.mark.parametrize("mode", ["frozen", "noaffine", "untracked"])
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("cfg", [CFGS[0], CFGS[1], CFGS[4], CFGS[8]], ids=_id)
def test_norm_modes(cfg, p, mode):
    _check_block(cfg, 128, p, mode=mode)


@pytest.mark.parametrize("graph", ["hub", "edgeless"])
@pytest.mark.parametrize("cfg", [CFGS[1], CFGS[4], CFGS[7], CFGS[8]], ids=_id)
def test_hub_row_empty_rows_and_edgeless_graph(cfg, graph):
    _check_block(cfg, 128, 0.5, graph=graph)


@pytest.mark.parametrize("C", [4, 64, 200, 512])
def test_keep_bits_layout(C):
    from deep_gcns_torch_b200 import _native
    keep = _draw_keep(301, C, 0.3)
    assert torch.equal(_native.keep_bits(keep).cpu(), pack_reference(keep.cpu()))


def test_deepergcn8_training_step_fused_matches_unfused():
    from bench_models import DeeperGCN
    from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block
    c = gu.load("model_deepergcn8")
    m = c.meta
    model = DeeperGCN(S(), m["num_layers"], m["hidden_channels"], m["in_channels"], m["num_tasks"])
    model.load_state_dict(c.sd)
    model = model.cuda().train()
    twin = copy.deepcopy(model)
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    labels = torch.randint(0, m["num_tasks"], (x.shape[0],), generator=torch.Generator().manual_seed(0)).cuda()
    p = m["dropout"]

    def step(mod, fused):
        h = mod.gcns[0](mod.enc(x), ei)
        for l in range(1, len(mod.gcns)):
            torch.manual_seed(100 + l)
            if fused:
                h = res_plus_block(mod.gcns[l], mod.norms[l - 1], h, ei, dropout=p, fused_training=True)
            else:
                keep = torch.empty(h.shape, device="cuda").bernoulli_(1 - p)
                h = mod.gcns[l](F.relu(mod.norms[l - 1](h)) * keep / (1 - p), ei) + h
        loss = F.nll_loss(torch.log_softmax(mod.pred(F.relu(mod.norms[-1](h))), dim=-1), labels)
        loss.backward()
        return loss
    loss_f, loss_u = step(model, True), step(twin, False)
    bu.assert_grads_close("loss", loss_f.reshape(1), loss_u.reshape(1))
    # Biases feeding only batch-statistics BatchNorms (the encoder's and the first GENConv's, whose output reaches
    # the loss through norms[0] and the skip connections into norms[-1]) have a gradient of 0 up to rounding:
    # their absolute term is taken from the largest gradient of the model.
    top = max(float(b.grad.abs().max()) for b in twin.parameters() if b.grad is not None)
    for (name, a), b in zip(model.named_parameters(), twin.parameters()):
        assert (a.grad is None) == (b.grad is None), name
        if a.grad is not None:
            zero = float(b.grad.abs().max()) < 1e-5 * top
            bu.assert_grads_close(name, a.grad, b.grad, floor=top if zero else 0.0)
    for (name, a), b in zip(model.named_buffers(), twin.buffers()):
        bu.assert_grads_close(name, a, b)


def test_checkpoint_gives_the_same_output_and_gradients():
    from torch.utils.checkpoint import checkpoint
    from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block
    g = torch.Generator().manual_seed(3)
    N, C = 2000, 128
    ei = torch.randint(0, N, (2, 20000), generator=g).cuda()
    conv, norm = _modules(dict(aggr="softmax", t=0.6, learn_t=True), C, "train", g)
    conv, norm = conv.cuda(), norm.cuda()
    h0 = torch.randn(N, C, generator=g).cuda()
    wgt = torch.randn(N, C, generator=g).cuda()
    results = []
    for wrapped in (False, True):
        c, n = copy.deepcopy(conv), copy.deepcopy(norm)
        h = h0.clone().requires_grad_(True)
        fn = lambda x: res_plus_block(c, n, x, ei, dropout=0.5, fused_training=True)
        torch.manual_seed(SEED)
        out = checkpoint(fn, h, use_reentrant=False) if wrapped else fn(h)
        (out * wgt).sum().backward()
        results.append([out.detach(), h.grad, c.mlp[0].weight.grad, c.mlp[0].bias.grad, n.weight.grad, n.bias.grad,
                        c.t.grad])
    assert torch.equal(results[0][0], results[1][0])
    for i, (a, b) in enumerate(zip(results[0][1:], results[1][1:])):
        bu.assert_grads_close("grad%d" % i, a, b)


def test_saved_bytes():
    from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block
    g = torch.Generator().manual_seed(4)
    N, C = 4000, 128
    ei = torch.randint(0, N, (2, 40000), generator=g).cuda()
    conv, norm = _modules(dict(aggr="softmax_sg", t=0.1), C, "train", g)
    conv, norm = conv.cuda(), norm.cuda()
    counts = {}
    for fused in (True, False):
        total = [0]

        def pack(t):
            total[0] += t.numel() * t.element_size()
            return t
        h = torch.randn(N, C, generator=g).cuda().requires_grad_(True)
        with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
            res_plus_block(conv, norm, h, ei, dropout=0.5, fused_training=fused)
        counts[fused] = total[0]
    # h (the block input, alive as the residual), a, the bits, the Linear weight (saved by reference, as nn.Linear
    # does) and C-sized vectors
    bound = 2 * N * C * 4 + N * ((C + 31) // 32) * 4 + C * C * 4 + 16 * C * 4
    assert counts[True] <= bound, counts
    assert counts[True] < 0.6 * counts[False], counts
