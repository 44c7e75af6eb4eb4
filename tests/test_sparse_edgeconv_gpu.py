"""Sparse-layout EdgeConv (gcn_lib/sparse/torch_vertex.py:106-114, EdgConv) on the GPU: forward against the unmodified
reference (goldens spconv_edge*, model_sparse_deepgcn), gradients against fp64 autograd of sparse_edge_util.edge_conv,
exact fixtures where every tie is real, and edge cases."""
import types

import pytest
import torch
from torch import nn

import backward_util as bu
import golden_util as gu
import sparse_edge_util as seu

pytestmark = pytest.mark.gpu
RTOL, ATOL = 1e-3, 1e-4
TIE_REL, KINK_REL = 1e-4, 1e-5      # gradient tests: near-tie / kink mask (sparse_edge_util.edge_tie_mask)
MAX_MASKED = 2e-3


def _case_module(c, name):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    act = name.split("_")[0]
    mod = S.EdgConv(c.meta["C"], c.meta["out"], act, None if name.endswith("_none") else "batch", True)
    mod.load_state_dict({k[len(name) + 1:]: v for k, v in c.sd.items() if k.startswith(name + ".")}, strict=True)
    return mod.cuda(), act


def test_edgconv_matches_reference():
    """Every activation (PReLU weight > 0 and < 0) x norm None / eval BatchNorm (some gamma < 0) / train BatchNorm
    (output, batch statistics, running statistics after two steps) on a graph with empty destinations, duplicate
    edges, self-loops and a row of more than 1024 edges."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    c = gu.load("spconv_edge")
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    assert int(torch.bincount(ei[1]).max()) > 1024 and int((torch.bincount(ei[1], minlength=c.meta["N"]) == 0).sum()) > 0
    for name in c.meta["cases"]:
        mod, _ = _case_module(c, name)
        msg = lambda s_, n=name: n + ": " + s_
        if name.endswith("_train"):
            mod.train()
            bn = mod.nn[1]
            with torch.no_grad():
                prm = mod._conv_params()                  # the batch statistics the layer normalises with
                _native.sparse_edge_conv_forward(x, csr_of(ei, x.shape[0]), ei.shape[1], prm)
                torch.testing.assert_close(prm.batch_mean.cpu(), c.outs["mean_" + name], rtol=RTOL, atol=ATOL, msg=msg)
                torch.testing.assert_close(prm.batch_var.cpu(), c.outs["var_" + name], rtol=RTOL, atol=ATOL, msg=msg)
                y = mod(x, ei)
                mod(x, ei)
            torch.testing.assert_close(bn.running_mean.cpu(), c.outs["running_mean_" + name], rtol=RTOL, atol=ATOL,
                                       msg=msg)
            torch.testing.assert_close(bn.running_var.cpu(), c.outs["running_var_" + name], rtol=RTOL, atol=ATOL,
                                       msg=msg)
            assert int(bn.num_batches_tracked) == 2
        else:
            mod.eval()
            with torch.no_grad():
                y = mod(x, ei)
        torch.testing.assert_close(y.cpu(), c.outs["y_" + name], rtol=RTOL, atol=ATOL, msg=msg)


def _same_rows(got, ref, k):
    return (got.cpu().view(2, -1, k)[0].sort(-1).values == ref.long().view(2, -1, k)[0].sort(-1).values).all(-1)


def test_graphconv_dynconv_and_blocks_match_reference():
    """GraphConv head, DynConv, Res / Dense / PlainDynBlock('edge') over two equally sized clouds with dilation; kNN
    rows adjudicated as sets, features compared on the rows whose neighbour set agrees."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    c = gu.load("spconv_edge_blocks")
    m = c.meta
    C0, C, k, d = m["C0"], m["C"], m["k"], m["dilation"]
    mods = {"head": S.GraphConv(C0, C, "edge", "relu", "batch", True),
            "dyn": S.DynConv(C, C, k, d, "edge", "leakyrelu", "batch", True),
            "res": S.ResDynBlock(C, k, d, "edge", "relu", "batch", True, res_scale=0.5),
            "dense": S.DenseDynBlock(C, 8, k, d, "edge", "prelu", "batch", True),
            "plain": S.PlainDynBlock(C, k, 1, "edge", "relu", None, True)}
    for name, mod in mods.items():
        mod.load_state_dict({key[len(name) + 1:]: v for key, v in c.sd.items() if key.startswith(name + ".")},
                            strict=True)
        mod.cuda().eval()
    x, batch = c.ins["x"].cuda(), c.ins["batch"].long().cuda()
    with torch.no_grad():
        head = mods["head"](x, c.outs["graph_head"].long().cuda())
        torch.testing.assert_close(head.cpu(), c.outs["y_head"], rtol=RTOL, atol=ATOL)
        h = c.outs["y_head"].cuda()
        for name in ("dyn", "res", "dense", "plain"):
            mod = mods[name]
            body = mod if name == "dyn" else mod.body
            same = _same_rows(body.dilated_knn_graph(h, batch), c.outs["graph_" + name], k)
            assert same.float().mean() > 0.99, name
            y = mod(h, batch)
            y = y[0] if isinstance(y, tuple) else y
            torch.testing.assert_close(y.cpu()[same], c.outs["y_" + name][same], rtol=RTOL, atol=ATOL,
                                       msg=lambda s_, n=name: n + ": " + s_)
            # on the reference's graph: every row
            yg = mod(h, batch, c.outs["graph_" + name].long().cuda())
            yg = yg[0] if isinstance(yg, tuple) else yg
            torch.testing.assert_close(yg.cpu(), c.outs["y_" + name], rtol=RTOL, atol=ATOL)


def _oracle_grads(mod, act, x, ei, training, gout):
    p = seu.edge_conv_params(mod.nn, torch.float64)
    leaves = {"x": x.detach().cpu().double().requires_grad_(True), "weight": p["weight"].requires_grad_(True),
              "bias": p["bias"].requires_grad_(True)}
    if "slope" in p:
        leaves["prelu"] = p["slope"].requires_grad_(True)
    if "norm" in p:
        leaves["bn_weight"] = p["norm"]["weight"].requires_grad_(True)
        leaves["bn_bias"] = p["norm"]["bias"].requires_grad_(True)
    y = seu.edge_conv(leaves["x"], ei.cpu(), p, act, training)
    (y * gout.double()).sum().backward()
    return y.detach(), {key: v.grad for key, v in leaves.items()}


def _kernel_grads(mod, x, ei, gout):
    xg = x.clone().requires_grad_(True)
    mod.zero_grad()
    y = mod(xg, ei)
    (y * gout.cuda()).sum().backward()
    lin = mod.nn[0]
    g = {"x": xg.grad, "weight": lin.weight.grad, "bias": lin.bias.grad}
    for m in list(mod.nn)[1:]:
        if isinstance(m, nn.PReLU):
            g["prelu"] = m.weight.grad
        if isinstance(m, nn.BatchNorm1d):
            g["bn_weight"], g["bn_bias"] = m.weight.grad, m.bias.grad
    return y.detach(), g


@pytest.mark.parametrize("training", [False, True])
def test_gradients_against_fp64(training):
    """x, W, b, gamma, beta and the PReLU weight against fp64 autograd of the restatement on the kernel's graph,
    eval and train mode; the upstream gradient is zeroed (on both sides) only where an fp32 top-2 gap or a kink may
    route the max differently."""
    c = gu.load("spconv_edge")
    x, ei = c.ins["x"].cuda(), c.ins["edge_index"].long().cuda()
    g = torch.Generator().manual_seed(3)
    for name in c.meta["cases"]:
        if name.endswith("_train") != training:
            continue
        mod, act = _case_module(c, name)
        mod.train(training)
        mask = seu.edge_tie_mask(mod.nn, x, ei, TIE_REL, KINK_REL, training)
        assert mask.double().mean() <= MAX_MASKED, (name, float(mask.double().mean()))
        gout = torch.randn(c.meta["N"], c.meta["out"], generator=g).masked_fill(mask.cpu(), 0.0)
        ref_y, ref = _oracle_grads(mod, act, x, ei, training, gout)
        y, got = _kernel_grads(mod, x, ei, gout)
        torch.testing.assert_close(y.cpu().double(), ref_y, rtol=RTOL, atol=ATOL)
        assert set(got) == set(ref)
        for key in ref:
            # train mode: BatchNorm removes the Linear's bias, whose gradient is a sum of terms that cancel to 0;
            # it gets an absolute tolerance on the scale of the weight's gradient
            floor = float(ref["weight"].abs().max()) if training and key == "bias" else 0.0
            bu.assert_grads_close("%s %s" % (name, key), got[key], ref[key], floor=floor)


def _exact_module(act, norm, slope, co, ci, seed):
    """EdgConv with weights / biases in sixteenths, a dead output channel (weight and bias 0: z == 0 exactly), and
    eval BatchNorm with eps = 0, running variance in {1/4, 1, 4}, dyadic mean / beta, gamma cycling through
    {-1.5, -0.5, 0, 0.5, 1.25} (gamma = 0: every edge of a row ties)."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    import exact_util as eu
    g = torch.Generator().manual_seed(seed)
    mod = S.EdgConv(ci, co, act, norm, True)
    with torch.no_grad():
        lin = mod.nn[0]
        lin.weight.copy_(eu.sixteenths(lin.weight.shape, g))
        lin.bias.copy_(eu.sixteenths((co,), g))
        lin.weight[1] = 0
        lin.bias[1] = 0
        for m in mod.nn:
            if isinstance(m, nn.PReLU):
                m.weight.fill_(slope)
            if isinstance(m, nn.BatchNorm1d):
                m.eps = 0.0
                m.weight.copy_(torch.tensor(eu.GAMMAS)[torch.arange(co) % len(eu.GAMMAS)])
                m.bias.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_mean.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_var.copy_(4.0 ** torch.randint(-1, 2, (co,), generator=g).float())
    return mod.cuda().eval()


@pytest.mark.parametrize("act,slope", [("relu", None), ("leakyrelu", None), ("prelu", 0.25), ("prelu", -0.5)])
@pytest.mark.parametrize("norm", [None, "batch"])
def test_exact_ties_route_to_the_first_edge(act, slope, norm):
    """Integer features, weights in sixteenths: every z, every BatchNorm output and every tie is exact.  The output
    is bit-equal to the fp64 restatement, and the gradients (the max's to the first edge in edge_index order, the
    activation's act'(0) = slope) match it without any mask."""
    g = torch.Generator().manual_seed(7)
    N, ci, co = 60, 5, 40
    x = torch.randint(-4, 5, (N, ci), generator=g).float()
    x[N - 5:] = 0                                             # zero rows: z = b, u = s b + t at every such edge
    x[10] = x[11]                                             # a copy: its edges tie with the original's
    src, dst = torch.randint(0, N, (700,), generator=g), torch.randint(0, N - 3, (700,), generator=g)
    ei = torch.stack((src, dst))
    ei = torch.cat((ei, ei[:, :80], torch.tensor([[10, 11, 10, 11], [7, 7, 8, 8]])), 1)   # duplicates and copies
    mod = _exact_module(act, norm, slope, co, ci, 1)
    gout = torch.randint(-4, 5, (N, co), generator=g).float() / 4
    xc, eic = x.cuda(), ei.cuda()
    ref_y, ref = _oracle_grads(mod, act, xc, eic, False, gout)
    y, got = _kernel_grads(mod, xc, eic, gout)
    if act == "leakyrelu":      # its slope 0.2 is not dyadic: u * 0.2 rounds differently in fp32 and fp64
        torch.testing.assert_close(y.cpu().double(), ref_y, rtol=1e-6, atol=0.0)
    else:
        assert torch.equal(y.cpu(), ref_y.float())
    tol = 1e-5 if act == "leakyrelu" else 1e-6        # (leaky relu: fp32 sums of terms carrying the slope 0.2)
    for key in ref:
        bu.assert_grads_close(key, got[key], ref[key], atol_frac=tol, rtol=tol)


def test_edge_cases():
    """No edges (norm None / eval BatchNorm): zeros and zero gradients.  One edge in train mode: BatchNorm1d's
    ValueError.  An edge_index not in CSR order: the same bits as the same edges sorted by target."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    torch.manual_seed(0)
    x = torch.randn(30, 8, device="cuda")
    empty = torch.zeros((2, 0), dtype=torch.long, device="cuda")
    for norm in (None, "batch"):
        mod = S.EdgConv(8, 12, "relu", norm).cuda().eval()
        xg = x.clone().requires_grad_(True)
        y = mod(xg, empty)
        assert torch.equal(y, torch.zeros(30, 12, device="cuda"))
        y.sum().backward()
        assert torch.equal(xg.grad, torch.zeros_like(x))
        assert all(bool((p.grad == 0).all()) for p in mod.parameters())
    with pytest.raises(ValueError):
        S.EdgConv(8, 12, "relu", "batch").cuda().train()(x, torch.tensor([[1], [2]], device="cuda"))
    ei = torch.randint(0, 30, (2, 400), device="cuda")
    order = torch.sort(ei[1], stable=True).indices
    for norm, train in ((None, False), ("batch", False), ("batch", True)):
        torch.manual_seed(1)
        mod = S.EdgConv(8, 12, "prelu", norm).cuda().train(train)
        mod.nn[0].bias.data.normal_()
        a = mod(x, ei)
        b = mod(x, ei[:, order].contiguous())
        assert torch.equal(a, b), norm


def test_layers_run_forward_and_backward_on_cuda():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    torch.manual_seed(0)
    B, n = 2, 256
    batch = torch.arange(B, device="cuda").repeat_interleave(n)
    x = torch.rand(B * n, 9, device="cuda", requires_grad=True)
    head = S.GraphConv(9, 64, "edge", "relu", "batch").cuda()
    blk = S.ResDynBlock(64, 16, 2, "edge", "relu", "batch").cuda()
    ei = S.DilatedKnnGraph(16, 1)(x[:, :3].detach(), batch)
    h = head(x, ei)
    y, b2 = blk(h, batch)
    assert b2 is batch and y.shape == (B * n, 64)
    y.square().mean().backward()
    assert torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in blk.parameters())


class SparseDeepGCN(nn.Module):
    """examples/sem_seg_sparse/architecture.py:8-60 (block 'res') on the drop-in sparse classes, with the reference's
    attribute names; its scatter_('max', ., batch) over equally sized clouds is a max over each cloud's rows."""

    def __init__(self, opt):
        from deep_gcns_torch_b200.gcn_lib import sparse as S
        super().__init__()
        c, k = opt.n_filters, opt.k
        self.n_blocks = opt.n_blocks
        self.knn = S.DilatedKnnGraph(k, 1, opt.stochastic, opt.epsilon)
        self.head = S.GraphConv(opt.in_channels, c, opt.conv, opt.act, opt.norm, opt.bias)
        self.backbone = S.MultiSeq(*[S.ResDynBlock(c, k, 1 + i, opt.conv, opt.act, opt.norm, opt.bias,
                                                   stochastic=opt.stochastic, epsilon=opt.epsilon)
                                     for i in range(self.n_blocks - 1)])
        fusion_dims = c + c * (self.n_blocks - 1)
        self.fusion_block = S.MLP([fusion_dims, 1024], opt.act, opt.norm, opt.bias)
        self.prediction = S.MultiSeq(*[S.MLP([fusion_dims + 1024, 512], opt.act, opt.norm, opt.bias),
                                       S.MLP([512, 256], opt.act, opt.norm, opt.bias, drop=opt.dropout),
                                       S.MLP([256, opt.n_classes], None, None, opt.bias)])

    def tail(self, feats, n_clouds):
        f = self.fusion_block(feats)
        fusion = f.view(n_clouds, -1, f.shape[1]).max(1)[0]
        fusion = torch.repeat_interleave(fusion, repeats=feats.shape[0] // n_clouds, dim=0)
        return self.prediction(torch.cat((fusion, feats), dim=1))

    def forward(self, pos, color, batch, n_clouds):
        x = torch.cat((pos, color), dim=1)
        feats = [self.head(x, self.knn(x[:, 0:3], batch))]
        for i in range(self.n_blocks - 1):
            feats.append(self.backbone[i](feats[-1], batch)[0])
        return self.tail(torch.cat(feats, dim=1), n_clouds)


def test_sparse_deepgcn_matches_reference_model():
    """The reference's SparseDeepGCN (2 clouds x 96 points, k = 4, 16 filters, 4 res blocks) restated on the drop-in
    classes, loading its state_dict strictly: block by block on the reference's block inputs (kNN rows as sets),
    the tail, and one train-mode forward + backward against the reference's gradients.  The golden's seed leaves
    no EdgeConv max within 2e-5 of a tie or 2e-6 of the kink; that the drop-in model's own layers have none within
    half of that is checked, so that both sides route every max alike."""
    c = gu.load("model_sparse_deepgcn")
    m = c.meta
    model = SparseDeepGCN(types.SimpleNamespace(**m))
    res = model.load_state_dict(c.sd, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    model = model.cuda().eval()
    B, k = m["B"], m["k"]
    pos, color, batch = c.ins["pos"].cuda(), c.ins["color"].cuda(), c.ins["batch"].long().cuda()
    feats = [c.outs["feat%d" % i] for i in range(m["n_blocks"])]
    with torch.no_grad():
        x = torch.cat((pos, color), 1)
        same = _same_rows(model.knn(x[:, :3], batch), c.outs["graph0"], k)
        assert same.float().mean() > 0.99
        f0 = model.head(x, c.outs["graph0"].long().cuda()).cpu()
        torch.testing.assert_close(f0, feats[0], rtol=RTOL, atol=ATOL)
        for i, blk in enumerate(model.backbone):
            x_in = feats[i].cuda()
            same = _same_rows(blk.body.dilated_knn_graph(x_in, batch), c.outs["graph%d" % (i + 1)], k)
            assert same.float().mean() > 0.99, i
            out = blk(x_in, batch)[0].cpu()
            torch.testing.assert_close(out[same], feats[i + 1][same], rtol=RTOL, atol=ATOL)
        y_tail = model.tail(torch.cat([f.cuda() for f in feats], 1), B).cpu()
        torch.testing.assert_close(y_tail, c.outs["y"], rtol=RTOL, atol=ATOL)
    # one train-mode step
    model.train()
    convs = [model.head.gconv] + [blk.body.gconv for blk in model.backbone]
    seen, handles = [], []
    for conv in convs:
        handles.append(conv.register_forward_hook(lambda mod, i, o: seen.append((mod, i[0].detach(), i[1]))))
    pos_g, color_g = pos.clone().requires_grad_(True), color.clone().requires_grad_(True)
    y = model(pos_g, color_g, batch, B)
    for h in handles:
        h.remove()
    for mod, xin, ei in seen:
        assert int(seu.edge_tie_mask(mod.nn, xin, ei, 1e-5, 1e-6, training=True).sum()) == 0
    torch.testing.assert_close(y.detach().cpu(), c.outs["y_train"], rtol=RTOL, atol=ATOL)
    (y * c.outs["grad_w"].cuda()).sum().backward()
    bu.assert_grads_close("pos", pos_g.grad, c.outs["grad_pos"])
    bu.assert_grads_close("color", color_g.grad, c.outs["grad_color"])
    for name, p in model.named_parameters():
        ref = c.outs["grad." + name]
        got = p.grad if p.grad.shape == ref.shape else p.grad.sum(1)
        # a Linear's bias in front of a train-mode BatchNorm has a gradient that cancels to 0 (see above)
        floor = float(c.outs["grad." + name[:-len("bias")] + "weight"].abs().max()) \
            if name.endswith(".0.bias") and "prediction.2" not in name else 0.0
        bu.assert_grads_close(name, got, ref, floor=floor)
