"""SyncBatchNorm in the dense graph convolutions, host side (no GPU needed):

- the ctypes mirror of dgcn_bn_sync and the new status;
- `_native.sync_group` takes torch.nn.SyncBatchNorm.forward's decision (torch's own forward is run as the judge);
- the fp64 per-rank oracle of synced statistics over uneven shards equals the full-batch train-mode oracle:
  outputs, running statistics (variance unbiased with the global count) and x-gradients, and the local parameter
  gradients of the ranks sum to the full-batch ones.  That is the comparison tests/test_sync_bn_gpu.py makes.
"""
import ctypes
import types

import pytest
import torch
import torch.distributed as dist
import torch.nn.functional as F
from torch import nn

from oracle import dense as od


def test_bn_sync_struct_matches_header():
    from deep_gcns_torch_b200 import _native, build
    assert ctypes.sizeof(_native.BnSyncC) == 24
    assert [getattr(_native.BnSyncC, f).offset for f in ("moments", "reduce", "user")] == [0, 8, 16]
    build.build()
    lib = _native.lib()
    assert _native.ERR_REDUCE == -5
    assert "reduce callback" in lib.dgcn_status_string(-5).decode()


class _Judge:
    """torch's own SyncBatchNorm.forward on a CPU tensor with the collective replaced by a recorder."""

    def __init__(self, monkeypatch):
        import torch.nn.modules.batchnorm as bnmod
        self.synced = False

        class _Rec:
            @staticmethod
            def apply(x, *args):
                self.synced = True
                return x
        monkeypatch.setattr(bnmod, "sync_batch_norm", _Rec)
        # let the CPU tensor past the device check that precedes the world-size test
        monkeypatch.setattr(torch._C, "_get_privateuse1_backend_name", lambda: "cpu")

    def __call__(self, bn):
        self.synced = False
        bn(torch.randn(2, bn.num_features, 5, 1))
        return self.synced


@pytest.mark.parametrize("initialized", [False, True])
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("own_group", [False, True])
@pytest.mark.parametrize("training", [False, True])
@pytest.mark.parametrize("track", [False, True])
def test_need_sync_decision_matches_torch(monkeypatch, initialized, world, own_group, training, track):
    from deep_gcns_torch_b200 import _native
    judge = _Judge(monkeypatch)
    seen = []

    def world_size(group=None):
        seen.append(group)
        return world
    monkeypatch.setattr(dist, "is_initialized", lambda: initialized)
    monkeypatch.setattr(dist, "get_world_size", world_size)
    monkeypatch.setattr(dist, "group", types.SimpleNamespace(WORLD=object()))
    group = object() if own_group else None
    bn = nn.SyncBatchNorm(4, track_running_stats=track, process_group=group).train(training)
    want = judge(bn)
    got = _native.sync_group(bn)
    assert (got is not None) == want
    if want:
        assert got is seen[-1] and got is (group or dist.group.WORLD)
    # a plain BatchNorm2d never syncs, and the decision is the same with no process group at all
    assert _native.sync_group(nn.BatchNorm2d(4).train(training)) is None


def test_no_process_group_means_local_statistics():
    from deep_gcns_torch_b200 import _native
    assert not dist.is_initialized()
    for training in (False, True):
        assert _native.sync_group(nn.SyncBatchNorm(4).train(training)) is None


def test_dense_parts_see_sync_batchnorm():
    """convert_sync_batchnorm must not hide the norm layer from the fused kernels (eval mode uses its running
    statistics and affine parameters, train mode its batch statistics)."""
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    m = nn.SyncBatchNorm.convert_sync_batchnorm(D.DynConv2d(16, 32, 9, 1, "edge", "relu", "batch"))
    _, act, _, bn = m.gconv._parts()
    assert act == "relu" and isinstance(bn, nn.SyncBatchNorm)
    assert m.gconv.eval()._conv_params().norm == _native.NORM_BATCH_EVAL
    assert m.gconv.train()._conv_params().norm == _native.NORM_BATCH_TRAIN
    assert m.gconv._conv_params().sync_group is None


def test_dense_parts_reject_layers_the_kernels_do_not_run():
    """A BasicConv edited to hold a layer the fused kernels do not run raises instead of running without it, by the
    rule of the sparse EdgConv's MLP."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    conv = D.EdgeConv2d(4, 8, "relu", "batch")
    conv.nn.append(nn.Dropout2d(0.5))
    with pytest.raises(NotImplementedError, match="Dropout2d"):
        conv(torch.randn(1, 4, 16, 1), torch.zeros((2, 1, 16, 3), dtype=torch.long))
    conv = D.MRConv2d(4, 8, "prelu")
    conv.nn[1] = nn.PReLU(8)
    with pytest.raises(NotImplementedError, match="PReLU"):
        conv._parts()


def test_sparse_fused_block_accepts_eval_sync_batchnorm():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.fused import fusable
    conv = S.GENConv(32, 32, aggr="softmax_sg", t=0.1, mlp_layers=1)
    norm = nn.SyncBatchNorm.convert_sync_batchnorm(nn.Sequential(nn.BatchNorm1d(32)))[0].eval()
    h = torch.randn(10, 32)
    with torch.no_grad(), pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch.Tensor, "is_cuda", property(lambda t: True))     # fusable also asks for a CUDA tensor
        assert fusable(conv, nn.BatchNorm1d(32).eval(), h)
        assert fusable(conv, norm, h)
        assert not fusable(conv, norm, h.unsqueeze(-1))
        assert not fusable(conv, norm.train(), h)


# ---- fp64 per-rank oracle of synced statistics -------------------------------------------------------------
def synced_oracle(xs, eis, gconv_nn, conv, act, grad_outs, momentum=0.1, eps=1e-5):
    """Rank r holds clouds xs[r] with graph eis[r].  Each rank computes its pre-norm activations; mean and biased
    variance come from the summed [sum | sum of squares | count]; each rank normalises its own positions with them.
    Every rank has its own copy of the parameters, so the gradient of sum_r <y_r, grad_outs[r]> w.r.t. rank r's copy
    is rank r's LOCAL gradient (what SyncBatchNorm leaves to the data-parallel wrapper).
    Returns ([y_r], [{x, weight, bias, bn_w, bn_b, slope: grad}], running_mean, running_var)."""
    p = od.params_from_module(gconv_nn, dtype=torch.float64)
    leaves, acts = [], []
    for x, ei in zip(xs, eis):
        lv = {"x": x.double().requires_grad_(True), "weight": p["weight"].clone().requires_grad_(True),
              "bn_w": p["norm"]["weight"].clone().requires_grad_(True),
              "bn_b": p["norm"]["bias"].clone().requires_grad_(True)}
        if "bias" in p:
            lv["bias"] = p["bias"].clone().requires_grad_(True)
        if "slope" in p:
            lv["slope"] = p["slope"].clone().requires_grad_(True)
        xi = od.batched_index_select(lv["x"], ei[1])
        xj = od.batched_index_select(lv["x"], ei[0])
        feat = torch.cat([xi, xj - xi], 1) if conv == "edge" else torch.cat([lv["x"], (xj - xi).max(-1, keepdim=True)[0]], 1)
        acts.append(od.activation(F.conv2d(feat, lv["weight"], lv.get("bias")), act, lv.get("slope")))
        leaves.append(lv)
    s1 = sum(a.sum((0, 2, 3)) for a in acts)                  # the all-reduce of [sum | sum^2 | count]
    s2 = sum((a * a).sum((0, 2, 3)) for a in acts)
    n = sum(a.numel() // a.shape[1] for a in acts)
    mean = s1 / n
    var = s2 / n - mean * mean
    ys = []
    for a, lv in zip(acts, leaves):
        v = lambda t: t.view(1, -1, 1, 1)
        y = (a - v(mean)) / torch.sqrt(v(var) + eps) * v(lv["bn_w"]) + v(lv["bn_b"])
        ys.append(y.max(-1, keepdim=True)[0] if conv == "edge" else y)
    sum((y * g.double()).sum() for y, g in zip(ys, grad_outs)).backward()
    bn = p["norm"]
    rm = (1 - momentum) * bn["running_mean"] + momentum * mean.detach()
    rv = (1 - momentum) * bn["running_var"] + momentum * var.detach() * n / (n - 1)
    grads = [{k: t.grad for k, t in lv.items()} for lv in leaves]
    return [y.detach() for y in ys], grads, rm, rv


def _random_graph(B, N, k, g):
    j = torch.randint(0, N, (B, N, k), generator=g)
    i = torch.arange(N).view(1, N, 1).expand(B, N, k)
    return torch.stack((j, i))


@pytest.mark.parametrize("conv,act,neg_gamma", [("edge", "relu", False), ("mr", "relu", False),
                                                ("edge", "prelu", True)])
def test_synced_oracle_equals_full_batch(conv, act, neg_gamma):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(1)
    C, N, k, shards = 8, 40, 6, (3, 5)
    B = sum(shards)
    m = D.GraphConv2d(C, C, conv, act, "batch")
    bn = m.gconv.nn[2]
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        if neg_gamma:
            bn.weight[::2] *= -1
        bn.bias.uniform_(-0.5, 0.5)
        bn.running_mean.uniform_(-1, 1)
        bn.running_var.uniform_(0.5, 2)
    x = torch.randn(B, C, N, 1, generator=g, dtype=torch.float64)
    ei = _random_graph(B, N, k, g)
    go = torch.randn(B, C, N, 1, generator=g, dtype=torch.float64)
    cut = [0, shards[0], B]
    xs = [x[cut[r]:cut[r + 1]] for r in range(2)]
    eis = [ei[:, cut[r]:cut[r + 1]] for r in range(2)]
    gos = [go[cut[r]:cut[r + 1]] for r in range(2)]
    ys, grads, rm, rv = synced_oracle(xs, eis, m.gconv.nn, conv, act, gos)

    # full batch: oracle.dense train-mode BatchNorm (torch's F.batch_norm) with its running-stat update
    y_full, g_full = _full_batch(x, ei, m.gconv.nn, conv, act, go)
    torch.testing.assert_close(torch.cat(ys), y_full, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(torch.cat([gr["x"] for gr in grads]), g_full["x"], rtol=1e-10, atol=1e-12)
    for name in g_full:
        if name != "x":
            torch.testing.assert_close(grads[0][name] + grads[1][name], g_full[name], rtol=1e-10, atol=1e-12)
    # the per-rank parameter gradients are the local ones: each differs from the full-batch gradient
    assert not torch.allclose(grads[0]["bn_w"], g_full["bn_w"])
    p = od.params_from_module(m.gconv.nn, dtype=torch.float64)["norm"]
    rm_t, rv_t = p["running_mean"].clone(), p["running_var"].clone()
    a = _activations(x, ei, m.gconv.nn, conv, act)
    F.batch_norm(a, rm_t, rv_t, None, None, True, 0.1, 1e-5)   # torch: unbiased with the full count
    torch.testing.assert_close(rm, rm_t, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(rv, rv_t, rtol=1e-12, atol=1e-12)


def _activations(x, ei, gconv_nn, conv, act):
    p = od.params_from_module(gconv_nn, dtype=torch.float64)
    xi, xj = od.batched_index_select(x, ei[1]), od.batched_index_select(x, ei[0])
    feat = torch.cat([xi, xj - xi], 1) if conv == "edge" else torch.cat([x, (xj - xi).max(-1, keepdim=True)[0]], 1)
    return od.activation(F.conv2d(feat, p["weight"], p.get("bias")), act, p.get("slope"))


def _full_batch(x, ei, gconv_nn, conv, act, go):
    from backward_util import oracle_grads
    return oracle_grads(x, ei, gconv_nn, conv, act, "batch", True, go)
