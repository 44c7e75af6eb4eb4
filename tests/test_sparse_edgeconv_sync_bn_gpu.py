"""nn.SyncBatchNorm.convert_sync_batchnorm on the sparse-layout EdgeConv (EdgConv, GraphConv / DynConv(conv='edge')
and the blocks built on them), on the GPU:

1. converted, eval: the same bits as the unconverted model, for EdgConv, GraphConv('edge'), ResDynBlock and the
   drop-in SparseDeepGCN stack;
2. converted, train, no process group: the same bits as the unconverted layer (outputs, running statistics,
   num_batches_tracked, the BatchNorm and PReLU gradients; the x, W and b gradients, which take dQ's fp32 atomic
   adds, to the order of those additions);
3. two ranks on one GPU (gloo through a file store, tests/sync_bn_sparse_worker.py): each rank's output and
   x-gradient slice, its batch statistics and running statistics, and its moments' edge count, against fp64
   autograd of sparse_edge_util.edge_conv on the whole batch; the sum over ranks of the local parameter gradients
   against the full-batch gradient, which neither rank's alone matches.  Cases: the sem_seg_sparse layer shape
   (8 clouds x 1024 points, k = 16, 64 -> 64) split 3 + 5 clouds, a ResDynBlock on its own kNN graph, a rank with
   nodes but no edges, a rank with one edge, and the module variants;
4. with >= 2 GPUs: one DDP step of the converted drop-in SparseDeepGCN over NCCL against a single-GPU full-batch
   step with BatchNorm1d (tests/sync_bn_sparse_ddp_check.py under torchrun).
"""
import copy
import os
import subprocess
import sys
import types

import pytest
import torch
from torch import nn

import backward_util as bu
import sparse_edge_util as seu
import sync_bn_sparse_worker as wk
from test_sparse_edgeconv_gpu import SparseDeepGCN
from test_sparse_edgeconv_shapes_gpu import _init_bn, _oracle

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TIE_REL, KINK_REL, MAX_MASKED = 1e-4, 1e-5, 2e-3     # as test_sparse_edgeconv_shapes_gpu.py
MEAN_REL, VAR_REL = 1e-6, 1e-5


def _deepgcn_opt():
    return types.SimpleNamespace(in_channels=9, n_filters=32, k=16, n_blocks=4, conv="edge", act="relu", norm="batch",
                                 bias=True, n_classes=13, dropout=0.0, stochastic=False, epsilon=0.2)


def _pair(make, seed):
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    torch.manual_seed(seed)
    plain = _init_bn(make(S), torch.Generator().manual_seed(seed))
    for m in plain.modules():
        if isinstance(m, nn.PReLU):
            m.weight.data.fill_(0.25)
    conv = nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    assert any(isinstance(m, nn.SyncBatchNorm) for m in conv.modules())
    return plain.cuda(), conv.cuda()


def _random_graph(N, E, g):
    return torch.randint(0, N, (2, E), generator=g)


LAYERS = {
    "EdgConv": (lambda S: S.EdgConv(24, 40, "prelu", "batch"), "graph"),
    "GraphConv-edge": (lambda S: S.GraphConv(24, 40, "edge", "relu", "batch"), "graph"),
    "ResDynBlock": (lambda S: S.ResDynBlock(24, 16, 2, "edge", "leakyrelu", "batch", res_scale=0.5), "batch"),
}


def _layer_args(kind, g):
    B, n = 3, 512
    x = torch.randn(B * n, 24, generator=g).cuda()
    if kind == "graph":
        return x, _random_graph(B * n, 12 * B * n, g).cuda()
    return x, torch.arange(B, device="cuda").repeat_interleave(n)


def _out(y):
    return y[0] if isinstance(y, tuple) else y


@pytest.mark.parametrize("name", list(LAYERS))
def test_converted_eval_same_bits(name):
    make, kind = LAYERS[name]
    plain, conv = _pair(make, 1)
    plain.eval(), conv.eval()
    x, arg = _layer_args(kind, torch.Generator().manual_seed(2))
    with torch.no_grad():
        assert torch.equal(_out(conv(x, arg)), _out(plain(x, arg)))
    x.requires_grad_(True)
    assert torch.equal(_out(conv(x, arg)), _out(plain(x, arg)))


def test_converted_sparse_deepgcn_eval_same_bits():
    plain, conv = _pair(lambda S: SparseDeepGCN(_deepgcn_opt()), 3)
    plain.eval(), conv.eval()
    g = torch.Generator().manual_seed(4)
    B, n = 2, 1024
    pos, color = torch.rand(B * n, 3, generator=g).cuda(), torch.rand(B * n, 6, generator=g).cuda()
    batch = torch.arange(B, device="cuda").repeat_interleave(n)
    with torch.no_grad():
        assert torch.equal(conv(pos, color, batch, B), plain(pos, color, batch, B))


@pytest.mark.parametrize("name", list(LAYERS))
def test_converted_train_without_process_group_same_bits(name):
    import torch.distributed as dist
    assert not (dist.is_available() and dist.is_initialized())
    make, kind = LAYERS[name]
    plain, conv = _pair(make, 6)
    plain.train(), conv.train()
    g = torch.Generator().manual_seed(7)
    x0, arg = _layer_args(kind, g)
    wgt = torch.randn(x0.shape[0], 40 if kind == "graph" else 24, generator=g).cuda()
    res = []
    for m in (plain, conv):
        edge = next(e for e in m.modules() if hasattr(e, "_parts"))
        lin, _, prelu, bn = edge._parts()
        x = x0.clone().requires_grad_(True)
        for _ in range(2):                      # two steps: the running statistics compound
            for p in m.parameters():
                p.grad = None
            (_out(m(x, arg)) * wgt).sum().backward()
        exact = {"y": _out(m(x, arg)).detach(), "running_mean": bn.running_mean, "running_var": bn.running_var,
                 "num_batches_tracked": bn.num_batches_tracked, "bn_w": bn.weight.grad, "bn_b": bn.bias.grad}
        if prelu is not None:
            exact["slope"] = prelu.grad
        res.append((exact, {"x": x.grad, "weight": lin.weight.grad, "bias": lin.bias.grad}))
    for key, a in res[0][0].items():
        assert torch.equal(res[1][0][key], a), key
    for key, a in res[0][1].items():
        bu.assert_grads_close(key, res[1][1][key], a)
    assert int(res[1][0]["num_batches_tracked"]) == 3


# ---- two ranks on one GPU ---------------------------------------------------------------------------------------
def _spec(kind="edge", ci=24, co=40, act="relu", bias=True, affine=True, track=True, momentum=0.1, **kw):
    return dict(kind=kind, ci=ci, co=co, act=act, bias=bias, affine=affine, track=track, momentum=momentum, **kw)


CLOUD, K = 1024, 16
TWO_RANK_CASES = {
    # name: (spec, per-rank (nodes, edges) of a random graph, or clouds of CLOUD points with K in-edges each)
    "sem-seg-layer": (_spec(ci=64, co=64), ("clouds", (3, 5))),
    "resdynblock": (_spec("resdyn", ci=64, co=64, k=K, d=2, res_scale=1.0), ("clouds", (3, 5))),
    "zero-edges": (_spec(), ("random", ((300, 0), (1030, 12 * 1030)))),
    "one-edge": (_spec(act="prelu"), ("random", ((50, 1), (1030, 12 * 1030)))),
    "prelu-negative": (_spec(act="prelu", slope=-0.5), ("random", ((400, 4800), (630, 7560)))),
    "leakyrelu": (_spec(act="leakyrelu"), ("random", ((400, 4800), (630, 7560)))),
    "bias-false": (_spec(bias=False), ("random", ((400, 4800), (630, 7560)))),
    "affine-false": (_spec(affine=False), ("random", ((400, 4800), (630, 7560)))),
    "momentum-none": (_spec(momentum=None), ("random", ((400, 4800), (630, 7560)))),
    "no-running-stats": (_spec(track=False), ("random", ((400, 4800), (630, 7560)))),
}


def _cloud_graph(n_clouds, g):
    N = n_clouds * CLOUD
    dst = torch.arange(N).repeat_interleave(K)
    src = torch.randint(0, CLOUD, (N * K,), generator=g) + (dst // CLOUD) * CLOUD
    return torch.stack((src, dst))


def _prepare(name, case_dir):
    """Module state, the ranks' inputs and masked upstream gradients, and the fp64 full-batch reference."""
    spec, (layout, sizes) = TWO_RANK_CASES[name]
    seed = 100 + sum(map(ord, name))
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    mod, conv = wk.build(spec)
    _init_bn(mod, g)
    for m in conv.nn:
        if isinstance(m, nn.PReLU):
            m.weight.data.fill_(spec.get("slope", 0.25))
    ci = spec["co"] if spec["kind"] == "resdyn" else spec["ci"]
    xs, eis, batches = [], [], []
    for r in range(2):
        if layout == "clouds":
            n_clouds = sizes[r]
            xs.append(torch.randn(n_clouds * CLOUD, ci, generator=g))
            batches.append(torch.arange(n_clouds).repeat_interleave(CLOUD))
            if spec["kind"] == "resdyn":
                with torch.no_grad():
                    eis.append(copy.deepcopy(mod).cuda().body.dilated_knn_graph(xs[r].cuda(), batches[r].cuda()).cpu())
            else:
                eis.append(_cloud_graph(n_clouds, g))
        else:
            n, e = sizes[r]
            xs.append(torch.randn(n, ci, generator=g))
            eis.append(_random_graph(n, e, g))
    off = [0, xs[0].shape[0], xs[0].shape[0] + xs[1].shape[0]]
    x = torch.cat(xs).cuda()
    ei = torch.cat([eis[0], eis[1] + off[1]], 1).cuda()
    mask = seu.edge_tie_mask(conv.nn, x, ei, TIE_REL, KINK_REL, True)
    frac = float(mask.double().mean())
    assert frac <= MAX_MASKED, (name, frac)
    go = torch.randn(x.shape[0], spec["co"], generator=g).cuda().masked_fill(mask, 0.0)
    y, grads, (mean, var) = _oracle(conv, x, ei, go, True)
    grads.pop("weight_terms")
    if spec["kind"] == "resdyn":                       # body(x) + x * res_scale
        y = y + x.double() * spec["res_scale"]
        grads["x"] = grads["x"] + go.double() * spec["res_scale"]
    E = ei.shape[1]
    ref = {"y": y.cpu(), "grads": {k: v.cpu() for k, v in grads.items()}, "mean": mean.cpu(), "var": var.cpu(),
           "E": E, "eis": eis, "off": off, "frac": frac}
    bn = conv.nn[1]
    if spec["track"]:
        mom = spec["momentum"] if spec["momentum"] is not None else 1.0
        ref["rm"] = (1 - mom) * bn.running_mean.double() + mom * mean.cpu()
        ref["rv"] = (1 - mom) * bn.running_var.double() + mom * var.cpu() * (E / (E - 1))
    gos = [go[off[r]:off[r + 1]].cpu() for r in range(2)]
    torch.save({"name": name, "spec": spec, "state": mod.state_dict(), "x": xs, "edge_index": eis, "batch": batches,
                "grad_out": gos}, os.path.join(case_dir, "case_%s.pt" % name))
    return ref


@pytest.fixture(scope="module")
def two_ranks(tmp_path_factory):
    case_dir = str(tmp_path_factory.mktemp("sync_bn_sparse"))
    refs = {name: _prepare(name, case_dir) for name in TWO_RANK_CASES}
    init_file = os.path.join(case_dir, "pg_init")
    worker = os.path.join(ROOT, "tests", "sync_bn_sparse_worker.py")
    procs = [subprocess.Popen([sys.executable, worker, str(r), "2", init_file, case_dir], cwd=ROOT,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    logs = []
    try:
        for p in procs:
            logs.append(p.communicate(timeout=600)[0])
    finally:
        for p in procs:                 # never leave a rank behind (a peer that died leaves the other waiting)
            if p.poll() is None:
                p.kill()
                p.wait()
    for r, (p, log) in enumerate(zip(procs, logs + [""] * (2 - len(logs)))):
        assert p.returncode == 0 and "SYNC_BN_SPARSE_WORKER_OK" in log, "rank %d:\n%s" % (r, log[-4000:])
    got = {name: [torch.load(os.path.join(case_dir, "result_%s_%d.pt" % (name, r))) for r in range(2)]
           for name in TWO_RANK_CASES}
    return refs, got


@pytest.mark.parametrize("name", list(TWO_RANK_CASES))
def test_two_ranks_match_full_batch(two_ranks, name):
    refs, got = two_ranks
    ref, ranks = refs[name], got[name]
    spec = TWO_RANK_CASES[name][0]
    off = ref["off"]
    mean, var = ref["mean"], ref["var"]
    std = var.sqrt()
    ratios = {}
    for r, res in enumerate(ranks):
        sl = slice(off[r], off[r + 1])
        assert torch.equal(res["edge_index"], ref["eis"][r])      # the graph the reference is computed on
        ratios["y%d" % r] = bu.assert_grads_close("%s/y rank %d" % (name, r), res["y"], ref["y"][sl])
        ratios["x%d" % r] = bu.assert_grads_close("%s/x rank %d" % (name, r), res["x"], ref["grads"]["x"][sl])
        # the global statistics, and the global edge count in the moments
        assert float(res["moments"][-1]) == ref["E"], (name, r, float(res["moments"][-1]))
        dm = (res["batch_mean"].double() - mean).abs()
        dv = (res["batch_var"].double() - var).abs()
        assert bool((dm <= MEAN_REL * (mean.abs() + std)).all()), (name, r, float((dm / (mean.abs() + std)).max()))
        assert bool((dv <= VAR_REL * var).all()), (name, r, float((dv / var).max()))
        if spec["track"]:
            assert int(res["num_batches_tracked"]) == 1
            torch.testing.assert_close(res["running_mean"].double(), ref["rm"], rtol=1e-4, atol=1e-6)
            torch.testing.assert_close(res["running_var"].double(), ref["rv"], rtol=1e-4, atol=1e-6)
        else:
            assert "running_mean" not in res
    empty = [r for r in range(2) if ref["eis"][r].shape[1] == 0]
    for key, gref in ref["grads"].items():
        if key == "x":
            continue
        total = ranks[0][key].double() + ranks[1][key].double()
        # a Linear's bias in front of batch statistics has a gradient that cancels to 0 (test_sparse_edgeconv_shapes)
        floor = float(ref["grads"]["weight"].abs().max()) if key == "bias" else 0.0
        ratios[key] = bu.assert_grads_close("%s/%s (sum over ranks)" % (name, key), total, gref, floor=floor)
        for r in range(2):
            if empty:               # a rank without edges holds no parameter gradient, its peer all of it
                assert not ranks[empty[0]][key].any(), (name, key)
            else:                   # the ranks' parameter gradients are local: one alone is not the full gradient
                assert not torch.allclose(ranks[r][key].double().reshape(gref.shape), gref, rtol=1e-3, atol=0), \
                    (name, key, r)
    print("sync-bn sparse two-rank case %s: worst |got - ref| / max|ref| %s; masked fraction %.2e" % (
        name, " ".join("%s=%.2e" % kv for kv in ratios.items()), ref["frac"]))


# ---- two or more GPUs: DDP over NCCL ----------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ddp_step_converted_sparse_deepgcn_matches_single_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29541",
           os.path.join(ROOT, "tests", "sync_bn_sparse_ddp_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "SYNC_BN_SPARSE_DDP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
