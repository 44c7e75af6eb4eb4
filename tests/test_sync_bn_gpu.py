"""nn.SyncBatchNorm.convert_sync_batchnorm on the dense graph convolutions, on the GPU:

1. converted, eval: the same bits as the unconverted model (running statistics and affine parameters are used;
   with the fused block epilogue under no_grad too);
2. converted, train, no process group: the same bits as the unconverted model (outputs, running statistics,
   num_batches_tracked, the BatchNorm and PReLU gradients; the x, W and b gradients, which the kernels
   accumulate with atomics, to the order of their fp32 additions);
3. two ranks on one GPU (gloo through a file store, tests/sync_bn_worker.py) on c4 layer shapes split 3 + 5
   clouds: each rank's output and x-gradient slice, the running statistics and the sum over ranks of the local
   parameter gradients against fp64 autograd of the full 8-cloud batch (tests/backward_util.py);
4. with >= 2 GPUs: one DDP step of a converted MRGCN stack over NCCL against a single-GPU full-batch step with
   BatchNorm2d (tests/sync_bn_ddp_check.py under torchrun).
"""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import backward_util as bu
from oracle import dense as od
from test_sync_bn_cpu import _activations

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _init_bn(mod, g, neg_gamma=True):
    for m in mod.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            c = m.num_features
            m.weight.data = torch.randn(c, generator=g) * 0.5 + 0.8
            if neg_gamma:
                m.weight.data[::3] *= -1
            m.bias.data = torch.randn(c, generator=g) * 0.2
            m.running_mean.data = torch.randn(c, generator=g) * 0.3
            m.running_var.data = torch.rand(c, generator=g) + 0.4
        if isinstance(m, torch.nn.PReLU):
            m.weight.data.fill_(0.25)
    return mod


def _pair(make, seed):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    torch.manual_seed(seed)
    plain = _init_bn(make(D), torch.Generator().manual_seed(seed))
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain))
    assert any(isinstance(m, torch.nn.SyncBatchNorm) for m in conv.modules())
    return plain.cuda(), conv.cuda()


def _graph(B, N, k, seed):
    g = torch.Generator().manual_seed(seed)
    j = torch.randint(0, N, (B, N, k), generator=g)
    i = torch.randint(0, N, (B, N, k), generator=g)
    return torch.stack((j, i)).cuda()


LAYERS = {
    "dyn-edge": (lambda D: D.DynConv2d(64, 64, 20, 1, "edge", "relu", "batch"), False),
    "dyn-mr": (lambda D: D.DynConv2d(64, 64, 20, 1, "mr", "relu", "batch"), False),
    "dyn-edge-prelu-d3": (lambda D: D.DynConv2d(64, 64, 9, 3, "edge", "prelu", "batch"), False),
    "graph-edge": (lambda D: D.GraphConv2d(64, 64, "edge", "relu", "batch"), True),
    "graph-mr": (lambda D: D.GraphConv2d(64, 64, "mr", "leakyrelu", "batch"), True),
}


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_converted_eval_same_bits(name):
    make, given = LAYERS[name]
    plain, conv = _pair(make, 1)
    plain.eval(), conv.eval()
    x = torch.randn(2, 64, 1024, 1, generator=torch.Generator().manual_seed(2)).cuda()
    args = (x, _graph(2, 1024, 20, 3)) if given else (x,)
    with torch.no_grad():
        assert torch.equal(conv(*args), plain(*args))
    x.requires_grad_(True)     # eval with autograd (no block epilogue)
    assert torch.equal(conv(*args), plain(*args))


@pytest.mark.parametrize("block", ["res", "dense"])
@pytest.mark.parametrize("conv_type", ["edge", "mr"])
def test_converted_eval_block_epilogue_same_bits(block, conv_type):
    make = {"res": lambda D: D.ResDynBlock2d(64, 20, 2, conv_type, "relu", "batch", res_scale=0.5),
            "dense": lambda D: D.DenseDynBlock2d(64, 32, 20, 1, conv_type, "relu", "batch")}[block]
    plain, conv = _pair(make, 4)
    plain.eval(), conv.eval()
    x = torch.randn(2, 64, 1024, 1, generator=torch.Generator().manual_seed(5)).cuda()
    with torch.no_grad():
        assert conv.body.gconv.can_fuse_block(x)
        assert torch.equal(conv(x), plain(x))


@pytest.mark.parametrize("name", sorted(LAYERS))
def test_converted_train_without_process_group_same_bits(name):
    import torch.distributed as dist
    assert not (dist.is_available() and dist.is_initialized())
    make, given = LAYERS[name]
    plain, conv = _pair(make, 6)
    plain.train(), conv.train()
    x0 = torch.randn(3, 64, 1024, 1, generator=torch.Generator().manual_seed(7)).cuda()
    ei = _graph(3, 1024, 20, 8) if given else None
    wgt = torch.randn(3, 64, 1024, 1, generator=torch.Generator().manual_seed(9)).cuda()
    res = []
    for m in (plain, conv):
        x = x0.clone().requires_grad_(True)
        for _ in range(2):                      # two steps: the running statistics compound
            for p in m.parameters():
                p.grad = None
            y = m(x, ei) if given else m(x)
            (y * wgt).sum().backward()
        nn_, bn = m.gconv.nn, m.gconv.nn[2]
        exact = {"y": y, "running_mean": bn.running_mean, "running_var": bn.running_var,
                 "num_batches_tracked": bn.num_batches_tracked, "bn_w": bn.weight.grad, "bn_b": bn.bias.grad}
        if isinstance(nn_[1], torch.nn.PReLU):
            exact["slope"] = nn_[1].weight.grad
        # x, W and b gradients are accumulated with atomics: equal up to the order of fp32 additions
        res.append((exact, {"x": x.grad, "weight": nn_[0].weight.grad, "bias": nn_[0].bias.grad}))
    for key, a in res[0][0].items():
        assert torch.equal(res[1][0][key], a), key
    for key, a in res[0][1].items():
        torch.testing.assert_close(res[1][1][key], a, rtol=1e-5, atol=1e-6 * float(a.abs().max()), msg=key)
    assert int(res[1][0]["num_batches_tracked"]) == 2


# ---- two ranks on one GPU ---------------------------------------------------------------------------------------
TWO_RANK_CASES = {
    "edge-d1": dict(kind="dyn", conv="edge", act="relu", k=20, d=1, neg=False),
    "edge-d27": dict(kind="dyn", conv="edge", act="relu", k=20, d=27, neg=False),
    "mr-d1": dict(kind="dyn", conv="mr", act="relu", k=20, d=1, neg=False),
    "graph-edge": dict(kind="graph", conv="edge", act="relu", k=20, d=1, neg=False),
    "edge-prelu-neg": dict(kind="dyn", conv="edge", act="prelu", k=20, d=1, neg=True),
}
SHARDS, C, N = (3, 5), 64, 1024


def _prepare(name, spec, case_dir):
    """Module state, inputs, masked upstream gradient and the fp64 full-batch reference of one case."""
    from deep_gcns_torch_b200.gcn_lib import dense as D
    B = sum(SHARDS)
    spec = dict(spec, C=C)
    for attempt in range(8):                                   # MRConv: a seed without max near-ties
        seed = 1000 + 17 * attempt + len(name)
        g = torch.Generator().manual_seed(seed)
        torch.manual_seed(seed)
        if spec["kind"] == "dyn":
            m = D.DynConv2d(C, C, spec["k"], spec["d"], spec["conv"], spec["act"], "batch")
        else:
            m = D.GraphConv2d(C, C, spec["conv"], spec["act"], "batch")
        _init_bn(m, g, neg_gamma=spec["neg"])
        x = torch.randn(B, C, N, 1, generator=g)
        if spec["kind"] == "dyn":
            with torch.no_grad():
                ei = copy.deepcopy(m).cuda().dilated_knn_graph(x.cuda()).cpu()
            knn = dict(K=spec["k"] * spec["d"], dilation=spec["d"])
        else:
            ei = _graph(B, N, spec["k"], seed).cpu()
            knn = None
        if spec["conv"] == "mr":
            z = bu._pre_activation(x, ei, od.params_from_module(m.gconv.nn, dtype=torch.float64), "mr")
            if int((z.abs() < bu.MR_TIE_REL * z.abs().clamp_min(1.0)).sum()):
                continue
        break
    else:
        raise AssertionError("no MRConv seed without pre-activations at the kink")
    go = torch.randn(B, C, N, 1, generator=g)
    frac, x_mask = 0.0, None
    if spec["conv"] == "mr":
        x_mask = _mr_tie_targets(x, ei)
        frac = x_mask.double().mean().item()
        assert frac <= bu.MAX_MASKED
    if spec["conv"] == "edge":
        mask = bu.edge_tie_mask(x, ei, m.gconv.nn, spec["act"], "batch", True)
        go[mask] = 0
        frac = mask.double().mean().item()
    y_ref, g_ref = bu.oracle_grads(x, ei, m.gconv.nn, spec["conv"], spec["act"], "batch", True, go, knn=knn)
    p = {k: v.detach().double().clone() for k, v in m.gconv.nn[2].state_dict().items() if k.startswith("running")}
    a = _activations(x.double(), ei, m.gconv.nn, spec["conv"], spec["act"])
    F.batch_norm(a, p["running_mean"], p["running_var"], None, None, True, 0.1, 1e-5)
    cut = [0, SHARDS[0], B]
    torch.save({"name": name, "spec": spec, "state": m.state_dict(), "x": x, "grad_out": go, "cut": cut,
                "edge_index": ei}, os.path.join(case_dir, "case_%s.pt" % name))
    return {"ei": ei, "y": y_ref, "grads": g_ref, "rm": p["running_mean"], "rv": p["running_var"], "cut": cut,
            "frac": frac, "x_mask": x_mask}


def _mr_tie_targets(x, ei):
    """(B,C,N,1) bool: x entries that receive MRConv's dr through a max whose top two x_j - x_i are within
    MR_TIE_REL (fp32 may pick either neighbour; the value of r, hence the output and the parameter gradients, is
    the same).  At 8 clouds of 1024 points and 64 channels about one such max occurs per random cloud batch."""
    xd = x.double()
    v = od.batched_index_select(xd, ei[0]) - od.batched_index_select(xd, ei[1])
    top2 = v.topk(2, dim=-1)
    gap = top2.values[..., 0] - top2.values[..., 1]
    mask = torch.zeros(x.shape, dtype=torch.bool)
    for b, c, i in (gap < bu.MR_TIE_REL * top2.values[..., 0].abs().clamp_min(1.0)).nonzero().tolist():
        for l in top2.indices[b, c, i].tolist():
            mask[b, c, int(ei[0, b, i, l]), 0] = True
    return mask


@pytest.fixture(scope="module")
def two_ranks(tmp_path_factory):
    case_dir = str(tmp_path_factory.mktemp("sync_bn"))
    refs = {name: _prepare(name, spec, case_dir) for name, spec in TWO_RANK_CASES.items()}
    init_file = os.path.join(case_dir, "pg_init")
    worker = os.path.join(ROOT, "tests", "sync_bn_worker.py")
    procs = [subprocess.Popen([sys.executable, worker, str(r), "2", init_file, case_dir], cwd=ROOT,
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for r in range(2)]
    logs = []
    try:
        for p in procs:
            logs.append(p.communicate(timeout=900)[0])
    finally:
        for p in procs:                 # never leave a rank behind (a peer that died leaves the other waiting)
            if p.poll() is None:
                p.kill()
                p.wait()
    for r, (p, log) in enumerate(zip(procs, logs + [""] * (2 - len(logs)))):
        assert p.returncode == 0 and "SYNC_BN_WORKER_OK" in log, "rank %d:\n%s" % (r, log[-4000:])
    got = {name: [torch.load(os.path.join(case_dir, "result_%s_%d.pt" % (name, r))) for r in range(2)]
           for name in TWO_RANK_CASES}
    return refs, got


@pytest.mark.parametrize("name", list(TWO_RANK_CASES))
def test_two_ranks_match_full_batch(two_ranks, name):
    refs, got = two_ranks
    ref, ranks = refs[name], got[name]
    cut = ref["cut"]
    ratios = {}
    for r, res in enumerate(ranks):
        sl = slice(cut[r], cut[r + 1])
        if TWO_RANK_CASES[name]["kind"] == "dyn":      # each rank used the graph the reference is computed on
            assert torch.equal(res["edge_index"], ref["ei"][:, sl])
        ratios["y%d" % r] = bu.assert_grads_close("%s/y rank %d" % (name, r), res["y"], ref["y"][sl])
        gx, gx_ref = res["x"].clone(), ref["grads"]["x"][sl].clone()
        if ref["x_mask"] is not None:
            gx[ref["x_mask"][sl]] = 0
            gx_ref[ref["x_mask"][sl]] = 0
        ratios["x%d" % r] = bu.assert_grads_close("%s/x rank %d" % (name, r), gx, gx_ref)
        assert int(res["num_batches_tracked"]) == 1
        torch.testing.assert_close(res["running_mean"].double(), ref["rm"], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(res["running_var"].double(), ref["rv"], rtol=1e-4, atol=1e-6)
    for key, gref in ref["grads"].items():
        if key == "x":
            continue
        total = ranks[0][key].double() + ranks[1][key].double()
        ratios[key] = bu.assert_grads_close("%s/%s (sum over ranks)" % (name, key), total, gref)
        # the ranks' parameter gradients are local: neither alone is the full-batch gradient
        assert not torch.allclose(ranks[0][key].double().reshape(gref.shape), gref, rtol=1e-3, atol=0)
    print("sync-bn two-rank case %s: worst |got - ref| / max|ref| %s; masked fraction %.2e" % (
        name, " ".join("%s=%.2e" % kv for kv in ratios.items()), ref["frac"]))


# ---- two or more GPUs: DDP over NCCL ----------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_ddp_step_converted_mrgcn_matches_single_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29537", os.path.join(ROOT, "tests", "sync_bn_ddp_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "SYNC_BN_DDP_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
