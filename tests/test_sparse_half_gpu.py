"""bf16 / fp16 rows in the sparse GENConv path on the GPU: the aggregate kernels read half rows as they are and
must return exactly what the same call returns on the rows upcast to fp32 (forward bit for bit; gradients equal
up to the reordering of fp32 atomics), without the fp32 copies."""
import copy
import os
import subprocess
import sys

import pytest
import torch
from torch import nn

from test_sparse_backward_gpu import CFGS

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HALF = [torch.bfloat16, torch.float16]


def _id(v):
    return str(v).replace("torch.", "") if isinstance(v, torch.dtype) else None


def _prm(cfg, msg_norm):
    from deep_gcns_torch_b200 import _native
    return _native.genconv_params(cfg["aggr"], cfg.get("t", 1.0), cfg.get("p", 1.0), cfg.get("y", 0.0), 1e-7,
                                  0.7 if msg_norm else None, add_residual=True)


def _graph(N=300, seed=0):
    """A 3000-edge hub row (segmented MODE 1 / 2 kernels), 2000 edges over rows 6..N-21, empty rows at the end."""
    g = torch.Generator().manual_seed(seed)
    dst = torch.cat((torch.full((3000,), 5, dtype=torch.int64), torch.randint(6, N - 20, (2000,), generator=g)))
    return torch.stack((torch.randint(0, N, (5000,), generator=g), dst)).cuda()


def _ulp(ref, dtype):
    """One unit in the last place of `ref` (fp32 values representable in dtype) in dtype."""
    fi = torch.finfo(dtype)
    mag = ref.float().abs().clamp_min(fi.tiny)
    return torch.exp2(torch.floor(torch.log2(mag))) * fi.eps


@pytest.mark.parametrize("C", [24, 48, 128, 200, 512, 1024])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_forward_is_bit_identical_to_the_upcast_call(dtype, C):
    from deep_gcns_torch_b200 import _native
    N = 300
    ei = _graph(N, seed=C)
    csr = _native.csr_build(ei, N)
    assert csr[3] is not None                                         # the hub row takes the segmented kernels
    g = torch.Generator().manual_seed(C)
    x = torch.randn(N, C, generator=g).to(dtype).cuda()
    ea = torch.randn(ei.shape[1], C, generator=g).to(dtype).cuda()
    for cfg in CFGS:
        for msg_norm in (False, True):
            prm, _keep = _prm(cfg, msg_norm)
            for e in (None, ea):
                got = _native.genconv_aggregate(x, x, csr, prm, e)
                want = _native.genconv_aggregate(x.float(), x.float(), csr, prm, None if e is None else e.float())
                assert got.dtype == torch.float32
                assert torch.equal(got, want), (cfg, msg_norm, e is not None)
            # split launches: row_list without the hub rows, then the rest with them
            rows = torch.randperm(N, generator=g)
            first, rest = rows[:N // 2].sort().values, rows[N // 2:].sort().values
            out = torch.full((N, C), float("nan"), device="cuda")
            _native.genconv_aggregate(x, x, csr, prm, out=out, rows=first.int().cuda(), skip_hubs=True)
            _native.genconv_aggregate(x, x, csr, prm, out=out, rows=torch.cat((rest, first[first == 5])).int().cuda())
            assert torch.equal(out, _native.genconv_aggregate(x.float(), x.float(), csr, prm)), cfg


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_forward_edgeless_graph_and_raw_aggregation(dtype):
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_vertex import _aggregate_rows
    N, C = 50, 40
    g = torch.Generator().manual_seed(1)
    x = torch.randn(N, C, generator=g).to(dtype).cuda()
    empty = _native.csr_build(torch.zeros((2, 0), dtype=torch.int64, device="cuda"), N)
    for cfg in CFGS:
        prm, _keep = _prm(cfg, True)
        assert torch.equal(_native.genconv_aggregate(x, x, empty, prm), _native.genconv_aggregate(x.float(), x.float(),
                                                                                                  empty, prm))
    ei = _graph(N=300)
    xr = torch.randn(300, 64, generator=g).to(dtype).cuda()
    for aggr in ("max", "mean", "add"):                               # sparse MRConv's aggregation
        assert torch.equal(_aggregate_rows(aggr, xr, ei)[0], _aggregate_rows(aggr, xr.float(), ei)[0]), aggr
    msgs = torch.randn(ei.shape[1], 64, generator=g).to(dtype).cuda()
    for cfg in CFGS:                                                  # GenMessagePassing.aggregate on messages
        mp = S.GENConv(64, 64, mlp_layers=1, **{k: v for k, v in cfg.items() if k not in ("msg_norm",
                                                                                         "learn_msg_scale")}).cuda()
        assert torch.equal(mp.aggregate(msgs, ei[1], dim_size=300), mp.aggregate(msgs.float(), ei[1], dim_size=300))


def _max_rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp_min(1e-30))


@pytest.mark.parametrize("C", [24, 48, 128, 200, 512])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_backward_against_the_upcast_path(dtype, C):
    """Both roles (separate x_src / x_dst tensors), edge_attr, and the scalars.  grad_x_dst and grad_edge_attr are
    computed without atomics: exact.  grad_x_src and the scalars are fp32 atomics: equal up to their order."""
    from deep_gcns_torch_b200 import _native
    N = 300
    ei = _graph(N, seed=C + 1)
    csr = _native.csr_build(ei, N)
    g = torch.Generator().manual_seed(C)
    xs = torch.randn(N, C, generator=g).to(dtype).cuda()
    xd = torch.randn(N, C, generator=g).to(dtype).cuda()
    ea = torch.randn(ei.shape[1], C, generator=g).to(dtype).cuda()
    go = torch.randn(N, C, generator=g).cuda()
    for cfg in CFGS:
        scal = {k: torch.tensor([float(cfg.get(k, d))], device="cuda") for k, d in (("t", 1.0), ("p", 1.0), ("y", 0.0))}
        prm, _keep = _native.genconv_params(cfg["aggr"], scal["t"], scal["p"], scal["y"], 1e-7,
                                            torch.tensor([0.7], device="cuda") if cfg.get("msg_norm") else None)
        soft = bool(cfg.get("learn_t"))
        got = _native.genconv_aggregate_backward(xs, xd, csr, prm, go, ea, softmax_grad=soft, need_edge_attr=True)
        want = _native.genconv_aggregate_backward(xs.float(), xd.float(), csr, prm, go, ea.float(), softmax_grad=soft,
                                                  need_edge_attr=True)
        gsrc, gdst, gea, gsc = got
        assert gsrc.dtype == torch.float32 and gdst.dtype == torch.float32 and gea.dtype == dtype
        assert torch.equal(gdst, want[1]), cfg
        assert torch.equal(gea, want[2].to(dtype)), cfg
        torch.testing.assert_close(gsrc, want[0], rtol=1e-5, atol=1e-6)
        # each scalar is one fp32 atomic sum over all rows: its order alone moves it by ~1e-5 relative
        torch.testing.assert_close(gsc, want[3], rtol=5e-5, atol=1e-6)


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_module_gradients_are_in_the_input_dtype(dtype):
    """GENConv.propagate with half x and edge_attr (x in both roles): autograd hands back half gradients equal to
    the upcast path's cast to the input dtype, up to one ulp (grad x sums fp32 atomics before the cast)."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    N, C = 300, 128
    ei = _graph(N, seed=7)
    g = torch.Generator().manual_seed(7)
    x0 = torch.randn(N, C, generator=g).to(dtype).cuda()
    ea0 = torch.randn(ei.shape[1], C, generator=g).to(dtype).cuda()
    wgt = torch.randn(N, C, generator=g).cuda()
    for cfg in CFGS:
        torch.manual_seed(1)
        mod = S.GENConv(C, C, mlp_layers=1, norm="layer", **cfg).cuda()
        ref = copy.deepcopy(mod)
        scale = lambda m: m.msg_norm.msg_scale if m.msg_norm is not None else None
        x, ea = x0.clone().requires_grad_(True), ea0.clone().requires_grad_(True)
        h = mod.propagate(ei, x=x, edge_attr=ea, msg_scale=scale(mod), residual=True)
        (h * wgt).sum().backward()
        xf, eaf = x0.clone().requires_grad_(True), ea0.clone().requires_grad_(True)
        hf = ref.propagate(ei, x=xf.float(), edge_attr=eaf.float(), msg_scale=scale(ref), residual=True)
        (hf * wgt).sum().backward()
        assert torch.equal(h, hf), cfg
        assert x.grad.dtype == dtype and ea.grad.dtype == dtype
        assert torch.equal(ea.grad, eaf.grad), cfg
        bound = _ulp(xf.grad, dtype) + 1e-6 * xf.grad.float().abs().max()   # (+ fp32 noise under cancellation)
        assert bool(((x.grad.float() - xf.grad.float()).abs() <= bound).all()), cfg
        for name in ("t", "p", "y"):
            a, b = getattr(mod, name, None), getattr(ref, name, None)
            if torch.is_tensor(a) and a.requires_grad:
                torch.testing.assert_close(a.grad, b.grad, rtol=1e-5, atol=1e-6)
        if mod.msg_norm is not None and mod.msg_norm.msg_scale.requires_grad:
            torch.testing.assert_close(mod.msg_norm.msg_scale.grad, ref.msg_norm.msg_scale.grad, rtol=1e-5, atol=1e-6)


def test_memory_is_what_the_call_returns():
    """N = 1M, C = 128, E = 8M, bf16 x and edge_attr: the peak rise during a call is the output (forward) or the
    gradients (backward) and nothing else: no fp32 copy of x or edge_attr, no fp32 (E, C) edge gradient."""
    from deep_gcns_torch_b200 import _native
    N, C, E = 1 << 20, 128, 8 << 20
    g = torch.Generator(device="cuda").manual_seed(0)
    ei = torch.randint(0, N, (2, E), generator=g, device="cuda")
    csr = _native.csr_build(ei, N)
    del ei
    x = torch.randn(N, C, generator=g, device="cuda").to(torch.bfloat16)
    ea = torch.randn(E, C, generator=g, device="cuda").to(torch.bfloat16)
    go = torch.randn(N, C, generator=g, device="cuda")
    hub = 0 if csr[3] is None else csr[3][3] * 3 * C * 4
    prm, _keep = _native.genconv_params("softmax", 0.5, msg_scale=0.7)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = _native.genconv_aggregate(x, x, csr, prm, ea)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= out.numel() * 4 + hub + (1 << 20)
    del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    gsrc, gdst, gea, gsc = _native.genconv_aggregate_backward(x, x, csr, prm, go, ea, need_edge_attr=True)
    torch.cuda.synchronize()
    returned = gsrc.numel() * 4 + gdst.numel() * 4 + gea.numel() * 2 + gsc.numel() * 4
    assert gea.dtype == torch.bfloat16
    assert torch.cuda.max_memory_allocated() - base <= returned + (1 << 20)


class _ProteinsStyle(nn.Module):
    """ogbn-proteins style res+ stack: an edge encoder Linear(8, C) applied once, its output fed to every GENConv."""

    def __init__(self, S, layers=4, C=64):
        super().__init__()
        self.node_encoder = nn.Linear(16, C)
        self.edge_encoder = nn.Linear(8, C)
        self.gcns = nn.ModuleList(S.GENConv(C, C, aggr="softmax", t=0.5, learn_t=True, msg_norm=True, mlp_layers=1,
                                            norm="batch") for _ in range(layers))
        self.norms = nn.ModuleList(nn.BatchNorm1d(C) for _ in range(layers))
        self.pred = nn.Linear(C, 5)

    def forward(self, x, edge_index, edge_attr):
        ea = self.edge_encoder(edge_attr)
        h = self.gcns[0](self.node_encoder(x), edge_index, ea)
        for l in range(1, len(self.gcns)):
            h = self.gcns[l](torch.relu(self.norms[l - 1](h)), edge_index, ea) + h
        return self.pred(torch.relu(self.norms[-1](h)))


def _upcast_inputs(_mod, args):
    return tuple(a.float() if torch.is_tensor(a) and a.is_floating_point() else a for a in args)


@pytest.mark.parametrize("stack", ["deepergcn8", "proteins"])
@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_autocast_stack_matches_upcast_inputs(dtype, stack):
    import bench_models
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    N, E = 2000, 30000
    g = torch.Generator().manual_seed(5)
    ei = torch.randint(0, N, (2, E), generator=g).cuda()
    torch.manual_seed(3)
    if stack == "deepergcn8":
        model = bench_models.DeeperGCN(S, layers=8, hidden=128, in_channels=32, tasks=10).cuda().train()
        inputs = (torch.randn(N, 32, generator=g).cuda(), ei)
    else:
        model = _ProteinsStyle(S).cuda().train()
        inputs = (torch.randn(N, 16, generator=g).cuda(), ei, torch.randn(E, 8, generator=g).cuda())
    ref = copy.deepcopy(model)
    for conv in ref.gcns:
        conv.register_forward_pre_hook(_upcast_inputs)
    seen = []
    real = _native.genconv_aggregate

    def spy(x_src, x_dst, csr, prm, edge_attr=None, **kw):
        seen.append((x_src.dtype, None if edge_attr is None else edge_attr.dtype))
        return real(x_src, x_dst, csr, prm, edge_attr, **kw)
    _native.genconv_aggregate = spy
    try:
        with torch.autocast("cuda", dtype=dtype):
            out = model(*inputs)
        n_half = len(seen)
        with torch.autocast("cuda", dtype=dtype):
            out_ref = ref(*inputs)
    finally:
        _native.genconv_aggregate = real
    want = (dtype, None if stack == "deepergcn8" else dtype)
    assert seen[:n_half] == [want] * len(model.gcns)                  # the aggregate really got half rows
    assert all(s == (torch.float32, want[1] and torch.float32) for s in seen[n_half:])
    assert torch.equal(out, out_ref)
    out.float().square().mean().backward()
    out_ref.float().square().mean().backward()
    # The two backward passes differ in the order of the fp32 atomics of grad x_src, i.e. by an ulp of the
    # half-precision activation gradients, which every layer below propagates.  Weight gradients are compared
    # normwise one by one; the bias and norm gradients sum those activation gradients over all rows with strong
    # cancellation (an MLP bias gradient is ~1e-3 of its terms) and are compared as part of the whole model.
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))
    got, want = [], []
    for (name, p), q in zip(model.named_parameters(), ref.parameters()):
        assert (p.grad is None) == (q.grad is None), name
        if p.grad is not None:
            got.append(p.grad.reshape(-1))
            want.append(q.grad.reshape(-1))
            if p.dim() >= 2:
                assert rel(p.grad, q.grad) <= 0.1, (name, rel(p.grad, q.grad))
    assert rel(torch.cat(got), torch.cat(want)) <= 0.02, rel(torch.cat(got), torch.cat(want))


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_gather_rows_keeps_the_dtype(dtype):
    from deep_gcns_torch_b200 import _native
    g = torch.Generator().manual_seed(2)
    for C in (128, 40, 30):                                           # 16-byte vectors (C % 8 == 0), element copies
        x = torch.randn(1000, C, generator=g).to(dtype).cuda()
        rows = torch.randint(0, 1000, (777,), generator=g).cuda()
        got = _native.gather_rows(x, rows)
        assert got.dtype == dtype and torch.equal(got, x.index_select(0, rows))


@pytest.mark.parametrize("dtype", HALF, ids=_id)
def test_partitioned_aggregate_on_half_rows_emulated_on_one_gpu(dtype):
    """Two partitions on one GPU, the halo copied row by row: half [local | halo] rows through PartitionedAggregate,
    forward bit-identical to the single-GPU half layer and backward equal up to fp32 atomics and the cast."""
    from deep_gcns_torch_b200 import partition as P
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(4)
    N, E, C, world = 5003, 90000, 128, 2
    ei = torch.randint(0, N, (2, E), generator=g)
    ei[1, :3000] = 11
    eic = ei.cuda()
    x0 = torch.randn(N, C, generator=g).to(dtype).cuda()
    wgt = torch.randn(N, C, generator=g).cuda()
    parts = [P.GraphPartition(eic, N, r, world) for r in range(world)]
    for aggr in ("softmax", "power_sum", "max"):
        torch.manual_seed(1)
        conv = S.GENConv(C, C, aggr=aggr, t=0.3, learn_t=True, p=1.5, y=0.2, msg_norm=True, mlp_layers=1).cuda()
        t, p, y = conv._scalars()
        x = x0.clone().requires_grad_(True)
        full = conv.propagate(eic, x=x, msg_scale=conv.msg_norm.msg_scale, residual=True)
        (full * wgt).sum().backward()
        xp = x0.clone().requires_grad_(True)
        outs = []
        for part in parts:
            x_local = xp[part.lo:part.hi]
            x_src = torch.cat((x_local, xp[part.halo_nodes]))             # the emulated exchange
            assert x_src.dtype == dtype
            outs.append(P.PartitionedAggregate.apply(x_src, x_local, part, conv._check_aggr(), conv.eps,
                                                     bool(getattr(conv, "learn_t", False)), t, p, y,
                                                     conv.msg_norm.msg_scale))
        out = torch.cat(outs)
        assert torch.equal(out, full), aggr
        (out * wgt).sum().backward()
        assert xp.grad.dtype == dtype
        # per partition, grad x_src and grad x_dst are cast to half separately before autograd adds them (in half),
        # where the single-GPU layer adds them in fp32 first: a few half-precision ulps of the largest entry
        assert _max_rel(xp.grad, x.grad) <= 4 * torch.finfo(dtype).eps, (aggr, _max_rel(xp.grad, x.grad))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_halo_exchange_bf16_two_ranks():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29541", os.path.join(ROOT, "tests", "halo_half_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "HALO_HALF_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]
