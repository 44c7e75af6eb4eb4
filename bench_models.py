#!/usr/bin/env python
"""Model-level timing of BASELINE configs 2 and 3 on one H100 (secondary; bench.py is the
headline benchmark): the reference's model assembly restated on top of the drop-in classes.

  c2  ResGCN-28 (examples/sem_seg_dense/architecture.py:7-56): DenseDilatedKnnGraph + head
      GraphConv2d + 27 ResDynBlock2d (dilation 1..27) + fusion / prediction BasicConvs,
      inputs (16, 9, 4096, 1), k=20.
  c3  DeeperGCN-56 'res+' (examples/ogb/ogbn_arxiv/model.py:80-140): 56 GENConv(128,128,
      softmax_sg, t=0.1, mlp_layers=1) + BatchNorm1d, synthetic arxiv-shaped graph.
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


class ResGCN28(torch.nn.Module):
    def __init__(self, D, in_channels=9, n_classes=13, k=20, channels=64, n_blocks=28):
        """examples/sem_seg_dense/architecture.py:7-56 restated (block='res', conv='edge', stochastic eps=0.2)."""
        super().__init__()
        self.n_blocks = n_blocks
        self.knn = D.DenseDilatedKnnGraph(k, 1, True, 0.2)
        self.head = D.GraphConv2d(in_channels, channels, "edge", "relu", "batch", True)
        self.backbone = torch.nn.Sequential(*[D.ResDynBlock2d(channels, k, 1 + i, "edge", "relu", "batch", True, True, 0.2)
                                              for i in range(n_blocks - 1)])
        fusion_dims = channels * n_blocks
        self.fusion_block = D.BasicConv([fusion_dims, 1024], "relu", "batch", True)
        self.prediction = torch.nn.Sequential(D.BasicConv([fusion_dims + 1024, 512], "relu", "batch", True),
                                              D.BasicConv([512, 256], "relu", "batch", True), torch.nn.Dropout(0.3),
                                              D.BasicConv([256, n_classes], None, None, True))

    def backbone_forward(self, inputs):
        feats = [self.head(inputs, self.knn(inputs[:, 0:3]))]
        for i in range(self.n_blocks - 1):
            feats.append(self.backbone[i](feats[-1]))
        return feats

    def backbone_forward_fused(self, inputs):
        """Same arithmetic; every block writes its output straight into its 64-channel slice of the
        (B, 64*n_blocks, N, 1) fusion buffer (examples/sem_seg_dense/architecture.py:52 builds it with torch.cat)
        and adds its skip connection in the consumer's store.  Inference only."""
        B, _, N, _ = inputs.shape
        c = self.head.gconv.nn[0].out_channels
        buf = torch.empty((B, c * self.n_blocks, N, 1), dtype=inputs.dtype, device=inputs.device)
        buf[:, :c].copy_(self.head(inputs, self.knn(inputs[:, 0:3])))
        for i in range(self.n_blocks - 1):
            self.backbone[i](buf[:, i * c:(i + 1) * c], out=buf[:, (i + 1) * c:(i + 2) * c])
        return buf

    def forward(self, inputs):
        feats = torch.cat(self.backbone_forward(inputs), dim=1)
        fusion = torch.max_pool2d(self.fusion_block(feats), kernel_size=[feats.shape[2], feats.shape[3]])
        fusion = torch.repeat_interleave(fusion, repeats=feats.shape[2], dim=2)
        return self.prediction(torch.cat((fusion, feats), dim=1)).squeeze(-1)


class MRGCN28(torch.nn.Module):
    """examples/modelnet_cls/architecture.py:11-81 restated: DilatedKnnGraph head (self excluded) +
    27 ResDynBlock2d('mr', dilation 1..27) + fusion / pooling / prediction."""

    def __init__(self, D, in_channels=3, n_classes=40, k=20, channels=64, n_blocks=28, emb=1024):
        super().__init__()
        self.n_blocks = n_blocks
        self.knn = D.DilatedKnnGraph(k, 1, False, 0.0)
        self.head = D.GraphConv2d(in_channels, channels, "mr", "relu", "batch", bias=False)
        self.backbone = torch.nn.Sequential(*[D.ResDynBlock2d(channels, k, i + 1, "mr", "relu", "batch", True, False, 0.0,
                                                              "matrix") for i in range(n_blocks - 1)])
        self.fusion_block = D.BasicConv([channels * n_blocks, emb], "leakyrelu", "batch", bias=False)
        self.prediction = torch.nn.Sequential(D.BasicConv([emb * 2, 512], "leakyrelu", "batch"),
                                              D.BasicConv([512, 256], "leakyrelu", "batch"),
                                              D.BasicConv([256, n_classes], None, None))

    def forward(self, inputs):
        feats = [self.head(inputs, self.knn(inputs[:, 0:3]))]
        for i in range(self.n_blocks - 1):
            feats.append(self.backbone[i](feats[-1]))
        fusion = self.fusion_block(torch.cat(feats, dim=1))
        x1 = F.adaptive_max_pool2d(fusion, 1)
        x2 = F.adaptive_avg_pool2d(fusion, 1)
        return self.prediction(torch.cat((x1, x2), dim=1)).squeeze(-1).squeeze(-1)


class DeeperGCN(torch.nn.Module):
    """examples/ogb/ogbn_arxiv/model.py:10-140 restated for block='res+', conv='gen' (same attribute names =
    same state_dict keys: tests/test_models_gpu.py loads the reference model's golden state_dict into it)."""

    def __init__(self, S, layers=56, hidden=128, in_channels=128, tasks=40):
        super().__init__()
        self.gcns = torch.nn.ModuleList(S.GENConv(hidden, hidden, aggr="softmax_sg", t=0.1, mlp_layers=1, norm="batch")
                                        for _ in range(layers))
        self.norms = torch.nn.ModuleList(S.norm_layer("batch", hidden) for _ in range(layers))
        self.node_features_encoder = torch.nn.Linear(in_channels, hidden)
        self.node_pred_linear = torch.nn.Linear(hidden, tasks)

    @property
    def enc(self):
        return self.node_features_encoder

    @property
    def pred(self):
        return self.node_pred_linear

    def forward(self, x, edge_index):
        h = self.gcns[0](self.enc(x), edge_index)
        for l in range(1, len(self.gcns)):
            h = self.gcns[l](F.relu(self.norms[l - 1](h)), edge_index) + h
        return torch.log_softmax(self.pred(F.relu(self.norms[-1](h))), dim=-1)

    def forward_fused(self, x, edge_index):
        """Same arithmetic with the opt-in fused 'res+' block (gcn_lib.sparse.fused): 2 launches per layer."""
        from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block
        h = self.gcns[0](self.enc(x), edge_index)
        for l in range(1, len(self.gcns)):
            h = res_plus_block(self.gcns[l], self.norms[l - 1], h, edge_index)
        return torch.log_softmax(self.pred(F.relu(self.norms[-1](h))), dim=-1)

    def forward_partitioned(self, x_local, part, layers=None, overlap=True, head=True):
        """Node-partitioned forward (deep_gcns_torch_b200.partition): every rank holds the rows
        [part.lo, part.hi) of x and of the result; one halo all-to-all per layer, overlapped with the
        interior rows; activations ping-pong between the partition's two persistent buffers."""
        from deep_gcns_torch_b200 import partition as P
        from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block_partitioned
        L = len(self.gcns) if layers is None else layers
        C = self.enc.out_features
        torch.addmm(self.enc.bias, x_local, self.enc.weight.t(), out=part.local_rows(C, 0))
        a = P.aggregate_partitioned(self.gcns[0], part, C, slot=0, overlap=overlap)
        lin = self.gcns[0].mlp[0]
        h = torch.addmm(lin.bias, a, lin.weight.t(), out=part.local_rows(C, 1))
        slot = 1
        for l in range(1, L):
            h = res_plus_block_partitioned(self.gcns[l], self.norms[l - 1], part, C, slot, scratch=a, overlap=overlap)
            slot ^= 1
        if not head:
            return h
        return torch.log_softmax(self.pred(F.relu(self.norms[L - 1](h))), dim=-1)


def graph_timeit(fn, steps=5):
    """The same call captured once into a CUDA graph (launch gaps between the model's kernels disappear) and
    replayed: ms per replay, and the captured output for a parity check."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fn()                                   # warm-up on the capture stream: caches, allocator pools
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = fn()
    graph.replay()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        graph.replay()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3, out


def timeit(fn, steps=5):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--which", default="c2,c3")
    a = ap.parse_args()
    from deep_gcns_torch_b200.gcn_lib import dense as D, sparse as S
    from oracle import sparse as osp
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    out = {}
    if "c2" in a.which:
        torch.manual_seed(0)
        model = ResGCN28(D).to(dev).eval()
        inputs = torch.rand(16, 4096, 9, generator=g).transpose(1, 2).unsqueeze(-1).contiguous().to(dev)
        with torch.no_grad():
            ms_bb = timeit(lambda: model.backbone_forward(inputs))
            ms_bb_fused = timeit(lambda: model.backbone_forward_fused(inputs))
            torch.manual_seed(3)
            unfused = torch.cat(model.backbone_forward(inputs), 1)
            torch.manual_seed(3)
            assert torch.equal(unfused, model.backbone_forward_fused(inputs))      # same bits, two passes fewer per block
            del unfused
            ms_all = timeit(lambda: model(inputs))
            try:
                torch.manual_seed(3)
                ms_graph, g_out = graph_timeit(lambda: model.backbone_forward_fused(inputs))
            except Exception as exc:
                ms_graph = "failed: %s: %s" % (type(exc).__name__, str(exc)[:200])
            per_layer = []
            feats = model.head(inputs, model.knn(inputs[:, 0:3]))
            for i in (0, 1, 2, 3, 7, 15, 26):
                blk = model.backbone[i]
                per_layer.append({"dilation": i + 1, "K": 20 * (i + 1), "ms": timeit(lambda: blk(feats), 3)})
        edges = 28 * 16 * 4096 * 20
        out["c2_resgcn28"] = {"backbone_ms": ms_bb, "backbone_ms_fused_blocks": ms_bb_fused,
                              "backbone_ms_fused_blocks_cuda_graph": ms_graph, "model_ms": ms_all, "edges_per_s_backbone": edges / (ms_bb * 1e-3),
                              "per_layer": per_layer}
    if "c4" in a.which:      # per-GPU share of config 4 (B=64 over 8 GPUs): forward + backward + SGD step
        torch.manual_seed(0)
        model = MRGCN28(D).to(dev).train()
        inputs = torch.rand(8, 3, 1024, 1, generator=g).to(dev)
        labels = torch.randint(0, 40, (8,), generator=g).to(dev)
        opt = torch.optim.SGD(model.parameters(), lr=0.01)

        def step():
            opt.zero_grad(set_to_none=True)
            loss = F.cross_entropy(model(inputs), labels)
            loss.backward()
            opt.step()
            return loss
        l0 = float(step())
        ms = timeit(step, 3)
        with torch.no_grad():
            model.eval()
            ms_fwd = timeit(lambda: model(inputs), 3)
        out["c4_mrgcn28_train_step_B8"] = {"fwd_bwd_step_ms": ms, "eval_fwd_ms": ms_fwd, "first_loss": l0,
                                           "edges_per_s_fwd_bwd": 28 * 8 * 1024 * 20 / (ms * 1e-3)}
    if "c3" in a.which:
        N = 169343
        s, d = torch.randint(0, N, (1166243,), generator=g), torch.randint(0, N, (1166243,), generator=g)
        ei = osp.to_undirected_with_self_loops(s, d, N).to(dev)
        x = torch.randn(N, 128, generator=g).to(dev)
        torch.manual_seed(0)
        model = DeeperGCN(S).to(dev).eval()
        with torch.no_grad():
            ms = timeit(lambda: model(x, ei))
            ms_fused = timeit(lambda: model.forward_fused(x, ei))
            ref_out = model(x, ei)
            torch.testing.assert_close(model.forward_fused(x, ei), ref_out, rtol=1e-3, atol=1e-4)
            try:
                ms_graph, g_out = graph_timeit(lambda: model.forward_fused(x, ei))
                torch.testing.assert_close(g_out, ref_out, rtol=1e-3, atol=1e-4)
            except Exception as exc:                       # report, do not hide
                ms_graph = "failed: %s: %s" % (type(exc).__name__, str(exc)[:200])
        out["c3_deepergcn56"] = {"model_ms": ms, "model_ms_fused_blocks": ms_fused,
                                 "model_ms_fused_blocks_cuda_graph": ms_graph,
                                 "edges_per_s": 56 * ei.shape[1] / (ms_fused * 1e-3), "E": int(ei.shape[1])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
