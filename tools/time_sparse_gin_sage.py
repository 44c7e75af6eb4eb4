"""Time the sparse-layout GIN and GraphSAGE (GraphConv(64, 64, conv) for conv = gin / sage / rsage) at the
examples/sem_seg_sparse graph shape: N = 16 x 4096 points, k = 16 (E = 1,048,576), BatchNorm, ReLU.

    python tools/time_sparse_gin_sage.py [--reps 20]

Measures, with CUDA events (warm-up, then the median of --reps runs), eval forward and train-mode forward + backward
of the layer on a fixed kNN-shaped graph (CSR cached), against the same op sequence in torch eager on the same GPU
(index_select, scatter_reduce sum / mean, remove / add self loops, Linear, BatchNorm1d, ReLU; TF32 off), and the
aggregation kernel alone.  Prints one JSON line, with the card's name, power limit and SM clock read in the same
run."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from time_sparse_edgeconv import card, median_ms  # noqa: E402


def eager_reference(conv, x, ei, lay):
    """torch_geometric's GINConv / the reference's SAGEConv as torch eager ops."""
    N = x.shape[0]
    src, dst = ei[0], ei[1]
    if conv == "gin":
        agg = torch.zeros_like(x).scatter_reduce(0, dst.view(-1, 1).expand(-1, x.shape[1]), x.index_select(0, src),
                                                 "sum", include_self=True)
        return lay.nn(agg + (1 + lay.eps) * x)
    keep = src != dst                                                  # remove_self_loops
    loop = torch.arange(N, device=x.device)
    src, dst = torch.cat((src[keep], loop)), torch.cat((dst[keep], loop))   # add_self_loops
    msg = x.index_select(0, src)
    if lay.relative:
        msg = msg - x.index_select(0, dst)
    msg = torch.matmul(msg, lay.weight)
    aggr = torch.zeros((N, msg.shape[1]), device=x.device).scatter_reduce(
        0, dst.view(-1, 1).expand(-1, msg.shape[1]), msg, "mean", include_self=False)
    out = lay.nn(torch.cat((x, aggr), 1))
    if lay.bias is not None:
        out = out + lay.bias
    return F.normalize(out, p=2, dim=-1) if lay.normalize else out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    B, n, k, C = 16, 4096, 16, 64
    N = B * n
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(N, C, device=dev, generator=g)
    # kNN-shaped: k in-edges per point from its own cloud, self loop first (DilatedKnnGraph's knn includes self)
    cloud = torch.arange(N, device=dev) // n
    nbr = cloud.view(-1, 1) * n + torch.randint(0, n, (N, k), device=dev, generator=g)
    nbr[:, 0] = torch.arange(N, device=dev)
    ei = torch.stack((nbr.reshape(-1), torch.arange(N, device=dev).repeat_interleave(k)))
    result = {"card": card(), "shape": {"N": N, "k": k, "E": int(ei.shape[1]), "C_in": C, "C_out": C},
              "layers": "GraphConv(64, 64, conv, 'relu', 'batch', True)", "ms": {}}
    for conv in ("gin", "sage", "rsage"):
        torch.manual_seed(0)
        mod = S.GraphConv(C, C, conv, "relu", "batch", True).to(dev)
        lay = mod.gconv
        csr = csr_of(ei, N)
        eps = lay.eps if conv == "gin" else None
        r = {}
        r["aggregate_only"] = median_ms(lambda: _native.gin_sage_aggregate(conv, x, csr, eps), a.reps)
        xg = x.clone().requires_grad_(True)

        def fwd():
            with torch.no_grad():
                mod(x, ei)

        def fwd_bwd():
            mod(xg, ei).sum().backward()

        def eager_fwd():
            with torch.no_grad():
                eager_reference(conv, x, ei, lay)

        def eager_fwd_bwd():
            eager_reference(conv, xg, ei, lay).sum().backward()

        mod.eval()
        r["eval_fwd"] = median_ms(fwd, a.reps)
        r["eager_eval_fwd"] = median_ms(eager_fwd, a.reps)
        mod.train()
        r["train_fwd_bwd"] = median_ms(fwd_bwd, a.reps)
        r["eager_train_fwd_bwd"] = median_ms(eager_fwd_bwd, a.reps)
        r["speedup_eval"] = r["eager_eval_fwd"] / r["eval_fwd"]
        r["speedup_train"] = r["eager_train_fwd_bwd"] / r["train_fwd_bwd"]
        with torch.no_grad():
            mod.eval()
            r["max_abs_diff_vs_eager"] = float((mod(x, ei) - eager_reference(conv, x, ei, lay)).abs().max())
        result["ms"][conv] = r
    result["card"]["after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
