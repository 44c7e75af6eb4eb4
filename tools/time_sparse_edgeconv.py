"""Time the sparse-layout EdgeConv (EdgConv / DynConv(conv='edge')) at the examples/sem_seg_sparse layer shape:
N = 16 x 4096 points, k = 16, C = 64 -> 64, BatchNorm, ReLU.

    python tools/time_sparse_edgeconv.py [--reps 20]

Measures, with CUDA events (warm-up, then the median of --reps runs):
  - eval forward and train-mode forward + backward of EdgConv on a fixed kNN graph (CSR cached), against the
    reference's op sequence in torch eager on the same GPU (index_select, cat, Linear, BatchNorm1d, ReLU,
    scatter_reduce amax; TF32 off);
  - the CSR build's share of one DynConv('edge') call (kNN graph + CSR build + EdgConv);
  - achieved bytes/s of the eval forward against a bytes-per-edge model of its edge pass.
Prints one JSON line, with the card's name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    out = {"name": torch.cuda.get_device_name()}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        out["power_limit_sm_clock_max_clock"] = q.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out["nvidia_smi"] = repr(e)
    return out


def median_ms(fn, reps, warmup=3):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


def eager_reference(x, ei, lin, bn):
    """gcn_lib/sparse/torch_vertex.py:106-114 as torch_geometric runs it: gather, cat, MLP, scatter max."""
    xi, xj = x.index_select(0, ei[1]), x.index_select(0, ei[0])
    h = torch.relu(bn(lin(torch.cat([xi, xj - xi], 1))))
    out = torch.zeros((x.shape[0], h.shape[1]), device=x.device, dtype=h.dtype)
    return out.scatter_reduce(0, ei[1].view(-1, 1).expand_as(h), h, "amax", include_self=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    B, n, k, C = 16, 4096, 16, 64
    N, E = B * n, B * n * k
    torch.manual_seed(0)
    dev = torch.device("cuda")
    x = torch.randn(N, C, device=dev)
    batch = torch.arange(B, device=dev).repeat_interleave(n)
    ei = S.DilatedKnnGraph(k, 1)(x, batch)
    conv = S.EdgConv(C, C, "relu", "batch").to(dev)
    ref_lin, ref_bn = conv.nn[0], conv.nn[1]
    res = {"shape": {"N": N, "k": k, "E": E, "C_in": C, "C_out": C}, "card": card()}

    conv.eval()
    with torch.no_grad():
        csr_of(ei, N)
        res["eval_forward_ms"] = median_ms(lambda: conv(x, ei), args.reps)
        res["eval_forward_eager_ms"] = median_ms(lambda: eager_reference(x, ei, ref_lin, ref_bn), args.reps)
    conv.train()
    xg = x.clone().requires_grad_(True)

    def train_step(fn):
        def run():
            y = fn()
            y.backward(gy)
        return run
    gy = torch.randn(N, C, device=dev)
    res["train_fwd_bwd_ms"] = median_ms(train_step(lambda: conv(xg, ei)), args.reps)
    res["train_fwd_bwd_eager_ms"] = median_ms(train_step(lambda: eager_reference(xg, ei, ref_lin, ref_bn)), args.reps)

    # CSR build's share of a DynConv('edge') call (a new graph every call: the CSR is built every time)
    dyn = S.DynConv(C, C, k, 1, "edge", "relu", "batch").to(dev).eval()
    with torch.no_grad():
        res["dynconv_eval_ms"] = median_ms(lambda: dyn(x, batch), args.reps)
        res["knn_graph_ms"] = median_ms(lambda: dyn.dilated_knn_graph(x, batch), args.reps)
        res["csr_build_ms"] = median_ms(lambda: _native.csr_build(ei, N), args.reps)
    res["csr_share_of_dynconv"] = res["csr_build_ms"] / res["dynconv_eval_ms"]

    # bytes model of the eval edge pass: per edge the int32 source index and the C_out-float Q row; per node the P
    # row, the rowptr pair and the output row (the node GEMM's traffic is not counted)
    edge_bytes = E * (4 + 4 * C) + N * (4 * C + 8 + 4 * C)
    res["eval_bytes_model"] = edge_bytes
    res["eval_bytes_per_edge"] = edge_bytes / E
    res["eval_achieved_GBps"] = edge_bytes / (res["eval_forward_ms"] * 1e-3) / 1e9
    res["speedup_eval"] = res["eval_forward_eager_ms"] / res["eval_forward_ms"]
    res["speedup_train"] = res["train_fwd_bwd_eager_ms"] / res["train_fwd_bwd_ms"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
