"""The sparse GIN / GraphSAGE aggregate on fp32 against bf16 / fp16 rows, and one PPI DeepGCN training step (conv
'gin') under torch.autocast(bfloat16) against fp32.

Aggregate shapes:
- sem_seg: the sem_seg_sparse graph, 16 clouds x 4096 points, k = 16 (the kNN graph of random points), C = 64;
- arxiv: N = 169,343, E = 2,484,941 with power-law in-degrees (hub rows), C = 128.
Every timed call runs after an L2 flush; the row dtypes alternate call by call, together with bf16 rows upcast by hand
(x.float() then the fp32 kernel, timed together).  Reported per (shape, conv, rows): median ms and the min..max spread,
the bytes model per edge (source row + source index: 2C + 4 B for half rows, 4C + 4 for fp32), the GB/s that model
gives, and the peak rise of torch.cuda.max_memory_allocated during one call.
Training step: forward + backward of examples/ppi's DeepGCN on a PPI-sized batch, fp32 against autocast bf16: median
ms and the peak rise.  The card's name, power limit and SM clock are read in the same run.

    python tools/time_gin_sage_half.py [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
CONVS = ("gin", "sage", "rsage")
UPCAST = "bfloat16 via x.float()"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, flush):
    flush.zero_()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    res = fn()
    b.record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del res
    return a.elapsed_time(b), peak


def graphs(dev):
    """(name, N, C, edge_index) of the two aggregate shapes."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator(device=dev).manual_seed(0)
    B, n = 16, 4096
    pos = torch.rand(B * n, 3, generator=g, device=dev)
    batch = torch.arange(B, device=dev).repeat_interleave(n)
    yield "sem_seg", B * n, 64, S.knn_graph_matrix(pos, 16, batch)
    N, E = 169_343, 2_484_941
    dst = (torch.rand(E, generator=g, device=dev) ** 3 * N).long()   # skewed: low ids collect thousands of edges
    src = torch.randint(0, N, (E,), generator=g, device=dev)
    yield "arxiv", N, 128, torch.stack((src, dst))


def time_aggregate(args, flush, dev, result):
    from deep_gcns_torch_b200 import _native
    for shape, N, C, ei in graphs(dev):
        csr = _native.csr_build(ei, N)
        E = ei.shape[1]
        x32 = torch.randn(N, C, generator=torch.Generator(device=dev).manual_seed(1), device=dev)
        xs = {dt: x32.to(dt) for dt in DTYPES}
        # rows: fp32, bf16 / fp16 read as they are, and bf16 upcast by hand (x.float() + the fp32 kernel: the fp32
        # copy a half input got before the kernels read half rows)
        name = {dt: str(dt).replace("torch.", "") for dt in DTYPES}
        elem = {**{name[dt]: dt.itemsize for dt in DTYPES}, UPCAST: 4}
        for conv in CONVS:
            call = {name[dt]: (lambda dt=dt: _native.gin_sage_aggregate(conv, xs[dt], csr)) for dt in DTYPES}
            call[UPCAST] = lambda: _native.gin_sage_aggregate(conv, xs[torch.bfloat16].float(), csr)
            for dt in DTYPES[1:]:                                           # what the timed calls compute
                assert torch.equal(call[name[dt]](), _native.gin_sage_aggregate(conv, xs[dt].float(), csr))
            for k in call:
                timed(call[k], flush)                                       # warm-up
            ms = {k: [] for k in call}
            peak = {}
            for _ in range(args.reps):
                for k in call:
                    t, peak[k] = timed(call[k], flush)
                    ms[k].append(t)
            for k in call:
                bpe = elem[k] * C + 4
                med = statistics.median(ms[k])
                row = {"shape": shape, "N": N, "E": E, "C": C, "hub_rows": csr[3] is not None, "conv": conv,
                       "rows": k, "ms": round(med, 3), "ms_min": round(min(ms[k]), 3),
                       "ms_max": round(max(ms[k]), 3), "bytes_per_edge": bpe,
                       "GB_s": round(bpe * E / (med * 1e-3) / 1e9, 1), "peak_rise_MB": round(peak[k] / 2 ** 20, 1)}
                result["aggregate"].append(row)
                print(json.dumps(row), flush=True)
        del csr, xs, x32, ei
        torch.cuda.empty_cache()


def time_ppi_step(args, flush, dev, result):
    """examples/ppi's DeepGCN (conv 'gin', 256 filters, 7 blocks) on 4 PPI-sized graphs at once (N = 9,716 nodes,
    E = 259,120 edges, 50 input features, 121 labels): one forward + BCE loss + backward."""
    import gin_sage_util as gsu
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    opt = dict(n_filters=256, act="relu", norm="batch", bias=True, n_heads=1, block="res", n_blocks=7,
               in_channels=50, n_classes=121, dropout=0.2, conv="gin")
    torch.manual_seed(0)
    model = gsu.ppi_deepgcn(S, opt).to(dev).train()
    g = torch.Generator(device=dev).manual_seed(2)
    N, E = 9_716, 259_120
    ei = torch.randint(0, N, (2, E), generator=g, device=dev)
    x = torch.randn(N, 50, generator=g, device=dev)
    y = (torch.rand(N, 121, generator=g, device=dev) < 0.3).float()
    lossf = torch.nn.BCEWithLogitsLoss()

    def step(autocast):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            out = model(x, ei)
        lossf(out.float(), y).backward()
        model.zero_grad(set_to_none=True)
        return None
    modes = {"fp32": False, "autocast bf16": True}
    for m in modes.values():
        timed(lambda: step(m), flush)
    ms = {k: [] for k in modes}
    peak = {}
    for _ in range(args.reps):
        for k, m in modes.items():
            t, peak[k] = timed(lambda: step(m), flush)
            ms[k].append(t)
    for k in modes:
        row = {"model": "PPI DeepGCN gin 256x7", "N": N, "E": E, "mode": k, "ms": round(statistics.median(ms[k]), 3),
               "ms_min": round(min(ms[k]), 3), "ms_max": round(max(ms[k]), 3),
               "peak_rise_MB": round(peak[k] / 2 ** 20, 1)}
        result["ppi_step"].append(row)
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)         # > the 50 MB L2
    result = {"card": card(), "aggregate": [], "ppi_step": []}
    print(json.dumps({"card": result["card"]}), flush=True)
    time_aggregate(args, flush, dev, result)
    time_ppi_step(args, flush, dev, result)
    result["card_after"] = card()
    print(json.dumps({"card_after": result["card_after"]}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_gin_sage_half.json"), "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
