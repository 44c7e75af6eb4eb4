"""GENConv aggregate on fp32 against bf16 / fp16 rows at the products shape (N = 2.449 M, E = 61.9 M, C = 128; the
'block' and 'uniform' graphs of bench_multigpu.local_edges with world = 1), and one GENConv(128, 128, mlp_layers=1)
forward + backward under torch.autocast with the rows upcast by hand (x.float(): the fp32-copy path) against the
native half path.

Every timed call runs after an L2 flush; the row dtypes alternate call by call.  Reported per (graph, aggregator,
dtype): median ms and the min..max spread, the gather model's bytes per edge (source row + source index per edge;
destination row, fp32 output row and rowptr entry per node), the GB/s that gives, and the peak rise of
torch.cuda.max_memory_allocated during one call.  The card name and power limit are read in the same run.

    python tools/time_genconv_half.py [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N, E, C = 2_449_029, 61_859_140, 128
DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def bytes_per_edge(elem):
    deg = E / N
    return elem * C + 4 + (elem * C + 4 * C + 4) / deg


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import bench_multigpu
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    from deep_gcns_torch_b200.gcn_lib.sparse.torch_message import csr_of
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)         # > the 50 MB L2
    result = {"card": card(), "shape": {"N": N, "E": E, "C": C}, "aggregate": [], "genconv_autocast": []}
    g = torch.Generator(device=dev).manual_seed(0)
    x32 = torch.randn(N, C, generator=g, device=dev)
    xs = {dt: x32.to(dt) for dt in DTYPES}
    for kind in ("block", "uniform"):
        src, dst = bench_multigpu.local_edges(N, E, 0, 1, kind, dev)
        ei = torch.stack((src, dst))
        del src, dst
        csr = _native.csr_build(ei, N)
        for aggr, kw in (("softmax", dict(t=0.1)), ("power", dict(p=2.0))):
            prm, _keep = _native.genconv_params(aggr, add_residual=True, **kw)
            call = {dt: (lambda dt=dt: _native.genconv_aggregate(xs[dt], xs[dt], csr, prm)) for dt in DTYPES}
            ref = call[torch.float32]()
            for dt in DTYPES[1:]:                                           # what the timed calls compute
                assert torch.equal(call[dt](), _native.genconv_aggregate(xs[dt].float(), xs[dt].float(), csr, prm))
            del ref
            for dt in DTYPES:
                timed(call[dt], flush)                                      # warm-up
            ms = {dt: [] for dt in DTYPES}
            peak = {}
            for _ in range(args.reps):
                for dt in DTYPES:
                    t, peak[dt] = timed(call[dt], flush)
                    ms[dt].append(t)
            for dt in DTYPES:
                bpe = bytes_per_edge(dt.itemsize)
                med = statistics.median(ms[dt])
                row = {"graph": kind, "aggr": aggr, "rows": str(dt).replace("torch.", ""), "ms": round(med, 3),
                       "ms_min": round(min(ms[dt]), 3), "ms_max": round(max(ms[dt]), 3),
                       "bytes_per_edge": round(bpe, 1), "GB_s": round(bpe * E / (med * 1e-3) / 1e9, 1),
                       "peak_rise_MB": round(peak[dt] / 2 ** 20, 1)}
                result["aggregate"].append(row)
                print(json.dumps(row), flush=True)
        # one GENConv layer, forward + backward under autocast: rows upcast by hand vs the native half path
        torch.manual_seed(0)
        conv = S.GENConv(C, C, aggr="softmax", t=0.1, mlp_layers=1, norm="batch").to(dev).train()
        csr_of(ei, N)                                                       # build the cached CSR outside the timing
        wgt = torch.randn(N, C, generator=g, device=dev)
        for dt in (torch.bfloat16, torch.float16):
            xh = xs[dt].clone().requires_grad_(True)

            def step(upcast):
                with torch.autocast("cuda", dtype=dt):
                    out = conv(xh.float() if upcast else xh, ei)
                (out.float() * wgt).sum().backward()
                xh.grad = None
                conv.zero_grad(set_to_none=True)
                return None
            for up in (True, False):
                timed(lambda: step(up), flush)
            ms = {True: [], False: []}
            peak = {}
            for _ in range(args.reps):
                for up in (True, False):
                    t, peak[up] = timed(lambda: step(up), flush)
                    ms[up].append(t)
            for up in (True, False):
                row = {"graph": kind, "autocast": str(dt).replace("torch.", ""),
                       "path": "upcast x.float()" if up else "native half rows", "ms": round(statistics.median(ms[up]), 3),
                       "ms_min": round(min(ms[up]), 3), "ms_max": round(max(ms[up]), 3),
                       "peak_rise_MB": round(peak[up] / 2 ** 20, 1)}
                result["genconv_autocast"].append(row)
                print(json.dumps(row), flush=True)
        del ei, csr
        torch.cuda.empty_cache()
    print(json.dumps({"card": result["card"]}))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_genconv_half.json"), "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
