"""Training step of DeeperGCN res+ blocks, fused (res_plus_block(..., fused_training=True)) against the four lines,
alternated step by step in one run; CUDA events, median and min..max, and the peak rise of max_memory_allocated per
step.  With --profile, a separate short torch.profiler pass lists the GPU kernel time per step of each variant.

    python tools/time_res_plus_train.py [--steps 10] [--warmup 2] [--only arxiv|products] [--profile] [--out FILE]

arxiv:    28 layers, N = 169,343, E = 2.5 M (uniform random), C = 128, softmax_sg t = 0.1, dropout 0.5, BatchNorm1d in
          training mode; forward + backward of the stack (loss = mean of the squared output).
products: one layer, N = 2,449,029, E = 61.9 M, C = 128, same block.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_gcns_torch_b200.gcn_lib import sparse as S  # noqa: E402
from deep_gcns_torch_b200.gcn_lib.sparse.fused import res_plus_block  # noqa: E402

SHAPES = {"arxiv": dict(N=169_343, E=2_501_829, layers=28), "products": dict(N=2_449_029, E=61_859_140, layers=1)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q[0] if q else "unavailable"}


def make(N, E, layers, C=128, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ei = torch.randint(0, N, (2, E), device="cuda", generator=g)
    torch.manual_seed(seed)
    convs = torch.nn.ModuleList(S.GENConv(C, C, aggr="softmax_sg", t=0.1, mlp_layers=1) for _ in range(layers))
    norms = torch.nn.ModuleList(torch.nn.BatchNorm1d(C) for _ in range(layers))
    h0 = torch.randn(N, C, device="cuda", generator=g)
    return convs.cuda().train(), norms.cuda().train(), h0, ei


def step(convs, norms, h0, ei, fused):
    h = h0.requires_grad_(True)
    for conv, norm in zip(convs, norms):
        h = res_plus_block(conv, norm, h, ei, dropout=0.5, fused_training=fused)
    h.square().mean().backward()


def measure(name, steps, warmup):
    cfg = SHAPES[name]
    convs, norms, h0, ei = make(**cfg)
    times, peaks = {True: [], False: []}, {True: [], False: []}
    for i in range(2 * (warmup + steps)):
        fused = i % 2 == 0
        for p in list(convs.parameters()) + list(norms.parameters()):
            p.grad = None
        h0.grad = None
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step(convs, norms, h0, ei, fused)
        b.record()
        torch.cuda.synchronize()
        if i >= 2 * warmup:
            times[fused].append(a.elapsed_time(b))
            peaks[fused].append((torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    res = {}
    for fused in (True, False):
        t = times[fused]
        res["fused" if fused else "four_lines"] = dict(median_ms=statistics.median(t), min_ms=min(t), max_ms=max(t),
                                                       peak_rise_mb=max(peaks[fused]), steps=len(t))
    res["shape"] = cfg
    del convs, norms, h0, ei
    torch.cuda.empty_cache()
    return res


def profile(name):
    from torch.profiler import ProfilerActivity, profile as prof
    cfg = SHAPES[name]
    convs, norms, h0, ei = make(**cfg)
    out = {}
    for fused in (True, False):
        step(convs, norms, h0, ei, fused)
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(2):
                step(convs, norms, h0, ei, fused)
            torch.cuda.synchronize()
        rows = sorted(((e.key, e.device_time_total / 2e3, e.count // 2) for e in p.key_averages()
                       if e.device_time_total > 0), key=lambda r: -r[1])
        out["fused" if fused else "four_lines"] = [dict(kernel=k[:110], ms_per_step=round(ms, 3), calls_per_step=n)
                                                   for k, ms, n in rows[:14]]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", choices=sorted(SHAPES))
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_res_plus_train: needs a CUDA device (nothing is timed on the CPU)")
    res = {"card": card()}
    for name in ([args.only] if args.only else list(SHAPES)):
        res[name] = measure(name, args.steps, args.warmup)
        if args.profile:
            res[name + "_profile"] = profile(name)
    res["card_after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(text)


if __name__ == "__main__":
    main()
