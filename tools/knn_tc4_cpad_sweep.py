#!/usr/bin/env python
"""How much of knn_tc4_kernel's time follows its tensor-core work: time the headline layer's selection at
C in {16, 32, 48, 64} and fit kernel ms against the wgmma count per candidate tile and filter warpgroup.

    python tools/knn_tc4_cpad_sweep.py [--products 1|3] [--tile 32|64] [--rounds R] [--steps S]

Workload: DynConv2d(C, 64, k=20, d=1, edge, relu, batch).eval() forward, B=16, N=4096 - the set-only consumer of
bench.py's layer.  Only the channel count changes, so the filter, flush and consumer work stays (nearly) the same
while the wgmma count per candidate tile per group is 2 (P C/16 + 1): P = 1 for the single fp16 product, P = 3 for
the three-product bf16 split (hi*hi, hi*mid, mid*hi).  --products names the scheme of the build being measured,
--tile its candidate tile: 32 (m64n32k16 wgmma, four groups per CTA) or 64 (m64n64k16 per half-tile, the two-group
builds before).  Either way one wgmma of the count is the same tensor work per candidate, so s and t0 of the two
tile widths compare directly.

Kernel time is the "knn" bracket of _native.kernel_timing (the selection kernel and its exact completion kernel,
CUDA events on the launch stream), inputs rotate over 8 seeded batches, the configurations are alternated within
every round and the median over rounds is fitted:  ms = t0 + s * wgmma.  The share of queries the pre-filter leaves
to the completion kernel at C = 64 comes from _native.tc_certification over the 8 batches.  Prints one JSON line.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

B, N, K, C_OUT = 16, 4096, 20, 64
CHANNELS = (16, 32, 48, 64)
N_ROTATE = 8


def wgmma_per_tile(c, products):
    return 2 * (products * ((c + 15) // 16) + 1)


def device_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        info["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
        info["sm_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception as exc:                       # reporting only
        info["power_limit_note"] = "not read: %s" % type(exc).__name__
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--products", type=int, default=1, choices=(1, 3),
                    help="tensor-core products per channel block of the build measured (1: fp16, 3: bf16 split)")
    ap.add_argument("--tile", type=int, default=32, choices=(32, 64),
                    help="candidates per tile of the build measured (32: m64n32k16 wgmma, 64: m64n64k16)")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=16)
    args = ap.parse_args()

    import numpy as np
    import torch
    from deep_gcns_torch_b200 import _native
    from deep_gcns_torch_b200.gcn_lib import dense as D
    if not torch.cuda.is_available():
        raise SystemExit("knn_tc4_cpad_sweep.py needs a CUDA device")
    dev = torch.device("cuda", 0)

    layers, inputs = {}, {}
    for c in CHANNELS:
        torch.manual_seed(c)
        layers[c] = D.DynConv2d(c, C_OUT, K, 1, "edge", "relu", "batch", True).to(dev).eval()
        g = torch.Generator().manual_seed(2000 + c)
        inputs[c] = [torch.randn(B, c, N, 1, generator=g).to(dev) for _ in range(N_ROTATE)]

    times = {c: [] for c in CHANNELS}
    with torch.no_grad():
        for c in CHANNELS:                         # warm-up: module load, every shape once
            for i in range(3):
                layers[c](inputs[c][i])
        torch.cuda.synchronize()
        _native.kernel_timing(True)
        try:
            for rnd in range(args.rounds):
                order = CHANNELS if rnd % 2 == 0 else CHANNELS[::-1]
                for c in order:
                    _native.kernel_timing_read("knn")
                    for i in range(args.steps):
                        layers[c](inputs[c][i % N_ROTATE])
                    torch.cuda.synchronize()
                    ms, n = _native.kernel_timing_read("knn")
                    times[c].append(ms / max(n, 1))
        finally:
            _native.kernel_timing(False)

        _native.tc_certification(True)
        try:
            _native.tc_certification_read()
            for i in range(N_ROTATE):
                layers[64](inputs[64][i])
            failed, queries = _native.tc_certification_read()
        finally:
            _native.tc_certification(False)

    x = np.array([wgmma_per_tile(c, args.products) for c in CHANNELS], dtype=np.float64)
    med = np.array([float(np.median(times[c])) for c in CHANNELS])
    s, t0 = np.polyfit(x, med, 1)
    pred_fp16, pred_bf16 = t0 + 10 * s, t0 + 26 * s
    out = {
        "what": "knn_tc4_kernel + completion kernel ms per launch vs m64n%dk16 wgmma per %d-candidate tile per group"
                % (args.tile, args.tile),
        "products": args.products, "tile": args.tile, "rounds": args.rounds, "steps_per_round": args.steps,
        "device": device_info(),
        "points": [{"C": c, "wgmma": int(w), "kernel_ms_median": m, "kernel_ms_min": min(times[c]),
                    "kernel_ms_max": max(times[c])} for c, w, m in zip(CHANNELS, x, med)],
        "slope_ms_per_wgmma": s, "t0_ms": t0,
        "pred_ms_at_10": pred_fp16, "pred_ms_at_26": pred_bf16,
        "pred_gain_26_to_10": (pred_bf16 - pred_fp16) / pred_bf16,
        "uncertified_c64": {"failed": failed, "queries": queries, "share": failed / max(queries, 1)},
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
