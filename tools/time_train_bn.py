"""Cost of the train-mode BatchNorm statistics: a train-mode forward + backward of one ResGCN-28 backbone layer
(DynConv2d EdgeConv, B = 8, N = 4096, C = 64, k = 16, dilation 1 and 4) and of one MRConv layer at the same shape,
timed with CUDA events for two source trees whose library is already built, alternated round by round.

    python tools/time_train_bn.py --trees PARENT_ROOT THIS_ROOT [--rounds 5] [--iters 20] [--out FILE]

Each measurement runs in a fresh interpreter that imports the package from its tree.  Prints one JSON line with the
median milliseconds per layer step of every tree, the card and its power limit."""
import argparse
import json
import os
import subprocess
import sys

LAYERS = {"edge-d1": ("edge", 1), "edge-d4": ("edge", 4), "mr-d1": ("mr", 1)}


def measure(iters):
    import torch
    from deep_gcns_torch_b200.gcn_lib import dense as D
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    x0 = torch.randn(8, 64, 4096, 1, generator=g).to(dev)
    go = torch.randn(8, 64, 4096, 1, generator=g).to(dev)
    res = {}
    for name, (conv, d) in LAYERS.items():
        torch.manual_seed(0)
        m = D.DynConv2d(64, 64, 16, d, conv, "relu", "batch").to(dev).train()
        x = x0.clone().requires_grad_(True)

        def step():
            y = m(x)
            y.backward(go)
        for _ in range(3):
            step()
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(iters):
            step()
        t1.record()
        t1.synchronize()
        res[name] = t0.elapsed_time(t1) / iters
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trees", nargs=2, required=False)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    ap.add_argument("--child", action="store_true")
    args = ap.parse_args()
    if args.child:                     # run from the tree under test: its package comes first on sys.path
        sys.path.insert(0, os.getcwd())
        print(json.dumps(measure(args.iters)))
        return
    runs = {t: [] for t in args.trees}
    for _ in range(args.rounds):
        for t in args.trees:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--iters", str(args.iters)],
                               cwd=t, capture_output=True, text=True, check=True)
            runs[t].append(json.loads(r.stdout.strip().splitlines()[-1]))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    out = {"card": q[0] if q else None, "rounds": args.rounds, "iters": args.iters, "ms_per_step": {}}
    for t, rs in runs.items():
        out["ms_per_step"][t] = {k: sorted(r[k] for r in rs)[len(rs) // 2] for k in LAYERS}
        out["ms_per_step"][t]["all_rounds"] = rs
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
