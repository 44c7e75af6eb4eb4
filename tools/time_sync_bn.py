"""Cost of SyncBatchNorm in data-parallel MRGCN-28 training (BASELINE config c4): the DDP step time of
bench_multigpu.ddp_mrgcn_block with and without nn.SyncBatchNorm.convert_sync_batchnorm, alternated.

    torchrun --nproc-per-node <GPUs> tools/time_sync_bn.py [--rounds 3]

Synced, the 28 graph convolutions add 56 all-reduces of 2*64 + 1 doubles per step (one forward, one backward
each); torch adds its own for the norms of the tail.  Rank 0 prints one JSON line with the card and its power
limit."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import bench_multigpu as bm
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    runs = {False: [], True: []}
    for _ in range(args.rounds):
        for m in (False, True):
            r = bm.ddp_mrgcn_block(dev, rank, world, sync_bn=m)
            assert r["parity_ok"], r["parity_note"]
            runs[m].append(r["step_ms"])
    if rank == 0:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip().splitlines()
        med = {m: sorted(v)[len(v) // 2] for m, v in runs.items()}
        out = {"gpus": world, "card": q[0] if q else torch.cuda.get_device_name(dev),
               "step_ms_local_bn": runs[False], "step_ms_sync_bn": runs[True],
               "sync_overhead_ms_median": med[True] - med[False]}
        print(json.dumps(out))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
