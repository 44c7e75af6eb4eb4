"""One rank of tests/test_sync_bn_gpu.py's two-rank check: `python sync_bn_worker.py RANK WORLD INIT_FILE CASE_DIR`.

Joins a gloo process group through a file store (several ranks may share one GPU: gloo all-reduces CUDA tensors
through host memory), then for every CASE_DIR/case_<name>.pt runs one training step of the converted
(SyncBatchNorm) layer on this rank's clouds and writes CASE_DIR/result_<name>_<rank>.pt: output, x-gradient,
LOCAL parameter gradients, running statistics, num_batches_tracked and the graph the layer used."""
import glob
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def build(spec):
    from deep_gcns_torch_b200.gcn_lib import dense as D
    if spec["kind"] == "dyn":
        return D.DynConv2d(spec["C"], spec["C"], spec["k"], spec["d"], spec["conv"], spec["act"], "batch")
    return D.GraphConv2d(spec["C"], spec["C"], spec["conv"], spec["act"], "batch")


def run_case(path, rank, dev):
    from deep_gcns_torch_b200 import _native
    case = torch.load(path)
    spec = case["spec"]
    lo, hi = case["cut"][rank], case["cut"][rank + 1]
    m = build(spec)
    m.load_state_dict(case["state"])
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m).to(dev).train()
    gc = m.gconv
    bn = gc.nn[2]
    assert isinstance(bn, torch.nn.SyncBatchNorm) and _native.sync_group(bn) is not None
    x = case["x"][lo:hi].to(dev).requires_grad_(True)
    if spec["kind"] == "dyn":
        with torch.no_grad():
            ei = m.dilated_knn_graph(x.detach())
        y = m(x)
    else:
        ei = case["edge_index"][:, lo:hi].to(dev)
        y = m(x, ei)
    (y * case["grad_out"][lo:hi].to(dev)).sum().backward()
    got = {"y": y.detach(), "x": x.grad, "weight": gc.nn[0].weight.grad, "bias": gc.nn[0].bias.grad,
           "bn_w": bn.weight.grad, "bn_b": bn.bias.grad, "running_mean": bn.running_mean,
           "running_var": bn.running_var, "num_batches_tracked": bn.num_batches_tracked, "edge_index": ei}
    if isinstance(gc.nn[1], torch.nn.PReLU):
        got["slope"] = gc.nn[1].weight.grad
    out = os.path.join(os.path.dirname(path), "result_%s_%d.pt" % (case["name"], rank))
    torch.save({k: v.detach().cpu() for k, v in got.items()}, out)


def main():
    rank, world, init_file, case_dir = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world)
    try:
        for path in sorted(glob.glob(os.path.join(case_dir, "case_*.pt"))):
            run_case(path, rank, dev)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()
    print("SYNC_BN_WORKER_OK", rank)


if __name__ == "__main__":
    main()
