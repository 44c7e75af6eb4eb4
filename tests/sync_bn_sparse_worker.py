"""One rank of tests/test_sparse_edgeconv_sync_bn_gpu.py's two-rank check:
`python sync_bn_sparse_worker.py RANK WORLD INIT_FILE CASE_DIR`.

Joins a gloo process group through a file store (both ranks may share one GPU: gloo all-reduces CUDA tensors through
host memory), then for every CASE_DIR/case_<name>.pt runs one training step of the converted (SyncBatchNorm)
sparse EdgeConv layer or block on this rank's nodes and writes CASE_DIR/result_<name>_<rank>.pt: output,
x-gradient, LOCAL parameter gradients, running statistics, num_batches_tracked, the batch statistics and moments
the layer normalised with, and the graph it used."""
import datetime
import glob
import os
import sys

import torch
import torch.distributed as dist
from torch import nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def build(spec):
    """(module, its EdgConv) of a case spec; the EdgConv's BatchNorm1d is rebuilt with the spec's options."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    if spec["kind"] == "resdyn":
        mod = S.ResDynBlock(spec["co"], spec["k"], spec["d"], "edge", spec["act"], "batch", res_scale=spec["res_scale"])
        conv = mod.body.gconv
    else:
        mod = conv = S.EdgConv(spec["ci"], spec["co"], spec["act"], "batch", spec["bias"])
    conv.nn[1] = nn.BatchNorm1d(spec["co"], momentum=spec["momentum"], affine=spec["affine"],
                                track_running_stats=spec["track"])
    return mod, conv


def grads_of(conv):
    lin = conv.nn[0]
    g = {"weight": lin.weight.grad}
    if lin.bias is not None:
        g["bias"] = lin.bias.grad
    for m in list(conv.nn)[1:]:
        if isinstance(m, nn.PReLU):
            g["prelu"] = m.weight.grad
        if isinstance(m, nn.SyncBatchNorm) and m.weight is not None:
            g["bn_weight"], g["bn_bias"] = m.weight.grad, m.bias.grad
    return g


def run_case(path, rank, dev):
    from deep_gcns_torch_b200 import _native
    case = torch.load(path)
    spec = case["spec"]
    mod, _ = build(spec)
    mod.load_state_dict(case["state"])
    mod = nn.SyncBatchNorm.convert_sync_batchnorm(mod).to(dev).train()
    conv = mod.body.gconv if spec["kind"] == "resdyn" else mod
    bn = conv.nn[1]
    assert isinstance(bn, nn.SyncBatchNorm) and _native.sync_group(bn) is not None
    seen = []
    conv.register_forward_hook(lambda m, i, o: seen.append(o.grad_fn.prm))
    x = case["x"][rank].to(dev).requires_grad_(True)
    if spec["kind"] == "resdyn":
        batch = case["batch"][rank].to(dev)
        with torch.no_grad():
            ei = mod.body.dilated_knn_graph(x.detach(), batch)
        y = mod(x, batch)[0]
    else:
        ei = case["edge_index"][rank].to(dev)
        y = mod(x, ei)
    (y * case["grad_out"][rank].to(dev)).sum().backward()
    prm = seen[0]
    got = dict(grads_of(conv), y=y.detach(), x=x.grad, edge_index=ei, batch_mean=prm.batch_mean,
               batch_var=prm.batch_var, moments=prm.moments)
    if bn.track_running_stats:
        got.update(running_mean=bn.running_mean, running_var=bn.running_var,
                   num_batches_tracked=bn.num_batches_tracked)
    out = os.path.join(os.path.dirname(path), "result_%s_%d.pt" % (case["name"], rank))
    torch.save({k: v.detach().cpu() for k, v in got.items()}, out)


def main():
    rank, world, init_file, case_dir = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3], sys.argv[4]
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", init_method="file://" + init_file, rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=300))
    try:
        for path in sorted(glob.glob(os.path.join(case_dir, "case_*.pt"))):
            run_case(path, rank, dev)
        torch.cuda.synchronize()
        dist.barrier()
    finally:
        dist.destroy_process_group()
    print("SYNC_BN_SPARSE_WORKER_OK", rank)


if __name__ == "__main__":
    main()
