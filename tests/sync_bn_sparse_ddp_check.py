"""torchrun entry (one rank per GPU, used by tests/test_sparse_edgeconv_sync_bn_gpu.py): one DDP training step of the
drop-in SparseDeepGCN (examples/sem_seg_sparse, conv 'edge', norm 'batch') converted with
nn.SyncBatchNorm.convert_sync_batchnorm, the clouds split evenly over the ranks, against one single-GPU step of the
unconverted model (BatchNorm1d) on the whole batch, run on rank 0: the loss and every parameter gradient must
agree."""
import copy
import os
import sys
import types

import torch
import torch.distributed as dist
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    from test_sparse_edgeconv_gpu import SparseDeepGCN
    from torch.nn.parallel import DistributedDataParallel as DDP
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    per_rank, points = 2, 1024
    opt = types.SimpleNamespace(in_channels=9, n_filters=32, k=16, n_blocks=4, conv="edge", act="relu", norm="batch",
                                bias=True, n_classes=13, dropout=0.0, stochastic=False, epsilon=0.2)
    torch.manual_seed(0)
    plain = SparseDeepGCN(opt).train()
    g = torch.Generator().manual_seed(1)
    B = per_rank * world
    pos, color = torch.rand(B * points, 3, generator=g), torch.rand(B * points, 6, generator=g)
    labels = torch.randint(0, opt.n_classes, (B * points,), generator=g)
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain)).to(dev)
    ddp = DDP(conv, device_ids=[dev.index])
    sl = slice(rank * per_rank * points, (rank + 1) * per_rank * points)
    batch = torch.arange(per_rank, device=dev).repeat_interleave(points)
    loss = F.cross_entropy(ddp(pos[sl].to(dev), color[sl].to(dev), batch, per_rank), labels[sl].to(dev))
    loss.backward()
    mean_loss = loss.detach().clone()
    dist.all_reduce(mean_loss)
    mean_loss /= world
    grads = [p.grad.detach().clone() for p in conv.parameters()]
    ok = torch.ones(1, device=dev)
    msg = ""
    if rank == 0:
        ref = plain.to(dev)
        full = torch.arange(B, device=dev).repeat_interleave(points)
        ref_loss = F.cross_entropy(ref(pos.to(dev), color.to(dev), full, B), labels.to(dev))
        ref_loss.backward()
        if abs(float(ref_loss) - float(mean_loss)) > 1e-4 * max(1.0, abs(float(ref_loss))):
            ok[0], msg = 0, "loss %.8g vs %.8g" % (float(mean_loss), float(ref_loss))
        ref_grads = dict(ref.named_parameters())
        for (name, p), got in zip(ref.named_parameters(), grads):
            scale = float(p.grad.abs().max())
            if name.endswith(".0.bias") and "prediction.2" not in name:
                # a Linear's bias in front of a train-mode BatchNorm has a gradient that cancels to 0
                scale = max(scale, float(ref_grads[name[:-len("bias")] + "weight"].grad.abs().max()))
            err = float((got - p.grad).abs().max())
            if not err <= 2e-3 * max(scale, 1e-12):
                ok[0], msg = 0, msg + " %s: max err %.3g at scale %.3g;" % (name, err, scale)
        print("rank 0: loss %.8g (ref %.8g) %s" % (float(mean_loss), float(ref_loss), msg))
    dist.broadcast(ok, 0)
    dist.destroy_process_group()
    if ok[0] > 0:
        print("SYNC_BN_SPARSE_DDP_OK")
    else:
        sys.exit(1)


if __name__ == "__main__":
    main()
