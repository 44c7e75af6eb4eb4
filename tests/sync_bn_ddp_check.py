"""torchrun entry (one rank per GPU, used by tests/test_sync_bn_gpu.py): one DDP training step of an MRGCN stack
converted with nn.SyncBatchNorm.convert_sync_batchnorm, the batch split evenly over the ranks, against one
single-GPU step of the unconverted model (BatchNorm2d) on the whole batch, run on rank 0: the loss and every
parameter gradient must agree."""
import copy
import os
import sys

import torch
import torch.distributed as dist
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    from bench_models import MRGCN28
    from deep_gcns_torch_b200.gcn_lib import dense as D
    from torch.nn.parallel import DistributedDataParallel as DDP
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    per_rank, points = 2, 1024
    torch.manual_seed(0)
    plain = MRGCN28(D, k=20, n_blocks=6).train()
    g = torch.Generator().manual_seed(1)
    inputs = torch.rand(per_rank * world, 3, points, 1, generator=g)
    labels = torch.randint(0, 40, (per_rank * world,), generator=g)
    conv = torch.nn.SyncBatchNorm.convert_sync_batchnorm(copy.deepcopy(plain)).to(dev)
    ddp = DDP(conv, device_ids=[dev.index])
    sl = slice(rank * per_rank, (rank + 1) * per_rank)
    loss = F.cross_entropy(ddp(inputs[sl].to(dev)), labels[sl].to(dev))
    loss.backward()
    mean_loss = loss.detach().clone()
    dist.all_reduce(mean_loss)
    mean_loss /= world
    grads = [p.grad.detach().clone() for p in conv.parameters()]
    ok = torch.ones(1, device=dev)
    msg = ""
    if rank == 0:
        ref = plain.to(dev)
        ref_loss = F.cross_entropy(ref(inputs.to(dev)), labels.to(dev))
        ref_loss.backward()
        if abs(float(ref_loss) - float(mean_loss)) > 1e-4 * max(1.0, abs(float(ref_loss))):
            ok[0], msg = 0, "loss %.8g vs %.8g" % (float(mean_loss), float(ref_loss))
        for (name, p), got in zip(ref.named_parameters(), grads):
            scale = float(p.grad.abs().max())
            err = float((got - p.grad).abs().max())
            if not err <= 2e-3 * max(scale, 1e-12):
                ok[0], msg = 0, msg + " %s: max err %.3g at scale %.3g;" % (name, err, scale)
        print("rank 0: loss %.8g (ref %.8g) %s" % (float(mean_loss), float(ref_loss), msg))
    dist.broadcast(ok, 0)
    dist.destroy_process_group()
    if ok[0] > 0:
        print("SYNC_BN_DDP_OK")
    else:
        sys.exit(1)


if __name__ == "__main__":
    main()
