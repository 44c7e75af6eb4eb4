"""torchrun entry (one rank per GPU, used by tests/test_sparse_half_gpu.py): HaloExchange + PartitionedAggregate on
bf16 rows across the ranks against the single-GPU layer on the whole graph, forward and backward."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=dev)
    from deep_gcns_torch_b200 import partition as P
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    g = torch.Generator().manual_seed(0)
    N, E, C = 20011, 300000, 128
    ei = torch.randint(0, N, (2, E), generator=g)
    ei[1, :5000] = 17
    x0 = torch.randn(N, C, generator=g).to(torch.bfloat16).to(dev)
    wgt = torch.randn(N, C, generator=g).to(dev)
    part = P.GraphPartition(ei.to(dev), N, rank, world, device=dev).exchange_halo_lists()
    lo, hi = part.lo, part.hi
    eps = torch.finfo(torch.bfloat16).eps
    for aggr in ("softmax", "power", "max"):
        torch.manual_seed(1)
        conv = S.GENConv(C, C, aggr=aggr, t=0.1, learn_t=True, p=2.0, msg_norm=True, mlp_layers=1,
                         norm="layer").to(dev)
        x = x0.clone().requires_grad_(True)
        full = conv.propagate(ei.to(dev), x=x, msg_scale=conv.msg_norm.msg_scale, residual=True)
        (full * wgt).sum().backward()
        x_local = x0[lo:hi].clone().requires_grad_(True)
        x_src = P.HaloExchange.apply(x_local, part, None)
        assert x_src.dtype == torch.bfloat16
        t, p, y = conv._scalars()
        out = P.PartitionedAggregate.apply(x_src, x_local, part, conv._check_aggr(), conv.eps, True, t, p, y,
                                           conv.msg_norm.msg_scale)
        assert torch.equal(out, full[lo:hi]), aggr
        (out * wgt[lo:hi]).sum().backward()
        want = x.grad[lo:hi].double()
        err = float((x_local.grad.double() - want).abs().max() / want.abs().max())
        assert x_local.grad.dtype == torch.bfloat16 and err <= 4 * eps, (aggr, err)
    dist.barrier()
    if rank == 0:
        print("HALO_HALF_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
