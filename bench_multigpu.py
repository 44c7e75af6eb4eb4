"""Multi-GPU blocks of bench.py (run when WORLD_SIZE > 1, OUTSIDE the headline's timed regions; their results
go into the JSON line's `extra`):

  sparse_halo  BASELINE config 5: node-partitioned DeeperGCN GENConv stack (res+, softmax_sg t=0.1, C=128) on
               a synthetic ogbn-products-shaped graph (N = 2,449,029, E = 61,859,140), one NCCL halo
               all-to-all per layer overlapped with the interior rows; block-structured AND uniform variants;
               parity against the single-GPU full-graph forward on a row sample.
  ddp_mrgcn    BASELINE config 4: one data-parallel MRGCN-28 training step (forward + backward + SGD),
               B = 64 clouds sharded over the ranks, weight-gradient all-reduce by torch DDP over NCCL.

Synthetic graphs (SURVEY.md 8d): every rank draws the edges whose TARGET it owns on its own device from a
per-rank seed.  'uniform': sources uniform over all nodes (worst-case halo: nearly every remote node).
'block': nodes v with v % 4 == 0 are boundary-type; 40 % of the in-edges of a boundary-type target come from
boundary-type nodes anywhere in the graph, every other edge stays inside the target's partition block - a
10 % edge cut concentrated on a quarter of the rows, the shape a locality-aware ordering (partition.bfs_order
on a graph with geometric locality, or a METIS partition) leaves behind.
"""
import time

import torch
import torch.distributed as dist
import torch.nn.functional as F

PRODUCTS_N, PRODUCTS_E, HIDDEN = 2449029, 61859140, 128


def local_edges(num_nodes, num_edges, rank, world, kind, dev, seed=0):
    """(src, dst) global ids of the edges whose target lies in rank's row range, drawn on `dev`."""
    from deep_gcns_torch_b200.partition import row_ranges
    lo, hi = row_ranges(num_nodes, world)[rank]
    e_lo, e_hi = row_ranges(num_edges, world)[rank]
    n_e = e_hi - e_lo
    g = torch.Generator(device=dev).manual_seed(1000 * seed + 17 * world + rank)
    dst = torch.randint(lo, hi, (n_e,), generator=g, device=dev)
    if kind == "uniform":
        src = torch.randint(0, num_nodes, (n_e,), generator=g, device=dev)
    else:
        inside = torch.randint(lo, hi, (n_e,), generator=g, device=dev)
        far = torch.randint(0, num_nodes // 4, (n_e,), generator=g, device=dev) * 4
        cross = ((dst % 4) == 0) & (torch.rand(n_e, generator=g, device=dev) < 0.4)
        src = torch.where(cross, far, inside)
    return src, dst


def local_features(num_nodes, rank, world, channels, dev, seed=0):
    from deep_gcns_torch_b200.partition import row_ranges
    lo, hi = row_ranges(num_nodes, world)[rank]
    g = torch.Generator(device=dev).manual_seed(5000 * seed + 31 * world + rank)
    return torch.randn(hi - lo, channels, generator=g, device=dev)


def _ev():
    return torch.cuda.Event(enable_timing=True)


def _time_ms(fn, reps, sync):
    """Device time of `reps` calls of fn (CUDA events on the current stream), max over ranks."""
    fn()
    sync()
    b, e = _ev(), _ev()
    b.record()
    for _ in range(reps):
        fn()
    e.record()
    sync()
    t = torch.tensor([b.elapsed_time(e) / reps], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def sparse_halo_block(dev, rank, world, layers=112, parity_layers=4, num_nodes=PRODUCTS_N, num_edges=PRODUCTS_E,
                      sample_rows=4096):
    from bench_models import DeeperGCN
    from deep_gcns_torch_b200 import _native, partition as P
    from deep_gcns_torch_b200.gcn_lib import sparse as S

    def sync():
        dist.barrier()
        torch.cuda.synchronize()

    out = {"model": "DeeperGCN res+ GENConv(softmax_sg, t=0.1, mlp_layers=1) x %d, C=%d" % (layers, HIDDEN),
           "N": num_nodes, "E": num_edges, "partition": "contiguous destination-row ranges x%d" % world}
    torch.manual_seed(0)
    model = DeeperGCN(S, layers=layers, hidden=HIDDEN, in_channels=HIDDEN, tasks=40).to(dev).eval()
    halo_group = P.high_priority_group()          # the exchange must not queue behind the aggregate's CTAs
    for kind in ("block", "uniform"):
        src, dst = local_edges(num_nodes, num_edges, rank, world, kind, dev)
        t0 = time.perf_counter()
        part = P.GraphPartition.from_local_edges(src, dst, num_nodes, rank, world, dev).exchange_halo_lists(halo_group)
        part.csr()
        torch.cuda.synchronize()
        build_ms = (time.perf_counter() - t0) * 1e3
        x_local = local_features(num_nodes, rank, world, HIDDEN, dev)
        C = HIDDEN
        conv, norm = model.gcns[1], model.norms[0]
        from deep_gcns_torch_b200.gcn_lib.sparse.fused import bn_eval_affine
        pre = bn_eval_affine(norm) + (True,)
        part.local_rows(C, 0).copy_(x_local)
        a = torch.empty(part.n_local, C, device=dev)
        with torch.no_grad():
            # one layer's pieces, each timed alone, then the overlapped layer
            def exchange_only():
                w = P.start_halo_exchange(part, C, 0)
                if w is not None:
                    w.wait()
            t, p, y = conv._scalars()
            prm, _k = _native.genconv_params(conv._check_aggr(), t, p, y, conv.eps, None, add_residual=True)
            xbuf = part.buffers(C, 0)[0]

            def aggregate_only():
                _native.genconv_aggregate(xbuf, xbuf[:part.n_local], part.csr(), prm, out=a, pre=pre)
            a2a_ms = _time_ms(exchange_only, 10, sync)
            aggregate_ms = _time_ms(aggregate_only, 10, sync)
            layer_ms = _time_ms(lambda: P.aggregate_partitioned(conv, part, C, 0, pre=pre, out=a), 10, sync)
            serial_ms = _time_ms(lambda: P.aggregate_partitioned(conv, part, C, 0, pre=pre, out=a, overlap=False), 10,
                                 sync)
            # the whole stack: aggregate + Linear + skip per layer, as the model runs it
            model_ms = _time_ms(lambda: model.forward_partitioned(x_local, part), 2, sync)
            # ---- parity: first `parity_layers` layers against the single-GPU full-graph forward -----------
            h_part = model.forward_partitioned(x_local, part, layers=parity_layers, head=False).clone()   # (a view of the persistent buffer)
            finite = bool(torch.isfinite(model.forward_partitioned(x_local, part)).all())
            g = torch.Generator(device=dev).manual_seed(99)
            rows = torch.randint(0, part.n_local, (sample_rows,), generator=g, device=dev)
            mine = h_part[rows].contiguous()
            gathered = [torch.empty_like(mine) for _ in range(world)] if rank == 0 else None
            dist.gather(mine, gathered, dst=0)
            row_ids = [torch.empty_like(rows) for _ in range(world)] if rank == 0 else None
            dist.gather(rows + part.lo, row_ids, dst=0)
            ok = torch.ones(1, device=dev)
            max_rel = 0.0
            if rank == 0:
                srcs, dsts, xs = [], [], []
                for r in range(world):
                    s_r, d_r = local_edges(num_nodes, num_edges, r, world, kind, dev)
                    srcs.append(s_r)
                    dsts.append(d_r)
                    xs.append(local_features(num_nodes, r, world, HIDDEN, dev))
                ei = torch.stack((torch.cat(srcs), torch.cat(dsts)))
                del srcs, dsts
                x_full = torch.cat(xs)
                del xs
                h = model.gcns[0](model.enc(x_full), ei)
                for l in range(1, parity_layers):
                    h = model.gcns[l](F.relu(model.norms[l - 1](h)), ei) + h        # the unfused module sequence
                ref = h[torch.cat(row_ids)]
                got = torch.cat(gathered)
                max_rel = float(((got - ref).abs() / (1e-4 + 1e-3 * ref.abs())).max())   # <= 1 passes rtol 1e-3 / atol 1e-4
                ok[0] = 1.0 if torch.allclose(got, ref, rtol=1e-3, atol=1e-4) else 0.0
                full_csr = _native.csr_build(ei, num_nodes)
                t0_ = _ev(); t1_ = _ev()
                _native.genconv_aggregate(x_full, x_full, full_csr, prm, pre=pre)
                torch.cuda.synchronize()
                t0_.record()
                for _ in range(5):
                    _native.genconv_aggregate(x_full, x_full, full_csr, prm, pre=pre)
                t1_.record()
                torch.cuda.synchronize()
                single_ms = t0_.elapsed_time(t1_) / 5
                del ei, x_full, h, full_csr
                torch.cuda.empty_cache()
            else:
                single_ms = 0.0
            dist.broadcast(ok, 0)
        stats = torch.tensor([part.n_halo, part.interior_rows.numel(), part.n_remote_edges, part.n_local,
                              int(part.send_rows.numel())], dtype=torch.float64, device=dev)
        smax = stats.clone()
        dist.all_reduce(stats)
        dist.all_reduce(smax, op=dist.ReduceOp.MAX)
        hidden = max(0.0, min(1.0, (a2a_ms + aggregate_ms - layer_ms) / max(min(a2a_ms, aggregate_ms), 1e-9)))
        out[kind] = {
            "ms_per_layer": layer_ms, "edges_per_s": num_edges / (layer_ms * 1e-3),
            "ms_per_layer_serial": serial_ms, "a2a_ms": a2a_ms, "aggregate_ms": aggregate_ms,
            "overlap_frac": hidden,
            "overlap_note": "(a2a_ms + aggregate_ms - ms_per_layer) / min(a2a_ms, aggregate_ms): share of the shorter "
                            "phase hidden behind the longer one",
            "model_ms": model_ms, "model_layers": layers, "model_edges_per_s": layers * num_edges / (model_ms * 1e-3),
            "model_output_finite": finite,
            "halo_rows": int(stats[0]), "halo_rows_max_rank": int(smax[0]),
            "halo_bytes": int(stats[0]) * HIDDEN * 4, "nvlink_bytes_per_layer": int(stats[4]) * HIDDEN * 4,
            "halo_vs_allgather": float(stats[0]) / (num_nodes * (world - 1)),
            "interior_row_frac": float(stats[1]) / float(stats[3]), "cut_edge_frac": float(stats[2]) / num_edges,
            "partition_build_ms": build_ms, "single_gpu_aggregate_ms": single_ms,
            "vs_single_gpu_over_world": (layer_ms / (single_ms / world)) if single_ms else None,
            "parity_ok": bool(ok[0] > 0), "parity_layers": parity_layers, "parity_rows": sample_rows * world,
            "parity_max_scaled_err": max_rel,
            "parity_note": "first %d layers, partitioned fused path vs single-GPU unfused full-graph modules on rank 0, "
                           "rtol 1e-3 atol 1e-4" % parity_layers,
        }
        if rank == 0 and single_ms:
            out[kind]["vs_single_gpu_over_world"] = layer_ms / (single_ms / world)
        del part, src, dst, x_local, a
        torch.cuda.empty_cache()
    return out


def ddp_mrgcn_block(dev, rank, world, global_batch=64, points=1024, k=20, sync_bn=False):
    """sync_bn: convert the model with nn.SyncBatchNorm.convert_sync_batchnorm, so every BatchNorm normalises over
    the whole global batch (two small all-reduces per graph convolution, forward and backward, plus torch's own for
    the tail's norms); otherwise each replica normalises over its own shard, as DataParallel does."""
    from bench_models import MRGCN28
    from deep_gcns_torch_b200.gcn_lib import dense as D
    from torch.nn.parallel import DistributedDataParallel as DDP

    def sync():
        dist.barrier()
        torch.cuda.synchronize()

    per_rank = global_batch // world
    torch.manual_seed(0)
    model = MRGCN28(D, k=k)
    if sync_bn:
        model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)
    model = model.to(dev).train()
    ddp = DDP(model, device_ids=[dev.index], broadcast_buffers=False)      # BN running statistics stay per replica
    g = torch.Generator().manual_seed(100 + rank)
    inputs = torch.rand(per_rank, 3, points, 1, generator=g).to(dev)
    labels = torch.randint(0, 40, (per_rank,), generator=g).to(dev)
    opt = torch.optim.SGD(ddp.parameters(), lr=0.0)                         # lr 0: repeated steps see the same weights

    def step(sync_grads=True):
        opt.zero_grad(set_to_none=True)
        if sync_grads:
            loss = F.cross_entropy(ddp(inputs), labels)
            loss.backward()
        else:
            with ddp.no_sync():
                loss = F.cross_entropy(ddp(inputs), labels)
                loss.backward()
        opt.step()
        return loss
    loss0 = float(step())
    # parity of the collective: DDP's averaged gradients == mean over ranks of the local gradients
    step(sync_grads=False)
    local = torch.cat([p.grad.flatten() for p in model.parameters() if p.grad is not None])
    dist.all_reduce(local)
    local /= world
    step(sync_grads=True)
    synced = torch.cat([p.grad.flatten() for p in model.parameters() if p.grad is not None])
    scale = float(local.abs().max())
    err = float((synced - local).abs().max())
    ok = bool(err <= 1e-4 * max(scale, 1e-30) + 1e-9) and bool(torch.isfinite(synced).all())
    step_ms = _time_ms(step, 3, sync)
    nosync_ms = _time_ms(lambda: step(False), 3, sync)
    flat = torch.empty_like(local)
    allreduce_ms = _time_ms(lambda: dist.all_reduce(flat), 5, sync)
    edges = 28 * global_batch * points * k
    return {"model": "MRGCN-28 (modelnet_cls DeepGCN, conv=mr, k=%d, dilation 1..27), fwd + bwd + SGD, train-mode BN" % k,
            "sync_bn": bool(sync_bn), "global_batch": global_batch, "per_rank_batch": per_rank, "points": points,
            "step_ms": step_ms, "step_ms_without_allreduce": nosync_ms, "allreduce_ms": allreduce_ms,
            "allreduce_exposed_ms": max(0.0, step_ms - nosync_ms), "grad_bytes": int(local.numel()) * 4,
            "edges_per_s_fwd_bwd": edges / (step_ms * 1e-3), "first_loss": loss0,
            "parity_ok": ok, "parity_note": "DDP gradients vs the mean over ranks of no_sync() local gradients, max abs "
                                            "err %.3g at scale %.3g" % (err, scale)}
