"""Golden vectors of the sparse-layout EdgeConv: the reference's EdgConv (gcn_lib/sparse/torch_vertex.py:106-114), its
GraphConv / DynConv / *DynBlock with conv='edge', and its SparseDeepGCN (examples/sem_seg_sparse/architecture.py),
executed unmodified on the unmodified gcn_lib (loaded through oracle/ref_shims.py, with torch_geometric's EdgeConv
restated by tests/sparse_edge_util.py), on seeded synthetic inputs.  Writes only these files:

    spconv_edge         EdgConv on a graph with empty destinations, duplicate edges, self-loops and a row of more
                        than 1024 edges: relu / leakyrelu / prelu (weight > 0 and < 0) x norm None / batch eval /
                        batch train (output, batch statistics, running statistics after two steps)
    spconv_edge_blocks  GraphConv head, DynConv, Res / Dense / PlainDynBlock('edge') over two equally sized clouds
    model_sparse_deepgcn  SparseDeepGCN, 2 clouds x 96 points, k = 4, 16 filters, 4 res blocks: eval forward block by
                        block, one train-mode forward + backward (parameter and input gradients)

    DGCN_REFERENCE_ROOT=<reference checkout> python tests/golden/gen_golden_spconv_edge.py
"""
import inspect
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_shims  # noqa: E402
from gen_golden import randomize_norm, save  # noqa: E402
from gen_golden_models import exec_reference, seed_large  # noqa: E402
import sparse_edge_util as seu  # noqa: E402

ACTS = (("relu", None), ("leakyrelu", None), ("prelu", 0.25), ("prelu", -0.3))
NORMS = ("none", "eval", "train")
TIE_REL, KINK_REL = 2e-5, 2e-6    # model golden: the seed is chosen so that no max is this close to a tie or kink


def signature(cls):
    return [[p.name, p.default if p.default is not inspect.Parameter.empty else "<empty>"]
            for p in inspect.signature(cls.__init__).parameters.values()]


def edge_graph(gen, N, E):
    """Random edges into N - 40 destinations (the last 40 nodes have no in-edges), 1100 more into node 5, 60
    duplicated edges and 30 self-loops, in random order."""
    src = torch.randint(0, N, (E,), generator=gen)
    dst = torch.randint(0, N - 40, (E,), generator=gen)
    hub = torch.stack((torch.randint(0, N, (1100,), generator=gen), torch.full((1100,), 5)))
    ei = torch.cat((torch.stack((src, dst)), hub), 1)
    dup = ei[:, torch.randint(0, ei.shape[1], (60,), generator=gen)]
    loops = torch.randint(0, N - 40, (30,), generator=gen).repeat(2, 1)
    ei = torch.cat((ei, dup, loops), 1)
    return ei[:, torch.randperm(ei.shape[1], generator=gen)].contiguous()


def spconv_edge(sparse, gen):
    N, C, CO = 200, 6, 36
    x = torch.randn(N, C, generator=gen)
    ei = edge_graph(gen, N, 1500)
    outs, sd, cases = {}, {}, []
    for act, slope in ACTS:
        for norm in NORMS:
            name = "%s%s_%s" % (act, "" if slope is None else ("_pos" if slope > 0 else "_neg"), norm)
            torch.manual_seed(len(cases))
            mod = sparse.EdgConv(C, CO, act, None if norm == "none" else "batch", True)
            randomize_norm(mod, gen)
            with torch.no_grad():
                mod.nn[0].bias.copy_(torch.randn(CO, generator=gen) * 0.1)
                for m in mod.modules():
                    if isinstance(m, torch.nn.PReLU):
                        m.weight.fill_(slope)
            sd.update({name + "." + k: v.clone() for k, v in mod.state_dict().items()})
            if norm == "train":
                mod.train()
                bn = mod.nn[1]
                seen = []
                h = bn.register_forward_hook(lambda m, i, o: seen.append(i[0].detach().clone()))
                with torch.no_grad():
                    outs["y_" + name] = mod(x, ei)
                    mod(x, ei)
                h.remove()
                outs["mean_" + name] = seen[0].mean(0)
                outs["var_" + name] = seen[0].var(0, unbiased=False)
                outs["running_mean_" + name] = bn.running_mean.clone()
                outs["running_var_" + name] = bn.running_var.clone()
            else:
                mod.eval()
                with torch.no_grad():
                    outs["y_" + name] = mod(x, ei)
            cases.append(name)
    meta = {"N": N, "C": C, "out": CO, "cases": cases, "signature_EdgConv": signature(sparse.EdgConv)}
    save("spconv_edge", meta, {"x": x, "edge_index": ei.to(torch.int32)}, sd, outs)


def spconv_edge_blocks(sparse, gen):
    B, n, C0, C, k, d = 2, 96, 6, 16, 4, 2
    x0 = torch.rand(B * n, C0, generator=gen)
    batch = torch.arange(B).repeat_interleave(n)
    torch.manual_seed(11)
    mods = {
        "head": sparse.GraphConv(C0, C, "edge", "relu", "batch", True),
        "dyn": sparse.DynConv(C, C, k, d, "edge", "leakyrelu", "batch", True),
        "res": sparse.ResDynBlock(C, k, d, "edge", "relu", "batch", True, res_scale=0.5),
        "dense": sparse.DenseDynBlock(C, 8, k, d, "edge", "prelu", "batch", True),
        "plain": sparse.PlainDynBlock(C, k, 1, "edge", "relu", None, True),
    }
    sd, outs = {}, {}
    head_graph = sparse.DilatedKnnGraph(k, 1)(x0[:, :3], batch)
    with torch.no_grad():
        for name, mod in mods.items():
            randomize_norm(mod, gen)
            mod.eval()
            sd.update({name + "." + key: v.clone() for key, v in mod.state_dict().items()})
        h = mods["head"](x0, head_graph)
        outs["y_head"] = h
        outs["graph_head"] = head_graph.to(torch.int32)
        for name in ("dyn", "res", "dense", "plain"):
            mod = mods[name]
            body = mod if name == "dyn" else mod.body
            outs["graph_" + name] = body.dilated_knn_graph(h, batch).to(torch.int32)
            y = mod(h, batch)
            outs["y_" + name] = y[0] if isinstance(y, tuple) else y
    meta = {"B": B, "n": n, "C0": C0, "C": C, "k": k, "dilation": d}
    save("spconv_edge_blocks", meta, {"x": x0, "batch": batch.to(torch.int32)}, sd, outs)


def near_ties(model, x, batch):
    """Number of (node, channel) maxima of the model's EdgConv layers within TIE_REL of a tie (outside ReLU's flat
    part) or whose winning edge is within KINK_REL of the kink, recomputed in fp64 from each layer's input."""
    convs = [model.head.gconv] + [blk.body.gconv for blk in model.backbone]
    graphs = [model.knn] + [blk.body.dilated_knn_graph for blk in model.backbone]
    inputs, eis, handles = [], [], []
    for c, g in zip(convs, graphs):
        handles.append(c.register_forward_hook(lambda m, i, o: inputs.append(i[0].detach().clone())))
        handles.append(g.register_forward_hook(lambda m, i, o: eis.append(o.detach().clone())))
    with torch.no_grad():
        model(types.SimpleNamespace(pos=x[:, :3], x=x[:, 3:], batch=batch))
    for h in handles:
        h.remove()
    return sum(int(seu.edge_tie_mask(c.nn, h, e, TIE_REL, KINK_REL, training=True).sum())
               for c, h, e in zip(convs, inputs, eis))


def model_sparse_deepgcn(gen):
    ns = exec_reference("examples/sem_seg_sparse/architecture.py", "ref_semseg_sparse")
    opt = dict(n_filters=16, k=4, act="relu", norm="batch", bias=True, epsilon=0.2, stochastic=False, conv="edge",
               n_blocks=4, block="res", in_channels=9, n_classes=13, dropout=0.0)
    B, n = 2, 96
    batch = torch.arange(B).repeat_interleave(n)
    for seed in range(50):
        torch.manual_seed(seed)
        model = ns["SparseDeepGCN"](types.SimpleNamespace(**opt))
        randomize_norm(model, gen)
        meta = seed_large(model, dict(opt, B=B, N=n, seed=seed))
        pos, color = torch.rand(B * n, 3, generator=gen), torch.rand(B * n, 6, generator=gen)
        if near_ties(model.train(), torch.cat((pos, color), 1), batch) == 0:
            break
    else:
        raise RuntimeError("no seed without near-ties")
    model.eval()
    feats, graphs, handles = [], [], []
    handles.append(model.head.register_forward_hook(lambda m, i, o: feats.append(o.detach().clone())))
    handles.append(model.knn.register_forward_hook(lambda m, i, o: graphs.append(o.to(torch.int32).clone())))
    for blk in model.backbone:
        handles.append(blk.register_forward_hook(lambda m, i, o: feats.append(o[0].detach().clone())))
        handles.append(blk.body.dilated_knn_graph.register_forward_hook(
            lambda m, i, o: graphs.append(o.to(torch.int32).clone())))
    data = types.SimpleNamespace(pos=pos, x=color, batch=batch)
    with torch.no_grad():
        y = model(data)
    for h in handles:
        h.remove()
    outs = {"y": y}
    for i, (f, g) in enumerate(zip(feats, graphs)):
        outs["feat%d" % i], outs["graph%d" % i] = f, g
    # one train-mode step: forward, backward of sum(y * w)
    sd = {k: v.clone() for k, v in model.state_dict().items() if k not in meta["seeded"]}
    model.train()
    pos_g, color_g = pos.clone().requires_grad_(True), color.clone().requires_grad_(True)
    y = model(types.SimpleNamespace(pos=pos_g, x=color_g, batch=batch))
    w = torch.randn(y.shape, generator=gen)
    (y * w).sum().backward()
    outs["y_train"], outs["grad_w"] = y.detach(), w
    outs["grad_pos"], outs["grad_color"] = pos_g.grad, color_g.grad
    for name, p in model.named_parameters():
        outs["grad." + name] = p.grad if name not in meta["seeded"] else p.grad.sum(1)
    save("model_sparse_deepgcn", meta, {"pos": pos, "color": color, "batch": batch.to(torch.int32)}, sd, outs)


def main():
    torch.set_num_threads(8)
    seu.install_reference_stand_ins()
    _, sparse = ref_shims.load_reference()
    gen = torch.Generator().manual_seed(2024)
    spconv_edge(sparse, gen)
    spconv_edge_blocks(sparse, gen)
    model_sparse_deepgcn(gen)


if __name__ == "__main__":
    main()
