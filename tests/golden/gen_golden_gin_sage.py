"""Golden vectors of the sparse-layout GIN and GraphSAGE: the reference's GraphConv with conv = 'gin' / 'sage' /
'rsage' (GinConv and RSAGEConv, gcn_lib/sparse/torch_vertex.py:136-261), its ResGraphBlock / DenseGraphBlock /
DynConv, and the static-graph DeepGCN of examples/ppi/architecture.py, executed unmodified on the unmodified gcn_lib
(loaded through oracle/ref_shims.py, with torch_geometric's GINConv and older SAGEConv restated by
tests/gin_sage_util.py), on seeded synthetic inputs.  Writes only these files:

    spconv_gin_sage         GraphConv(6, 12, conv) for conv in gin / sage / rsage x (relu, no norm) / (leakyrelu,
                            batch eval) / (relu, batch train) on a graph with empty destinations, duplicate edges,
                            self loops (several on one row) and a row of 1100 edges; the train case also after a
                            second step (running statistics)
    spconv_gin_sage_blocks  ResGraphBlock, DenseGraphBlock and DynConv (kNN graph of two clouds) per conv
    spconv_ppi_<conv>       the PPI DeepGCN (16 filters, 3 blocks, res) per conv: eval forward

    DGCN_REFERENCE_ROOT=<reference checkout> python tests/golden/gen_golden_gin_sage.py
"""
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
import gen_golden_models  # noqa: E402
from gen_golden_models import exec_reference, seed_large  # noqa: E402
from gen_golden_spconv_edge import edge_graph  # noqa: E402
import gin_sage_util as gsu  # noqa: E402

CONVS = ("gin", "sage", "rsage")
CASES = (("relu", "none"), ("leakyrelu", "eval"), ("relu", "train"))
PPI_OPT = dict(n_filters=16, act="relu", norm="batch", bias=True, n_heads=1, block="res", n_blocks=3,
               in_channels=50, n_classes=121, dropout=0.0)


def loopy_graph(gen, N, E):
    """edge_graph (empty rows, duplicates, self loops, a 1100-edge row) plus three self loops on node 7."""
    ei = torch.cat((edge_graph(gen, N, E), torch.full((2, 3), 7)), 1)
    return ei[:, torch.randperm(ei.shape[1], generator=gen)].contiguous()


def spconv_gin_sage(sparse, gen):
    N, C, CO = 200, 6, 12
    x = torch.randn(N, C, generator=gen)
    ei = loopy_graph(gen, N, 1500)
    outs, sd, cases, keys = {}, {}, [], {}
    for conv in CONVS:
        for act, norm in CASES:
            name = "%s_%s_%s" % (conv, act, norm)
            torch.manual_seed(len(cases))
            mod = sparse.GraphConv(C, CO, conv, act, None if norm == "none" else "batch", True)
            randomize_norm(mod, gen)
            sd.update({name + "." + k: v.clone() for k, v in mod.state_dict().items()})
            keys[name] = [[k, list(v.shape)] for k, v in mod.state_dict().items()]
            if norm == "train":
                mod.train()
                with torch.no_grad():
                    outs["y_" + name] = mod(x, ei)
                    mod(x, ei)
                bn = next(m for m in mod.modules() if isinstance(m, torch.nn.BatchNorm1d))
                outs["running_mean_" + name] = bn.running_mean.clone()
                outs["running_var_" + name] = bn.running_var.clone()
            else:
                mod.eval()
                with torch.no_grad():
                    outs["y_" + name] = mod(x, ei)
            cases.append(name)
    meta = {"N": N, "C": C, "out": CO, "cases": cases, "state_dict": keys}
    save("spconv_gin_sage", meta, {"x": x, "edge_index": ei.to(torch.int32)}, sd, outs)


def spconv_gin_sage_blocks(sparse, gen):
    B, n, C, k = 2, 64, 8, 6
    x = torch.rand(B * n, C, generator=gen)
    batch = torch.arange(B).repeat_interleave(n)
    ei = loopy_graph(gen, B * n, 600)
    sd, outs = {}, {}
    torch.manual_seed(12)
    for conv in CONVS:
        mods = {"res": sparse.ResGraphBlock(C, conv, "relu", "batch", True, res_scale=0.5),
                "dense": sparse.DenseGraphBlock(C, 4, conv, "leakyrelu", "batch", True),
                "dyn": sparse.DynConv(C, C, k, 1, conv, "relu", "batch", True)}
        with torch.no_grad():
            for name, mod in mods.items():
                randomize_norm(mod, gen)
                mod.eval()
                sd.update({"%s_%s.%s" % (conv, name, key): v.clone() for key, v in mod.state_dict().items()})
            outs["y_%s_res" % conv] = mods["res"](x, ei)[0]
            outs["y_%s_dense" % conv] = mods["dense"](x, ei)[0]
            outs["y_%s_dyn" % conv] = mods["dyn"](x, batch)
    outs["graph_dyn"] = sparse.DilatedKnnGraph(k, 1)(x, batch).to(torch.int32)
    meta = {"B": B, "n": n, "C": C, "k": k, "convs": list(CONVS)}
    save("spconv_gin_sage_blocks", meta, {"x": x, "batch": batch.to(torch.int32), "edge_index": ei.to(torch.int32)},
         sd, outs)


def spconv_ppi(gen):
    ns = exec_reference("examples/ppi/architecture.py", "ref_ppi")
    N = 90
    x = torch.randn(N, PPI_OPT["in_channels"], generator=gen)
    ei = loopy_graph(gen, N, 500)
    ei = ei[:, ei[1] != 5]                 # edge_graph's 1100-edge row is for the layer goldens only
    for i, conv in enumerate(CONVS):
        torch.manual_seed(100 + i)
        opt = dict(PPI_OPT, conv=conv)
        model = ns["DeepGCN"](types.SimpleNamespace(**opt))
        randomize_norm(model, gen)
        meta = seed_large(model, dict(opt, N=N))
        model.eval()
        with torch.no_grad():
            y = model(types.SimpleNamespace(x=x, edge_index=ei, batch=None))
        sd = {k: v.clone() for k, v in model.state_dict().items() if k not in meta["seeded"]}
        meta["state_dict"] = [[k, list(v.shape)] for k, v in model.state_dict().items()]
        save("spconv_ppi_" + conv, meta, {"x": x, "edge_index": ei.to(torch.int32)}, sd, {"y": y})


def main():
    torch.set_num_threads(8)
    gen_golden_models.SEEDED_MIN = 4096     # the PPI heads' Linear weights are drawn from seeds, not stored
    gsu.install_reference_stand_ins()
    _, sparse = ref_shims.load_reference()
    gen = torch.Generator().manual_seed(2025)
    spconv_gin_sage(sparse, gen)
    spconv_gin_sage_blocks(sparse, gen)
    spconv_ppi(gen)


if __name__ == "__main__":
    main()
