"""Golden vector of the PPI DeepGCN with MRConv, the model examples/ppi/opt.py builds by default (conv='mr'): the
static-graph DeepGCN of examples/ppi/architecture.py with gen_golden_gin_sage.PPI_OPT's shape (16 filters, 3 res
blocks), executed unmodified on the unmodified gcn_lib (loaded through oracle/ref_shims.py, as
gen_golden_gin_sage.py does), eval forward on a seeded graph with empty destinations, duplicate edges and self loops.
Writes only this file:

    spconv_ppi_mr

    DGCN_REFERENCE_ROOT=<reference checkout> python tests/golden/gen_golden_ppi_mr.py
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
from gen_golden_gin_sage import PPI_OPT, loopy_graph  # noqa: E402
import gin_sage_util as gsu  # noqa: E402


def main():
    torch.set_num_threads(8)
    gen_golden_models.SEEDED_MIN = 4096     # the PPI heads' Linear weights are drawn from seeds, not stored
    gsu.install_reference_stand_ins()
    ref_shims.load_reference()
    ns = exec_reference("examples/ppi/architecture.py", "ref_ppi")
    gen = torch.Generator().manual_seed(2026)
    N = 90
    x = torch.randn(N, PPI_OPT["in_channels"], generator=gen)
    ei = loopy_graph(gen, N, 500)
    ei = ei[:, ei[1] != 5]                 # edge_graph's 1100-edge row is for the layer goldens only
    torch.manual_seed(103)
    opt = dict(PPI_OPT, conv="mr")
    model = ns["DeepGCN"](types.SimpleNamespace(**opt))
    randomize_norm(model, gen)
    meta = seed_large(model, dict(opt, N=N))
    model.eval()
    with torch.no_grad():
        y = model(types.SimpleNamespace(x=x, edge_index=ei, batch=None))
    sd = {k: v.clone() for k, v in model.state_dict().items() if k not in meta["seeded"]}
    meta["state_dict"] = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    save("spconv_ppi_mr", meta, {"x": x, "edge_index": ei.to(torch.int32)}, sd, {"y": y})


if __name__ == "__main__":
    main()
