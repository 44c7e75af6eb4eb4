"""Microbenchmark of the pieces of one DeeperGCN res+ layer at the arxiv shape (N=169343, C=128):
aggregate with / without the fused pre-activation, Linear variants for the skip connection."""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_gcns_torch_b200 import _native  # noqa: E402
from oracle import sparse as osp  # noqa: E402


def timeit(fn, n=30):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    b.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return b.elapsed_time(e) / n


def main():
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    N, C = 169343, 128
    s, d = torch.randint(0, N, (1166243,), generator=g), torch.randint(0, N, (1166243,), generator=g)
    ei = osp.to_undirected_with_self_loops(s, d, N).to(dev)
    h = torch.randn(N, C, generator=g).to(dev)
    csr = _native.csr_build(ei, N)
    prm, _k = _native.genconv_params("softmax_sg", 0.1, 1.0, 0.0, 1e-7, None, add_residual=True)
    sc, sh = torch.rand(C, device=dev) + 0.5, torch.randn(C, device=dev) * 0.1
    lin = torch.nn.Linear(C, C).to(dev)
    bn = torch.nn.BatchNorm1d(C).to(dev).eval()
    a = torch.empty_like(h)
    out = torch.empty_like(h)
    res = {}
    with torch.no_grad():
        res["aggregate_plain_ms"] = timeit(lambda: _native.genconv_aggregate(h, h, csr, prm, out=a))
        res["aggregate_pre_ms"] = timeit(lambda: _native.genconv_aggregate(h, h, csr, prm, out=a, pre=(sc, sh, True)))
        res["bn_relu_ms"] = timeit(lambda: F.relu(bn(h)))
        res["linear_ms"] = timeit(lambda: lin(a))
        res["linear_plus_add_ms"] = timeit(lambda: lin(a) + h)
        res["addmm_beta_ms"] = timeit(lambda: torch.addmm(h, a, lin.weight.t(), out=out))
        res["addmm_beta_bias_ms"] = timeit(lambda: torch.addmm(h, a, lin.weight.t(), out=out).add_(lin.bias))
        res["linear_out_add_ms"] = timeit(lambda: F.linear(a, lin.weight, lin.bias).add_(h))
        res["tc_linear_residual_ms"] = timeit(lambda: _native.linear_residual(a, lin.weight, lin.bias, h, out=out))
        _native.kernel_timing(True)
        _native.kernel_timing_read("linear")
        for _ in range(10):
            _native.linear_residual(a, lin.weight, lin.bias, h, out=out)
        ms, n = _native.kernel_timing_read("linear")
        _native.kernel_timing(False)
        res["tc_linear_kernel_ms"] = ms / max(n, 1)
        res["tc_linear_hbm_gbs"] = 3 * N * C * 4 / (ms / max(n, 1) * 1e-3) / 1e9
    print(json.dumps(res))


if __name__ == "__main__":
    main()
