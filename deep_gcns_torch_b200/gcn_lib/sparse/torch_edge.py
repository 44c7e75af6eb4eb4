"""Sparse-layout graph construction - API of the reference's gcn_lib/sparse/torch_edge.py
(`knn='matrix'` builders) on the fused distance/selection kernels of the dense path:
the same launch as `gcn_lib.dense.DenseDilatedKnnGraph` with flattened, globally
numbered output (2, N_total*k) instead of (2, B, N, k)."""
import torch
from torch import nn

from ... import _native
from ..dense.torch_edge import _stochastic_columns

__all__ = ["Dilated", "DilatedKnnGraph", "knn_matrix", "knn_graph_matrix", "pairwise_distance"]


def pairwise_distance(x):
    """sparse/torch_edge.py:52-62, for API completeness only ((B,N,C) -> (B,N,N))."""
    inner = -2 * torch.matmul(x, x.transpose(2, 1))
    sq = torch.sum(x * x, dim=-1, keepdim=True)
    return sq + inner + sq.transpose(2, 1)


def _clouds(x, batch):
    """sparse/torch_edge.py:73-77: `batch[-1] + 1` equally sized clouds stored back to back."""
    batch_size = 1 if batch is None else int(batch[-1]) + 1
    if x.shape[0] % batch_size != 0:
        raise RuntimeError("shape '[%d, -1, %d]' is invalid for input of size %d"
                           % (batch_size, x.shape[-1], x.numel()))       # what x.view says in the reference
    return batch_size, x.shape[0] // batch_size


def _knn_flat(x, k, dilation, cols, batch):
    """(N_total, C) -> (nn_idx, center_idx), each (1, N_total*k) int64 with global point numbers.  bf16 / fp16
    features (torch.autocast) are widened to fp32 in the transposed copy the selection kernels read anyway, so the
    graph is the one of x.float()."""
    with torch.no_grad():
        B, n = _clouds(x, batch)
        dtype = torch.float32 if x.dtype in (torch.bfloat16, torch.float16) else x.dtype
        xb = x.detach().reshape(B, n, x.shape[-1]).transpose(1, 2).to(dtype, memory_format=torch.contiguous_format)
        xb = xb.unsqueeze(-1)                                                                     # (B,C,n,1)
        ei, _ = _native.knn_graph(xb, k, dilation, cols=cols)                                   # (2,B,n,k) local ids
        start = torch.arange(0, B * n, n, device=x.device).view(1, B, 1, 1)
        ei = ei + start
    return ei[0].reshape(1, -1), ei[1].reshape(1, -1)


def knn_matrix(x, k=16, batch=None):
    """sparse/torch_edge.py:65-90: nearest neighbours by pairwise distance, self included,
    ascending; returns (nn_idx, center_idx), both (1, N_total*k)."""
    return _knn_flat(x, k, 1, None, batch)


def knn_graph_matrix(x, k=16, batch=None):
    """sparse/torch_edge.py:93-103: edge_index (2, N_total*k), row 0 = neighbour, row 1 = centre."""
    nn_idx, center_idx = knn_matrix(x, k, batch)
    return torch.cat((nn_idx, center_idx), dim=0)


class Dilated(nn.Module):
    """sparse/torch_edge.py:6-29: keep every `dilation`-th of each point's k*dilation neighbours
    (or a random k of them with probability epsilon while training)."""

    def __init__(self, k=9, dilation=1, stochastic=False, epsilon=0.0):
        super().__init__()
        self.dilation = dilation
        self.stochastic = stochastic
        self.epsilon = epsilon
        self.k = k

    def forward(self, edge_index, batch=None):
        cols = _stochastic_columns(self.k, self.dilation, self.stochastic, self.epsilon, self.training)
        if cols is None:
            return edge_index[:, ::self.dilation]
        num = self.k * self.dilation
        sel = torch.as_tensor(cols, device=edge_index.device)
        return edge_index.view(2, -1, num)[:, :, sel].reshape(2, -1)


class DilatedKnnGraph(nn.Module):
    """sparse/torch_edge.py:32-49 with knn='matrix' (the default).  The dilation happens inside the
    selection kernel.  Any other `knn` selects torch_cluster.knn_graph in the reference, a third-party
    CUDA extension this package does not re-implement."""

    def __init__(self, k=9, dilation=1, stochastic=False, epsilon=0.0, knn="matrix"):
        super().__init__()
        self.dilation = dilation
        self.stochastic = stochastic
        self.epsilon = epsilon
        self.k = k
        self._dilated = Dilated(k, dilation, stochastic, epsilon)
        if knn != "matrix":
            raise NotImplementedError("knn='%s' is torch_cluster.knn_graph in the reference; only 'matrix' is built" % knn)
        self.knn = knn_graph_matrix

    def forward(self, x, batch):
        cols = _stochastic_columns(self.k, self.dilation, self.stochastic, self.epsilon, self.training)
        nn_idx, center_idx = _knn_flat(x, self.k, self.dilation, cols, batch)
        return torch.cat((nn_idx, center_idx), dim=0)
