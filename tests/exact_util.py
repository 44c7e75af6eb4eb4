"""Exact-arithmetic fixtures of the tie and kink tests (no GPU needed here).

Coordinates and features are integers in [-4, 4], padding rows are zeros, conv weights and biases are multiples of
1/16 in [-1, 1] and eval-mode running statistics are dyadic.  With C <= 64 every squared distance, every EdgeConv
node row P = (W1 - W2) x + b, Q = W2 x, every pre-activation - on the kernels' factorised form and on the reference's
W [x_i; x_j - x_i] alike - and every MRConv x_j - x_i is exact in fp32, bf16 and fp16.  So each tie between two
neighbours and each z == 0 is real: no evaluation order may break it differently, and the kernels must give torch's
answer without any near-tie mask (tests/test_exact_ties_cpu.py checks these premises)."""
import torch

GAMMAS = (-1.5, -0.5, 0.0, 0.5, 1.25)   # BatchNorm scales, cycled over the channels (0: every edge ties in y)
DEAD = 3                                 # the output channel with weight 0 (constant pre-activation = its bias)


def cloud(kind, C, N, seed):
    """One (C, N) fp32 cloud: 'pad1' (the last point zero), 'pad25' / 'pad60' (the last 25 % / 60 % zero), 'zeros'
    (every point zero), 'dup3' (every point three times in a row) or 'dups' (random, with a few exact copies)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 5, (C, N), generator=g).float()
    if kind == "zeros":
        return torch.zeros(C, N)
    if kind == "dup3":
        return x[:, torch.arange(N) // 3].contiguous()
    if kind.startswith("pad"):
        n_pad = 1 if kind == "pad1" else N * int(kind[3:]) // 100
        x[:, N - n_pad:] = 0
    if kind in ("pad25", "dups"):
        x[:, 7] = x[:, 3]                      # copies of live points, in and out of the first query tile
        x[:, N // 2] = x[:, 3]
        x[:, N // 3] = x[:, N - 5]             # (a copy of a padding point under 'pad25')
    return x


def batch(kinds, C, N, seed=0):
    """(B, C, N, 1) fp32 batch, one cloud per kind."""
    return torch.stack([cloud(k, C, N, seed + 7 * i) for i, k in enumerate(kinds)]).unsqueeze(-1)


def lex_knn(x, K, exclude_self=False):
    """(B, N, K) int64: the K nearest points of every query in (squared distance, index)-lexicographic order,
    computed exactly in fp64 on x's device (integer coordinates: the distances are integers)."""
    xt = x.squeeze(-1).transpose(1, 2).double()
    B, N, _ = xt.shape
    sq = (xt * xt).sum(-1)
    d = sq.unsqueeze(2) - 2 * xt @ xt.transpose(1, 2) + sq.unsqueeze(1)
    key = d * N + torch.arange(N, device=x.device, dtype=torch.float64)      # < 2^53: exact, and unique per row
    if exclude_self:
        key.diagonal(dim1=1, dim2=2).fill_(float("inf"))
    return key.topk(K, dim=-1, largest=False, sorted=True).indices


def edge_index_of(nbr):
    """(2, B, N, k) int64 edge_index of a (B, N, k) neighbour list (row 1: the centres)."""
    B, N, k = nbr.shape
    i = torch.arange(N, device=nbr.device).view(1, N, 1).expand(B, N, k)
    return torch.stack((nbr.long(), i))


def sixteenths(shape, g):
    """Multiples of 1/16 in [-1, 1]."""
    return torch.randint(-16, 17, shape, generator=g).float() / 16


def set_params(mod, bias, slope=None, seed=0):
    """Exact parameters of a DynConv2d / GraphConv2d: weights in sixteenths with output channel DEAD dead (weight
    0), bias 'on' (sixteenths, DEAD's 1/2), 'zero' or absent ('none': the module was built with bias=False);
    PReLU slope `slope`; BatchNorm scales cycling through GAMMAS, shifts in eighths, running mean in eighths and
    running variance in {1/2, 1, 2, 4}."""
    g = torch.Generator().manual_seed(seed)
    nn_ = mod.gconv.nn
    conv = nn_[0]
    co = conv.weight.shape[0]
    with torch.no_grad():
        conv.weight.copy_(sixteenths(conv.weight.shape, g))
        conv.weight[DEAD] = 0
        if bias == "on":
            conv.bias.copy_(sixteenths((co,), g))
            conv.bias[DEAD] = 0.5
        elif bias == "zero":
            conv.bias.zero_()
        else:
            assert conv.bias is None
        for m in nn_:
            if isinstance(m, torch.nn.PReLU):
                m.weight.fill_(slope)
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(torch.tensor(GAMMAS)[torch.arange(co) % len(GAMMAS)])
                m.bias.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_mean.copy_(torch.randint(-8, 9, (co,), generator=g).float() / 8)
                m.running_var.copy_(2.0 ** torch.randint(-1, 3, (co,), generator=g).float())
    return mod
