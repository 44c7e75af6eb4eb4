"""CPU restatement of the dense path's train-mode BatchNorm statistics (common.cuh: bn_acc_add, bn_acc_moments,
bn_merge; basic_conv.cu: bn_merge_kernel), fp32 emulated with np.float32, in the kernels' order:

- each thread sums a - pivot and (a - pivot)^2 along its chain (pivot = its first value),
- threads of a warp merge (count, mean, M2) with Chan's formula along an xor-shuffle tree, warps in order,
- the partial rows are merged in fp64: thread-strided (256 threads), then a shared-memory tree.

The shapes are those of the writers (partials x warps x lanes x chain length).  The parent's scheme, fp32 sums of
a and a^2 with var = E[a^2] - E[a]^2 from their fp64 totals, is restated as well, to show that these shapes and
conditionings do expose the cancellation the new scheme removes."""
import numpy as np
import pytest

F32 = np.float32
GPU_VAR_TOL = 1e-5           # tests/test_bn_batch_stats_gpu.py: |var - var64| <= 1e-5 var64

# name: (partials, warps merged in order, lanes merged by xor shuffles, chain length per lane, empty partials)
SHAPES = {
    # knn_tc_kernel, wide TRAIN consumer: B=1 N=512 k=9, 4 CTAs, 4 warps, 2 query slots per warp, 16 queries x 9
    # per lane; 132 rows of the completion kernel, empty when every query is certified
    "tc-wide B1 N512 k9": (4, 4, 2, 144, 132),
    # slab path, row_consume: one partial per query row, B=16 N=4096 k=20
    "slab B16 N4096 k20": (16 * 4096, 1, 1, 20, 0),
    # graph_gather_kernel: B=2 N=1024 k=20, 32 nodes per CTA, 8 warps of 4 nodes x 20 edges per lane
    "gather B2 N1024 k20": (2 * 32, 8, 1, 80, 0),
    # knn_small_kernel, cta_epilogue: B=1 N=128 k=9, 8 warps of 16 queries x 9 per lane
    "small B1 N128 k9": (1, 8, 1, 144, 0),
}


def _fma(a, b, c):
    return (a.astype(np.float64) * b + c).astype(F32)


def _merge32(a, b):
    """bn_merge: (n, mean, m2) float32 arrays."""
    n = a[0] + b[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        f = np.where(n > 0, b[0] / np.where(n > 0, n, F32(1)), F32(0)).astype(F32)
    delta = b[1] - a[1]
    return n, _fma(delta, f, a[1]), a[2] + b[2] + delta * (delta * (a[0] * f))


def _merge64(a, b):
    n = a[0] + b[0]
    f = np.where(n > 0, b[0] / np.where(n > 0, n, 1.0), 0.0)
    delta = b[1] - a[1]
    return n, a[1] + delta * f, a[2] + b[2] + delta * (delta * (a[0] * f))


def new_scheme(vals, empty=0):
    """vals (P, W, S, L) float32 -> (count, mean, biased var) in fp64 as bn_merge_kernel forms them; `empty`
    zero-count partial rows follow the P rows (the completion kernel's rows when nothing was left to it)."""
    P, W, S, L = vals.shape
    n = np.zeros((P, W, S), F32)
    piv, d1, d2 = n.copy(), n.copy(), n.copy()
    for l in range(L):                                  # bn_acc_add
        a = vals[..., l]
        piv = np.where(n == 0, a, piv)
        d = a - piv
        n, d1, d2 = n + F32(1), d1 + d, _fma(d, d, d2)
    m = (d1 / np.where(n > 0, n, F32(1))).astype(F32)   # bn_acc_moments
    mo = (n, np.where(n > 0, piv + m, F32(0)), np.where(n > 0, np.maximum(_fma(-d1, m, d2), F32(0)), F32(0)))
    o = 1
    while o < S:                                        # xor shuffles: lane i merges with lane i ^ o
        perm = np.arange(S) ^ o
        mo = _merge32(mo, tuple(t[..., perm] for t in mo))
        o <<= 1
    mo = tuple(t[..., 0] for t in mo)                   # (P, W)
    acc = tuple(t[:, 0] for t in mo)
    for w in range(1, W):                               # warps in order
        acc = _merge32(acc, tuple(t[:, w] for t in mo))
    return merge_partials(tuple(np.concatenate([t, np.zeros(empty, F32)]) for t in acc))


def merge_partials(acc):
    """bn_merge_kernel on float32 partial rows (n, mean, m2), each (P,)."""
    P = acc[0].shape[0]
    T = 256
    part = tuple(t.astype(np.float64) for t in acc)
    th = (np.zeros(T), np.zeros(T), np.zeros(T))
    for i0 in range(0, P, T):                           # thread t merges rows t, t + 256, ...
        idx = np.arange(i0, min(i0 + T, P))
        cnt = len(idx)
        row = tuple(np.concatenate([p[idx], np.zeros(T - cnt)]) for p in part)
        th = _merge64(th, row)
    o = T >> 1
    while o > 0:
        lo = tuple(t[:o] for t in th)
        hi = tuple(t[o:2 * o] for t in th)
        th = tuple(np.concatenate([m, t[o:]]) for m, t in zip(_merge64(lo, hi), th))
        o >>= 1
    n, mean, m2 = (float(t[0]) for t in th)
    return n, mean, (m2 / n if n > 0 else 0.0)


def parent_scheme(vals):
    """The scheme the new one replaces: fp32 chains of a and a^2, fp32 lane / warp sums, fp64 over partials."""
    s1 = vals.sum(axis=-1, dtype=F32)
    s2 = np.zeros(vals.shape[:-1], F32)
    for l in range(vals.shape[-1]):
        s2 = _fma(vals[..., l], vals[..., l], s2)
    s1, s2 = s1.sum(axis=(1, 2), dtype=F32), s2.sum(axis=(1, 2), dtype=F32)
    n = vals[0].size * vals.shape[0]
    mean = s1.astype(np.float64).sum() / n
    return n, mean, max(s2.astype(np.float64).sum() / n - mean * mean, 0.0)


def _values(shape, r, seed):
    P, W, S, L, _ = shape
    g = np.random.default_rng(seed)
    return (r + g.standard_normal((P, W, S, L))).astype(F32)      # std 1, mean r


def _rel_var_err(vals, scheme):
    n, mean, var = scheme(vals)
    v64 = vals.astype(np.float64)
    ref = v64.var()
    assert n == vals.size
    return abs(var - ref) / ref, abs(mean - v64.mean())


@pytest.mark.parametrize("name", sorted(SHAPES))
@pytest.mark.parametrize("r", [1, 10, 100, 1000])
def test_new_scheme_variance_has_ten_times_margin(name, r):
    vals = _values(SHAPES[name], r, seed=r + len(name))
    err, merr = _rel_var_err(vals, lambda v: new_scheme(v, SHAPES[name][4]))
    assert err <= GPU_VAR_TOL / 10, (name, r, err)
    assert merr <= 1e-6 * r + 1e-5, (name, r, merr)


@pytest.mark.parametrize("name", ["small B1 N128 k9", "gather B2 N1024 k20"])
def test_parent_scheme_fails_at_r1000(name):
    """The restated parent scheme misses the GPU test's bound at r = 1000 on these shapes (the new GPU test fails
    on the parent kernels for the same reason)."""
    vals = _values(SHAPES[name], 1000, seed=7)
    err, _ = _rel_var_err(vals, parent_scheme)
    assert err > GPU_VAR_TOL, (name, err)


def test_report_r1e4():
    """Past the asserted range: r = 1e4 at the tensor-core shape.  Reported, not asserted - the per-partial fp32
    means carry ~ r * 2^-24 of rounding each, which the merge sees as spread."""
    vals = _values(SHAPES["tc-wide B1 N512 k9"], 1e4, seed=3)
    err, _ = _rel_var_err(vals, new_scheme)
    print("pivot-shifted sums at r = 1e4, B=1 N=512 k=9: relative variance error %.2e" % err)


def test_empty_partials_merge_without_nan():
    """Partials with zero count (CTAs whose queries were all left to the completion kernel, tail tiles, completion
    CTAs that found no work), including empty ones first in the fp64 merge order."""
    g = np.random.default_rng(5)
    P = 600
    n = np.zeros(P, F32)
    mean, m2 = np.zeros(P, F32), np.zeros(P, F32)
    live = np.arange(P) >= 300                         # the first 300 rows - first of every thread - are empty
    live &= g.random(P) < 0.5
    vals = (5.0 + g.standard_normal((P, 9))).astype(F32)
    for p in np.nonzero(live)[0]:
        n[p], mean[p] = 9, vals[p].astype(np.float64).mean()
        m2[p] = ((vals[p].astype(np.float64) - vals[p].astype(np.float64).mean()) ** 2).sum()
    cnt, mu, var = merge_partials((n, mean.astype(F32), m2.astype(F32)))
    ref = vals[live].astype(np.float64)
    assert np.isfinite([cnt, mu, var]).all()
    assert cnt == ref.size
    assert abs(mu - ref.mean()) <= 1e-6 * abs(ref.mean())
    assert abs(var - ref.var()) <= 1e-6 * ref.var()
    # the fp32 merges inside a CTA: an empty side on either hand, and two empty sides
    e = (F32(0), F32(0), F32(0))
    x = (F32(4), F32(2.5), F32(1.25))
    assert _merge32(e, x) == x and _merge32(x, e) == x
    assert _merge32(e, e) == e


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_constant_channel_exact(name):
    P, W, S, L, empty = SHAPES[name]
    vals = np.full((P, W, S, L), F32(3.7), F32)
    n, mean, var = new_scheme(vals, empty)
    assert var == 0.0
    assert F32(mean) == F32(3.7)
    assert n == vals.size
