"""CPU restatement of the slab path's multi-select (select_rows_fast_kernel, step 3 in
deep_gcns_torch_b200/csrc/knn.cu): histogram the keys below the bound into 256 distance bins, find the
bins holding the wanted ranks, sort only those bins' keys, read rank r at position r - (#keys in unmarked
bins below its bin).  The algorithm - not the CUDA code - is checked here against a full sort."""
import numpy as np


def _ordered(f):
    u = np.asarray(f, dtype=np.float32).view(np.uint32)
    return np.where(u & 0x80000000, ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def multiselect(dist, ranks, dlo, dhi):
    """dist: float32 distances of the compacted keys (all <= dhi); returns the indices of the wanted ranks
    in (distance, index) order."""
    dist = np.asarray(dist, dtype=np.float32)
    keys = (_ordered(dist).astype(np.uint64) << np.uint64(32)) | np.arange(dist.size, dtype=np.uint64)
    dlo, dhi = np.float32(dlo), np.float32(dhi)
    scale = np.float32(255.99) / (dhi - dlo) if dhi > dlo else np.float32(0)
    t = (dist - dlo) * scale                                     # fp32, like the kernel
    bins = np.where(t > 0, np.minimum(255, t.astype(np.int64)), 0)
    hist = np.bincount(bins, minlength=256)
    pre = np.concatenate([[0], np.cumsum(hist)])                 # exclusive prefix, pre[256] = total
    mark = np.zeros(256, dtype=bool)
    mybin = []
    for r in ranks:
        b = int(np.searchsorted(pre, r, side="right")) - 1       # last b with pre[b] <= r
        b = min(b, 255)
        mark[b] = True
        mybin.append(b)
    unmarked_below = np.concatenate([[0], np.cumsum(np.where(mark, 0, hist))])[:256]
    kept = np.sort(keys[mark[bins]])
    out = [int(kept[r - unmarked_below[b]] & np.uint64(0xFFFFFFFF)) for r, b in zip(ranks, mybin)]
    return out, int(kept.size)


def _check(dist, ranks, dlo, dhi):
    order = np.lexsort((np.arange(dist.size), _ordered(dist)))   # (distance, index) ascending
    got, kept = multiselect(dist, ranks, dlo, dhi)
    assert got == [int(order[r]) for r in ranks]
    return kept


def test_multiselect_equals_full_sort_random():
    rng = np.random.default_rng(0)
    for n, k, d in ((1300, 20, 27), (420, 20, 3), (700, 9, 16), (2048, 64, 8), (64, 20, 3)):
        dist = rng.gamma(8.0, 10.0, size=n).astype(np.float32)
        ranks = [l * d for l in range(k)]
        assert ranks[-1] < n
        srt = np.sort(dist)
        kept = _check(dist, ranks, srt[min(32, n - 1)], srt[-1])
        assert kept <= n
        # random (stochastic-dilation) rank sets
        ranks = sorted(rng.choice(k * d, size=k, replace=False).tolist())
        _check(dist, ranks, srt[min(32, n - 1)], srt[-1])


def test_multiselect_ties_clusters_and_degenerate_range():
    rng = np.random.default_rng(1)
    # massive ties: every key identical -> one bin, everything sorted, index order decides
    dist = np.full(300, 7.25, dtype=np.float32)
    _check(dist, [0, 3, 299], 7.25, 7.25)
    # two clusters + exact duplicates + keys below the lower sample (bin 0) + a zero self distance
    dist = np.concatenate([[0.0], rng.normal(10, 1e-4, 200), rng.normal(50, 1e-3, 200), np.full(50, 50.0)]).astype(np.float32)
    rng.shuffle(dist)
    hi = float(dist.max())
    for lo in (0.0, 9.9999, 10.0, 49.0):
        _check(dist, [0, 1, 57, 200, 201, 300, 449, 450], lo, hi)
    # grid of exactly representable distances (many exact ties across bins)
    dist = (rng.integers(0, 40, size=1000) / 8.0).astype(np.float32)
    _check(dist, list(range(0, 1000, 37)), 0.5, float(dist.max()))
