"""CPU restatement of knn_tc4_kernel's fp16 pre-filter bound (knn_tc4.cuh, DESIGN.md 6) and of the list length /
band cap it needs.

eps = 2 ((|e_i| sqrt(smax) + |h_i| sqrt(emax)) (1 + 2^-9) + (2 Cpad + 16) 2^-23 |x_i| sqrt(smax))
      + 2^-20 (|x_i|^2 + smax)
with h = fp16(x), e >= |h - x| per channel (|x| where h is subnormal: the MMA may flush it) and emax the cloud's
max |e_j|^2 must bound |approx - exact| for the key |x_j|^2 - 2 x_i.x_j, where approx comes from one fp16 product per channel
(round to nearest, subnormals kept or flushed to zero) accumulated in fp32 together with the bf16 split of
-|x_j|^2/2, and exact is the fp32 FMA chain of the exact re-rank.  The count model emulates the set-only membership
step (packed 20-bit list entries, the band [lo, hi], the certificate hi < cut and the band cap) on random 64-d
clouds: the chosen list lengths and band cap leave at most 1e-4 of the queries to the completion kernel, a list of
24 entries with 12 band places would leave more than 1e-3."""
import numpy as np
import pytest
import torch

F16_MIN_NORMAL = 2.0 ** -14


def err2(x):
    """Squared rounding error per point of the fp16 operand (tc_f16_err2 summed over the channels of each row)."""
    x = np.asarray(x, np.float64)
    h = np.clip(x, -65504.0, 65504.0).astype(np.float16).astype(np.float64)
    e = np.abs(h - x)
    e = np.where((h != 0) & (np.abs(h) < F16_MIN_NORMAL), np.maximum(e, np.abs(x)), e)
    return (e ** 2).sum(-1)


def eps_fp16(ei2, hi2, emax, sqq, smax, cpad):
    return (2 * ((np.sqrt(ei2) * np.sqrt(smax) + np.sqrt(hi2) * np.sqrt(emax)) * (1 + 2 ** -9)
                 + (2 * cpad + 16) * 2 ** -23 * np.sqrt(sqq * smax)) + 2 ** -20 * (sqq + smax))


def eps_fp16_worst(sqq, smax, cpad):
    """The bound from |h - x| <= 2^-11 |x| (+ 2^-14 absolute below the normal range) alone, without the measured
    rounding errors: what the list length would have to cover without them."""
    return (2 * (2 ** -10 + 2 ** -21 + (2 * cpad + 16) * 2 ** -23) * np.sqrt(sqq * smax) + 2 ** -20 * (sqq + smax)
            + 2 ** -13 * np.sqrt(cpad) * (np.sqrt(sqq) + np.sqrt(smax)))


def to_f16(x, ftz):
    """The prologue's conversion (clamp, round to nearest); ftz: the MMA reads subnormal inputs as zero."""
    h = np.clip(x, -65504.0, 65504.0).astype(np.float16).astype(np.float64)
    if ftz:
        h = np.where(np.abs(h) < F16_MIN_NORMAL, 0.0, h)
    return h


def bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(torch.bfloat16).double().numpy()


def keys(xq, xc, ftz):
    """(approx, exact) keys |x_j|^2 - 2 x_q.x_j of the candidates xc (M, C) for the query xq (C,), both fp32."""
    xq = xq.astype(np.float32)
    xc = xc.astype(np.float32)
    hq, hc = to_f16(xq.astype(np.float64), ftz), to_f16(xc.astype(np.float64), ftz)
    # exact fp32 FMA chains (sq like sqnorm_kernel, the dot like the re-rank): products exact in float64, one
    # rounding to fp32 per step
    sqc = np.zeros(len(xc), np.float32)
    dot = np.zeros(len(xc), np.float32)
    for c in range(xc.shape[1]):
        sqc = (sqc.astype(np.float64) + xc[:, c].astype(np.float64) ** 2).astype(np.float32)
        dot = (dot.astype(np.float64) + np.float64(xq[c]) * xc[:, c]).astype(np.float32)
    exact = sqc.astype(np.float64) - 2 * dot.astype(np.float64)
    # tensor core: fp16 products (exact in fp32) accumulated in fp32, then the 3-term bf16 split of -|x_j|^2/2
    acc = np.zeros(len(xc), np.float32)
    for c in range(xc.shape[1]):
        acc = (acc.astype(np.float64) + hq[c] * hc[:, c]).astype(np.float32)
    rem = -0.5 * sqc.astype(np.float64)
    for _ in range(3):
        t = bf16(rem.astype(np.float32))
        acc = (acc.astype(np.float64) + t).astype(np.float32)
        rem = (rem - t).astype(np.float32).astype(np.float64)
    approx = -2 * acc.astype(np.float64)
    return approx, exact, sqc.astype(np.float64)


def check_bound(xq, xc, ftz):
    approx, exact, sqc = keys(xq, xc, ftz)
    sqq = float(np.sum(xq.astype(np.float64) ** 2))
    smax = max(float(sqc.max()), sqq)
    cpad = (xc.shape[1] + 15) // 16 * 16
    err = np.abs(approx - exact)
    hq = to_f16(xq.astype(np.float64), False)
    emax = max(float(err2(xc).max()), float(err2(xq)))
    eps = eps_fp16(float(err2(xq)), float((hq ** 2).sum()), emax, sqq, smax, cpad)
    assert err.max() <= eps, (err.max(), eps)
    assert eps <= eps_fp16_worst(sqq, smax, cpad) * 1.01
    return err.max() / eps


@pytest.mark.parametrize("ftz", [False, True])
def test_bound_random_vectors(ftz):
    rng = np.random.default_rng(11)
    for c in (16, 40, 64):
        x = rng.standard_normal((513, c)).astype(np.float32)
        check_bound(x[0], x[1:], ftz)
        x = (rng.standard_normal((513, c)) * np.exp(rng.uniform(-6, 6, (513, 1)))).astype(np.float32)
        check_bound(x[0], x[1:], ftz)


@pytest.mark.parametrize("ftz", [False, True])
def test_bound_adversarial_vectors(ftz):
    """Every component halfway between two fp16 values (the largest relative rounding error, all of one sign so
    nothing cancels), mixed magnitudes down to the subnormal range in one vector."""
    rng = np.random.default_rng(12)
    c = 64
    e = rng.integers(-3, 4, (257, c)).astype(np.float64)
    half = ((1 + 2.0 ** -11) * 2.0 ** e).astype(np.float32)           # exactly representable in fp32
    assert np.all(np.abs(half.astype(np.float16).astype(np.float64) - half) == 2.0 ** -11 * 2.0 ** e)
    worst = check_bound(half[0], half[1:], ftz)
    assert worst > 0.25                                                 # the bound is not loose by orders here
    mags = 2.0 ** rng.integers(-24, 6, (257, c))
    mixed = (rng.choice([-1.0, 1.0], (257, c)) * mags * (1 + 2.0 ** -11)).astype(np.float32)
    check_bound(mixed[0], mixed[1:], ftz)


@pytest.mark.parametrize("ftz", [False, True])
def test_bound_subnormal_inputs(ftz):
    rng = np.random.default_rng(13)
    for scale in (2.0 ** -16, 2.0 ** -20, 2.0 ** -24):
        x = (rng.standard_normal((257, 64)) * scale).astype(np.float32)
        assert (np.abs(x) < F16_MIN_NORMAL).mean() > 0.9
        check_bound(x[0], x[1:], ftz)
    # a normal query against subnormal candidates and the other way round
    x = rng.standard_normal((257, 64)).astype(np.float32)
    x[1:] *= np.float32(2.0 ** -18)
    check_bound(x[0], x[1:], ftz)
    check_bound(x[1], np.concatenate([x[:1], x[2:]]), ftz)


def test_bound_near_the_range_limit():
    """Just inside the range guard (max |x|^2 < 2^30, so every |x_c| < 2^15 and nothing is clamped), and the
    clamp itself: values beyond 65504 become 65504, never inf."""
    rng = np.random.default_rng(14)
    x = rng.standard_normal((257, 64))
    x = x / np.sqrt((x ** 2).sum(1, keepdims=True)) * (2.0 ** 15 - 1)   # |x|^2 just under 2^30
    x = x.astype(np.float32)
    assert float((x.astype(np.float64) ** 2).sum(1).max()) < 2.0 ** 30
    check_bound(x[0], x[1:], False)
    big = np.array([1e6, -1e6, 65519.0, 65521.0, np.inf, -np.inf])
    h = to_f16(big, False)
    assert np.all(np.isfinite(h)) and np.all(np.abs(h) <= 65504.0)


# ---- count model of the set-only membership step -----------------------------------------------------------------
N, C = 4096, 64


def packed_lower(d2, sqq):
    """The list entry's 20-bit value: accumulator low 12 bits rounded toward a smaller distance, then 12 distance
    bits truncated - a lower bound of the approximate squared distance."""
    acc = ((sqq - d2) / 2).astype(np.float32)
    b = acc.view(np.uint32).copy()
    b = np.where((b & 0x80000000) != 0, b & 0xFFFFF000, b | 0xFFF).astype(np.uint32)
    d = np.maximum(np.float32(sqq) - np.float32(2) * b.view(np.float32), 0).astype(np.float32)
    return (d.view(np.uint32) & 0xFFFFF000).view(np.float32)


def uncertified_share(K, variants, clouds, queries, seed):
    """{(KP, MB): share of queries the set-only path leaves uncertified} on `clouds` 64-d randn clouds."""
    rng = np.random.default_rng(seed)
    kpmax = max(kp for kp, _ in variants)
    fails = {v: 0 for v in variants}
    total = 0
    for _ in range(clouds):
        x = rng.standard_normal((N, C)).astype(np.float32)
        X = x.astype(np.float64)
        sq = (X ** 2).sum(1)
        smax = sq.max()
        h16 = to_f16(X, False)
        q = rng.choice(N, queries, replace=False)
        sqq = sq[q][:, None]
        approx = sqq - 2 * (h16[q] @ h16.T) + sq[None, :]
        e2 = err2(X)
        eps = eps_fp16(e2[q][:, None], (h16[q] ** 2).sum(1)[:, None], e2.max(), sqq, smax, C)
        assert np.all(np.abs(approx - (sqq - 2 * (X[q] @ X.T) + sq[None, :])) <= eps)
        v = packed_lower(approx, sqq.astype(np.float32))
        v = np.sort(np.partition(v, kpmax, axis=1)[:, :kpmax + 1], axis=1).astype(np.float64)
        e, s = eps[:, 0], sqq[:, 0]
        for kp, mb in variants:
            vK, vK1, cut = v[:, K - 1], v[:, K], v[:, kp - 1]
            hi = vK + 2 ** -10 * (vK + s) + 2 * e
            lo = vK1 - 2 ** -10 * (vK1 + s) - 2 * e
            w = v[:, :kp]
            nb = ((w >= lo[:, None]) & (w <= hi[:, None])).sum(1)
            fails[(kp, mb)] += int((~((hi < cut) & (nb <= mb))).sum())
        total += queries
    return {k: f / total for k, f in fails.items()}


def test_count_model_list_length_and_band_cap_k20():
    share = uncertified_share(20, [(32, 16), (24, 12)], clouds=12, queries=1024, seed=2)
    assert share[(32, 16)] <= 1e-4, share
    assert share[(24, 12)] > 1e-3, share        # the model has teeth: a list of 24 would not do


def test_count_model_list_length_k9():
    share = uncertified_share(9, [(20, 16)], clouds=12, queries=1024, seed=3)
    assert share[(20, 16)] <= 1e-4, share
