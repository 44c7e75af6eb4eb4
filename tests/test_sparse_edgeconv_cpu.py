"""Sparse-layout EdgeConv without a GPU: the fp32 identity the kernel rests on, max_e f(z_e) == max(f(z_max), f(z_min))
for f(z) = act(fmaf(s, z, t)), on adversarial values; the restatement's first-edge routing; the module's API against
the reference (golden spconv_edge) and its errors."""
import fractions
import inspect
import itertools

import numpy as np
import pytest
import torch
from torch import nn

import golden_util as gu
import sparse_edge_util as seu


def fmaf(s, z, t):
    """fp32 fmaf: s * z + t rounded once to the nearest fp32 (ties to even), from the exact rational value."""
    exact = fractions.Fraction(float(s)) * fractions.Fraction(float(z)) + fractions.Fraction(float(t))
    guess = np.float32(float(exact))
    cands = [np.nextafter(guess, np.float32(-np.inf)), guess, np.nextafter(guess, np.float32(np.inf))]
    cands = [c for c in cands if np.isfinite(c)]
    best = min(cands, key=lambda c: (abs(fractions.Fraction(float(c)) - exact), int(c.view(np.int32)) & 1))
    return best


def act(u, slope):
    """common.cuh act_apply: u >= 0 ? u : u * slope, in fp32."""
    return u if u >= 0 else np.float32(u * np.float32(slope))


def f(z, s, t, slope):
    return act(fmaf(s, z, t), slope)


ADVERSARIAL_Z = [np.float32(v) for v in
                 (0.0, -0.0, 1e-38, -1e-38, 1.4e-45, -1.4e-45, 1e-7, -1e-7, 0.5, -0.5, 1.0, -1.0, 3.0, -2.75, 1e4,
                  -1e4, 0.1, -0.1, 0.30000001, -0.29999998)]
SCALES = [np.float32(v) for v in (1.0, -1.0, 0.0, -0.0, 2.5, -0.3, 1e-20, -7.0)]
SHIFTS = [np.float32(v) for v in (0.0, -0.0, 0.1, -0.1, 1.0, -3.0, 1e-30)]
SLOPES = [np.float32(v) for v in (0.0, 0.2, 0.25, 1.0, -0.3, -1.0)]     # relu, leaky relu, prelu (> 0, < 0), none


@pytest.mark.parametrize("slope", SLOPES)
def test_max_of_f_is_attained_at_the_extremes_of_z(slope):
    """For every activation slope (PReLU weight < 0 included: f is V-shaped), every affine (s < 0, s = 0, +-0) and
    sets of z around the kink: max_e f(z_e) == max(f(z_max), f(z_min)) bit for bit in fp32."""
    g = np.random.default_rng(0)
    checked = 0
    for s, t in itertools.product(SCALES, SHIFTS):
        kink = -t / s if s != 0 else np.float32(0.0)                    # z where s z + t crosses 0
        near = [np.float32(kink), np.nextafter(np.float32(kink), np.float32(1)),
                np.nextafter(np.float32(kink), np.float32(-1))] if np.isfinite(kink) else []
        pool = ADVERSARIAL_Z + near
        for _ in range(12):
            zs = list(g.choice(pool, size=int(g.integers(1, 7)), replace=True))
            ys = [f(z, s, t, slope) for z in zs]
            want = max(ys)
            got = max(f(max(zs), s, t, slope), f(min(zs), s, t, slope))
            assert got == want, (s, t, slope, zs)
            checked += 1
    assert checked == len(SCALES) * len(SHIFTS) * 12


def test_fmaf_emulation_rounds_once():
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24: the product alone rounds to 1 + 2^-11, the fused sum with -1 keeps 2^-24
    s = np.float32(1 + 2 ** -12)
    assert fmaf(s, s, np.float32(-1.0)) == np.float32(2 ** -11 + 2 ** -24)
    assert fmaf(np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12), np.float32(0.0)) == np.float32(1 + 2 ** -11)


def test_restatement_routes_a_tied_max_to_the_first_edge():
    """sparse_edge_util.seg_max_first (torch_scatter's scatter_max): the gradient of a tied max goes to the first edge
    in edge order only; an empty row is 0 and takes none."""
    y = torch.tensor([[1.0, 2.0], [3.0, 2.0], [3.0, 0.5], [5.0, 5.0]], dtype=torch.float64, requires_grad=True)
    dst = torch.tensor([0, 0, 0, 2])
    out, arg = seu.seg_max_first(y, dst, 3)
    assert out.tolist() == [[3.0, 2.0], [0.0, 0.0], [5.0, 5.0]]
    assert arg.tolist() == [[1, 0], [-1, -1], [3, 3]]
    out.sum().backward()
    assert y.grad.tolist() == [[0.0, 1.0], [1.0, 0.0], [0.0, 0.0], [1.0, 1.0]]


def test_restatement_matches_the_reference_shim_forward():
    """sparse_edge_util.edge_conv against its stand-in for torch_geometric's EdgeConv (oracle/ref_shims.py's
    MessagePassing and scatter amax), on the golden's graph with BatchNorm in train mode."""
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    c = gu.load("spconv_edge")
    x, ei = c.ins["x"], c.ins["edge_index"].long()
    mod = S.EdgConv(c.meta["C"], c.meta["out"], "prelu", "batch")
    name = "prelu_neg_train"
    mod.load_state_dict({k[len(name) + 1:]: v for k, v in c.sd.items() if k.startswith(name + ".")}, strict=True)
    shim = seu.EdgeConvStandIn(mod.nn.train())
    with torch.no_grad():
        ref = shim(x, ei)
    got = seu.edge_conv(x, ei, seu.edge_conv_params(mod.nn), "prelu", training=True)
    torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(got, c.outs["y_" + name], rtol=1e-4, atol=1e-5)


def test_state_dict_and_signature_match_reference():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    c = gu.load("spconv_edge")
    sig = [[p.name, p.default if p.default is not inspect.Parameter.empty else "<empty>"]
           for p in inspect.signature(S.EdgConv.__init__).parameters.values()]
    assert sig == c.meta["signature_EdgConv"]
    for name in c.meta["cases"]:
        act = name.split("_")[0]
        mod = S.EdgConv(c.meta["C"], c.meta["out"], act, None if name.endswith("_none") else "batch", True)
        ref_keys = [k[len(name) + 1:] for k in c.sd if k.startswith(name + ".")]
        assert list(mod.state_dict().keys()) == ref_keys, name
        mod.load_state_dict({k: c.sd[name + "." + k] for k in ref_keys}, strict=True)
    assert isinstance(S.GraphConv(4, 8, "edge").gconv, S.EdgConv)
    assert isinstance(S.ResDynBlock(8, 4, 1, "edge").body.gconv, S.EdgConv)


def test_unsupported_configurations_raise():
    from deep_gcns_torch_b200.gcn_lib import sparse as S
    with pytest.raises(NotImplementedError):
        S.EdgConv(4, 8, aggr="add")
    with pytest.raises(NotImplementedError):
        S.EdgConv(4, 8, norm="layer")
    x, ei = torch.randn(5, 4), torch.zeros((2, 3), dtype=torch.long)
    with pytest.raises(NotImplementedError):
        nn.SyncBatchNorm.convert_sync_batchnorm(S.EdgConv(4, 8, "relu", "batch"))(x, ei)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.EdgConv(4, 8)(x, ei)
    with pytest.raises(RuntimeError, match="CUDA"):
        S.GraphConv(4, 8, "edge")(x.double(), ei)


@pytest.mark.parametrize("name", list(seu.EXACT_SHAPES))
def test_exact_fixture_premises(name):
    """The premises of tests/test_sparse_edgeconv_shapes_gpu.py's exact grid, for every fixture it builds: fp32 z from
    the kernel's factorised form P_i + Q_j, with P and Q each summed in two orders (one channel at a time ascending,
    and in chunks of 32 descending), is bit-equal to fp64 z of the reference's W [x_i; x_j - x_i] + b; in eval (eps = 0) so is
    u = s z + t; the offset channels are un-centred (|mean| / std of z > 100 on the last channel); and in train mode
    no fp64 top-two gap of distinct z, nor a winning |u|, is within edge_tie_mask's near-tie / kink bounds."""
    N, ci, co, hub, seed = seu.EXACT_SHAPES[name]
    acts = seu.ALL_ACTS if name in seu.BIG_SHAPES else seu.ALL_ACTS[:1]
    for act, slope in acts:
        for train in (False, True):
            mod, x, ei, _ = seu.exact_fixture(N, ci, co, act, slope, train, seed, hub)
            w, b = mod.nn[0].weight.detach(), mod.nn[0].bias.detach()
            src, dst = ei[0], ei[1]
            z64 = torch.nn.functional.linear(torch.cat([x[dst], x[src] - x[dst]], 1).double(), w.double(), b.double())
            assert z64.abs().max() < 2.0 ** 20
            w1, w2 = w[:, :ci], w[:, ci:]
            for order, chunk in ((torch.arange(ci), 1), (torch.arange(ci).flip(0), 32)):
                P = b.expand(N, co).clone()
                Q = torch.zeros(N, co)
                for c0 in range(0, ci, chunk):
                    cs = order[c0:c0 + chunk]
                    P += x[:, cs] @ (w1 - w2)[:, cs].T
                    Q += x[:, cs] @ w2[:, cs].T
                assert torch.equal((P[dst] + Q[src]).double(), z64), (name, act, train)
            bn = mod.nn[1]
            if not train:
                s = bn.weight.detach() / torch.sqrt(bn.running_var + bn.eps)
                t = bn.bias.detach() - bn.running_mean * s
                z32 = z64.float()
                assert torch.equal((s * z32 + t).double(), s.double() * z64 + t.double())
            else:
                if co >= 3:
                    zc = z64[:, co - 1]
                    assert float(zc.mean().abs() / zc.std()) > 100
                assert int(seu.edge_tie_mask(mod.nn, x, ei, 1e-4, 1e-5, True, exact=True).sum()) == 0, (name, act)
                if co >= 2:
                    assert bool((z64[:, 1] == 0).all())
