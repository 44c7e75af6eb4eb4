"""Shared pieces of the gradient tests of the dense graph convolutions (no GPU needed here):

- oracle_grads: fp64 torch autograd through oracle.dense on the graph the kernel used;
- edge_tie_mask: the (b, c, i) entries of EdgeConv's max whose winning edge an fp32 kernel may legitimately pick
  differently from fp64 - the tests zero the upstream gradient there, on both sides;
- assert_no_mr_ties: MRConv's precondition that no such entry exists (seeds are chosen to satisfy it);
- assert_grads_close: the elementwise gradient comparison;
- kernel_names: the kernels a call launched, from torch.profiler.
"""
import torch
import torch.nn.functional as F

from oracle import dense as od

TIE_REL = 1e-4        # EdgeConv: top-two gap of the per-edge value below TIE_REL * max(1, |value|) is a near-tie
KINK_REL = 1e-5       # ... and so is a winning edge's |z| below this (ten times the fp32 error of z ~ 1)
MAX_MASKED = 1e-3     # ... and at most this share of the (b, c, i) entries may be masked
MR_TIE_REL = 1e-6     # MRConv: x_j - x_i of fp32 inputs can only change rank when the fp64 gap is below ~1e-7
ATOL_FRAC, RTOL = 1e-4, 1e-3


def check_graph(x, nn_idx, K, dilation=1, cols=None, exclude_self=False, max_frac=2e-3):
    """The kernel's (B,N,k) neighbour list against the oracle's sorted K list (self excluded or not), dilated
    by `dilation` or cut at `cols`; every mismatching slot must be an fp32 distance near-tie."""
    x = x.detach().cpu().contiguous()
    full = (od.knn_exclude_self(x, K) if exclude_self else od.knn_matrix(x, K))[0]
    ref = full[..., torch.as_tensor(cols)] if cols is not None else full[..., ::dilation]
    n_bad, n_unexplained = od.knn_mismatch_report(x, nn_idx.cpu().long(), ref)
    assert n_unexplained == 0, "kNN index mismatch that is not an fp32 near-tie"
    assert n_bad <= max_frac * nn_idx.numel(), (n_bad, nn_idx.numel())


def _pre_activation(x, edge_index, p, conv):
    """fp64 pre-activation: EdgeConv (B,Co,N,k) per edge, MRConv (B,Co,N,1) per node."""
    xd = x.detach().cpu().double()
    xi = od.batched_index_select(xd, edge_index[1])
    xj = od.batched_index_select(xd, edge_index[0])
    if conv == "edge":
        feat = torch.cat([xi, xj - xi], dim=1)
    else:
        feat = torch.cat([xd, (xj - xi).max(-1, keepdim=True)[0]], dim=1)
    return F.conv2d(feat, p["weight"], p.get("bias"))


def _kink(z, act):
    """Where an fp32 z may fall on the other side of the activation's kink at 0."""
    if act is None or str(act).lower() == "none":
        return torch.zeros_like(z, dtype=torch.bool)
    return z.abs() < KINK_REL


def edge_tie_mask(x, edge_index, gconv_nn, act, norm, training):
    """(B,Co,N,1) bool: EdgeConv entries whose max an fp32 kernel may route to a different edge than fp64.

    The max over the edges of y = s*act(z) + t picks the edge of largest act(z) when s > 0, of smallest when
    s < 0, and the first edge when s == 0 (gamma = 0: every y equals t, an exact tie that torch.max and the
    kernel both give to edge 0, so it is never masked).  The kernel ranks act(z) with the sign of s in every mode
    (edge_bwd_kernel), and its fp32
    error lives in z, so the gap is measured there: on v = sign(s) * act(z), not on y, where a channel with
    gamma near 0 would tie everywhere although its edges are well apart.  An entry is masked when another
    edge's v is within TIE_REL * max(1, |v|) of the top - unless every edge that close sits robustly in ReLU's
    flat part (z below -TIE_REL), where any choice carries a zero gradient - or when the winning edge's z is
    within KINK_REL of the activation's kink at 0.  Asserts that at most MAX_MASKED of the entries are masked,
    so the mask cannot hide a systematic error."""
    edge_index = edge_index.cpu()
    p = od.params_from_module(gconv_nn, dtype=torch.float64)
    z = _pre_activation(x, edge_index, p, "edge")
    v = od.activation(z, act, p.get("slope"))
    sign = torch.ones_like(z[:, :, :1, :1])
    if norm is not None and str(norm).lower() == "batch":
        sign = torch.sign(p["norm"]["weight"]).to(v.dtype).view(1, -1, 1, 1)
    v = v * sign
    top, arg = v.max(-1, keepdim=True)
    close = (top - v) < TIE_REL * top.abs().clamp_min(1.0)
    flat = (z < -TIE_REL * z.abs().clamp_min(1.0)) if str(act).lower() == "relu" else torch.zeros_like(close)
    tie = (close.sum(-1, keepdim=True) > 1) & (close & ~flat).any(-1, keepdim=True) & (sign != 0)
    mask = tie | _kink(z.gather(-1, arg), act)
    frac = mask.double().mean().item()
    assert frac <= MAX_MASKED, "near-tie mask covers %.2e of the entries" % frac
    return mask


def assert_no_mr_ties(x, edge_index, gconv_nn=None, act=None):
    """MRConv precondition: every (b, c, i) has a top-two gap of x_j - x_i of at least MR_TIE_REL relative, so
    an fp32 difference of the fp32 inputs ranks the edges as fp64 does.  With the layer's parameters, also no
    node-level pre-activation within MR_TIE_REL of the activation's kink."""
    edge_index = edge_index.cpu()
    xd = x.detach().cpu().double()
    v = od.batched_index_select(xd, edge_index[0]) - od.batched_index_select(xd, edge_index[1])
    if v.shape[-1] > 1:
        top2 = v.topk(2, dim=-1).values
        gap = top2[..., 0] - top2[..., 1]
        n = int((gap < MR_TIE_REL * top2[..., 0].abs().clamp_min(1.0)).sum())
        assert n == 0, "%d MRConv max near-ties: pick another seed" % n
    if gconv_nn is not None and act is not None and str(act).lower() != "none":
        z = _pre_activation(x, edge_index, od.params_from_module(gconv_nn, dtype=torch.float64), "mr")
        n = int((z.abs() < MR_TIE_REL * z.abs().clamp_min(1.0)).sum())
        assert n == 0, "%d MRConv pre-activations at the kink: pick another seed" % n


def oracle_grads(x, edge_index, gconv_nn, conv, act, norm, training, grad_out, knn=None, skip=None):
    """fp64 autograd of oracle.dense.graph_conv on `edge_index` (the graph the kernel used; with `knn`, a dict of
    check_graph's arguments, it is first adjudicated against the oracle's own kNN).  skip: None, a float
    (ResDynBlock2d: body(x) + x * skip) or "cat" (DenseDynBlock2d: cat(x, body(x))).
    Returns (output, {x, weight, bias, bn_w, bn_b, slope: gradient}) in fp64, only the entries that exist."""
    edge_index = edge_index.cpu()
    if knn is not None:
        check_graph(x, edge_index[0], **knn)
    p = od.params_from_module(gconv_nn, dtype=torch.float64)
    leaves = {"x": x.detach().cpu().double().requires_grad_(True), "weight": p["weight"].requires_grad_(True)}
    if "bias" in p:
        leaves["bias"] = p["bias"].requires_grad_(True)
    if "slope" in p:
        leaves["slope"] = p["slope"].requires_grad_(True)
    if "norm" in p:
        leaves["bn_w"] = p["norm"]["weight"].requires_grad_(True)
        leaves["bn_b"] = p["norm"]["bias"].requires_grad_(True)
    y = od.graph_conv(leaves["x"], edge_index, p, conv, act, norm, training)
    if skip == "cat":
        y = torch.cat((leaves["x"], y), 1)
    elif skip is not None:
        y = y + leaves["x"] * skip
    (y * grad_out.double()).sum().backward()
    return y.detach(), {k: v.grad for k, v in leaves.items()}


def kernel_names(fn, attempts=3):
    """(fn(), the names of the events torch.profiler recorded while it ran on the GPU), for the tests that check
    which kernel a route launched.  A capture holding fewer kernel records than the runtime's kernel launch calls
    (CUPTI can drop a session's kernel records) says nothing about the route: fn is run and captured again, up to
    `attempts` times, and the last capture is returned whatever it holds."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    for _ in range(attempts):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        ev = prof.events()
        launches = sum(1 for e in ev if e.device_type == DeviceType.CPU and "LaunchKernel" in e.name)
        kernels = sum(1 for e in ev if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memset", "Memcpy")))
        if kernels >= launches:
            break
    return res, {e.key for e in prof.key_averages()}


def assert_grads_close(name, got, ref, atol_frac=ATOL_FRAC, rtol=RTOL, floor=0.0, slack=0.0):
    """Elementwise |got - ref| <= atol_frac * max(max|ref|, floor) + rtol * |ref| + slack (slack: a tensor of ref's
    shape, or 0).  Returns the worst |got - ref| / max|ref|; on failure names the tensor, the worst index and both
    values."""
    got = got.detach().cpu().double().reshape(ref.shape)
    ref = ref.detach().cpu().double()
    scale = ref.abs().max().clamp_min(1e-30)
    err = (got - ref).abs()
    bound = atol_frac * max(float(scale), floor) + rtol * ref.abs() + (slack.detach().cpu().double()
                                                                       if torch.is_tensor(slack) else slack)
    worst = int((err / bound).argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ref.shape))
    ratio = float(err.max() / scale)
    assert bool((err <= bound).all()), (
        "%s: %d of %d elements out of tolerance; worst at %s: got %.6g, ref %.6g (|err|/max|ref| = %.3e, "
        "max |err|/max|ref| = %.3e)" % (name, int((err > bound).sum()), ref.numel(), idx, float(got[idx]),
                                        float(ref[idx]), float(err[idx] / scale), ratio))
    return ratio
