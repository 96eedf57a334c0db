"""A float64 per-element error bound of the fused MLP forward (test infrastructure).

`forward_bound` returns the float64 reference of raw = [rgb, sigma, semantic, instance] and of the trunk output h,
each with a bound B of the same shape: what the kernel computes differs from the reference by at most B, element by
element.  The bound follows the kernel's program (mlp_program.h, pnr_api.cu): the trunk with its skip concatenation,
the sigma head on the CUDA cores, the view layer with feature_linear folded into it, the rgb head on the CUDA cores,
and the semantic / instance heads.

Local terms.  Every layer adds a local error at its output, bounded by

    split term + accumulation term   (+ |W| k_in for the kink units of its input, see below).

Split term.  The 16-bit operand parts of x leave a residual r(x) (`part_residual`; tests/test_cpu_operand_split.py
checks it against the bytes):
    fp16x3  max(2^-23 |x|, 2^-25)     bf16x3  2^-17 |x|
    fp16    max(2^-11 |x|, 2^-25)     bf16    2^-8 |x|
The fp16 floor is half the subnormal spacing 2^-24.  A product w h computed as (w_hi + w_lo)(h_hi + h_lo) - w_lo h_lo
(x3) or w_hi h_hi (1 pass) differs from w h by at most
    |w| r(h) + r(w) |h| + r(w) r(h) [+ |w_lo| |h_lo| in the x3 modes],   |x_lo| <= r1(x) + r(x),
with r1 the residual of hi alone, and |h| <= |h_ref| + E_in for the kernel's operand.

Accumulation term.  c 2^-23 (|W| |h| + |b|), c = the fp32 additions on the longest path of an output: one per wgmma
(passes x K16 steps) plus the bias add of the epilogue; K + 1 for the CUDA-core dot products of the sigma and rgb
heads.  A unit of 2^-23 covers an adder that truncates as well as one that rounds to nearest.  acc=False drops the
term: the bound of a replay that accumulates exactly (test_cpu_program.replay).

Propagation.  Every layer is linear, so the kernel's pre-activation error is exactly W (the error of its input) plus
its local error.  The error of every unit is kept as a sum over SOURCES (the encoder inputs, each layer's local
error) of a per-sample matrix times the source: e = sum_s A_s sigma_s with |sigma_s| <= delta_s, so
E = sum_s |A_s| delta_s.  The signs of W stay in A_s: errors that cancel through a layer are not counted twice, which
is what keeps the bound within a small factor of the real error through a deep network (|W| e_in per layer
compounds the worst case at every layer and loses three orders of magnitude in three layers).  The ReLU of a unit
whose reference pre-activation clears its bound (|pre| > E) takes the same branch in the kernel: its slope, 0 or 1,
is exact.  A unit within E of its kink may take either branch: its output error is s e for some s in [0, 1], i.e.
e / 2 + (s - 1/2) e, so it stays in the sums with slope 1/2 and adds k = E / 2 on those units, which enters the next
layer as the local term |W| k.

Encoder inputs.  h(x): exact (the fp32 oracle encoder is bit-identical to the kernel's).  gamma(x): p itself is exact;
each sin / cos of the exact fp32 argument p 2^k is within CUDA's documented 2 ulp of sincosf.  gamma(d) in rays mode
also carries the error of d / |d| formed in the kernel (`VIEWDIR_REL`).

BACKWARD (`backward_bound`: pnr_mlp_backward_trunk, the stash it writes and d(trunk input)), pinned to the kernel's D
ReLU masks M_i, so there are no kink terms: every slope is the mask's exact 0 or 1.  The kernel works in units scaled by
grad_scale = gs (a power of two: the scaling and the stash's unscaling are exact), and so does the model:
  Last layer.  g_{D-1} = gs dZ_{D-1} = M_{D-1} (gs grad_h), exact.
  Step l.  acc = g_l W_l^T over the h columns of layer l's input (and, at layer 0 and the skip layer, over its embedded
  columns), with W_l packed transposed from the same fp32 weights: a tensor-core layer with K = W and no bias add.  Its
  local error is the split term of both operands, evaluated at the SCALED magnitude |g_l| + E (so the fp16 floor
  2^-25 is 2^-25 / gs after unscaling), plus c 2^-23 |g_l| |W_l| with c = passes x W / 16 (no bias add).  Then
  g_{l-1} = M_{l-1} acc: the error propagates through the pinned mask, the signs of W kept in the source matrices.
  d(trunk input).  The skip layer writes its embedded columns first; layer 0 adds its own to them: one fp32
  rounding of the sum, 2^-23 (|ref| + E).  Everything the kernel writes is divided by gs at the end.
With acc=False (the replay accumulates exactly) the accumulation terms and the rounding of the sum drop out.
A split whose fp16 lo part rounds toward zero still passes, in the forward as in the backward (the backward checked on
the replay, every regime and grad_h regime): twice the floor stays within bounds that count every error at its worst
sign."""
from __future__ import annotations

import torch

from oracle import reference_renderer as O

# (relative, floor) of the residual of the operand split, and of the hi part alone
PART = {"fp16x3": (2.0 ** -23, 2.0 ** -25), "bf16x3": (2.0 ** -17, 0.0), "fp16": (2.0 ** -11, 2.0 ** -25),
        "bf16": (2.0 ** -8, 0.0)}
ONE_PART = {"fp16": (2.0 ** -11, 2.0 ** -25), "bf16": (2.0 ** -8, 0.0)}
PASSES = {"fp16x3": 3, "bf16x3": 3, "fp16": 1, "bf16": 1}
U = 2.0 ** -23                  # accumulation unit (truncating or rounding fp32 adder)
SINCOS = 2.0 ** -22             # 2 ulp of a fp32 result: |err| <= 2^-22 |sin| (+ 2 ulp of the subnormals)
# d / |d| in the kernel: |d|^2 exact for the dyadic directions the tests use, then a correctly rounded sqrt and
# division: (1 + 2^-24)^2 / (1 - 2^-24) - 1 < 3 2^-24 <= 2^-22 relative per component
VIEWDIR_REL = 2.0 ** -22


def part_residual(x, precision):
    rel, floor = PART[precision]
    return torch.clamp(rel * x.abs(), min=floor)


def _lo(x, precision):
    """Bound of |lo part| (x3 modes): the residual of hi, rounded once more."""
    rel, floor = ONE_PART[precision[:4]]
    return torch.clamp(rel * x.abs(), min=floor) + part_residual(x, precision)


class Err:
    """The error of a block of units: {source: A} with A [S, N, Ns] (or a diagonal [S, N]), and k [S, N], the bound of
    the units that left the sums at a ReLU kink (0 elsewhere)."""

    def __init__(self, terms, k):
        self.terms, self.k = terms, k

    def bound(self, delta):
        E = self.k.clone()
        for s, A in self.terms.items():
            E += A.abs() * delta[s] if A.dim() == 2 else (A.abs() @ delta[s][..., None])[..., 0]
        return E


def _times(W, A):
    """W [N, K] times A ([S, K, Ns] or diagonal [S, K])."""
    return W[None] * A[:, None, :] if A.dim() == 2 else W @ A


def linear(segs, b, precision, acc, delta, name, dW=None):
    """One tensor-core layer.  segs: (W [N, K], h_ref [S, K], Err of h, bound E of h) per K segment of the operand
    (the skip layer's [gamma(x) | h], the view layer's [h | gamma(d)]).  dW: the kernel's own error of the first
    segment's weights (the fold).  b None: no bias add (a backward step).  Registers the layer's local bound as source
    `name` in delta; returns (pre-activation reference, its Err)."""
    c = 1 if b is not None else 0
    if b is None:
        b = segs[0][1].new_zeros(segs[0][0].shape[0])
    ref = b[None].clone()
    local = torch.zeros_like(ref.expand(segs[0][1].shape[0], -1)).clone()
    absh = torch.zeros_like(local)
    terms = {}
    for i, (W, h, err, E) in enumerate(segs):
        aW = W.abs() if (dW is None or i) else W.abs() + dW
        a = h.abs() + E                                    # |h| of the kernel's operand
        ref = ref + h @ W.T
        rw, ra = part_residual(aW, precision), part_residual(a, precision)
        local += ra @ aW.T + a @ rw.T + ra @ rw.T + err.k @ aW.T
        if PASSES[precision] == 3:
            local += _lo(a, precision) @ _lo(aW, precision).T
        if dW is not None and i == 0:
            local += a @ dW.T
        absh += a @ aW.T
        c += PASSES[precision] * -(-W.shape[1] // 16)
        for s, A in err.terms.items():
            terms[s] = terms[s] + _times(W, A) if s in terms else _times(W, A)
    if acc:
        local += c * U * (absh + b.abs()[None])
    delta[name] = local
    terms[name] = torch.ones_like(local)
    return ref, Err(terms, torch.zeros_like(local))


def relu(ref, err, delta, E=None):
    """ReLU of the reference and of the error: exact slopes where |ref| > E, a kink bound k = E elsewhere."""
    E = err.bound(delta) if E is None else E
    kink = ref.abs() <= E
    m = torch.where(kink, 0.5, (ref > E).to(ref.dtype))
    terms = {s: (A * m if A.dim() == 2 else A * m[..., None]) for s, A in err.terms.items()}
    return torch.relu(ref), Err(terms, torch.where(kink, 0.5 * E, torch.zeros_like(E)))


def dot_head(w, b, h, err, E, acc, delta, name):
    """A CUDA-core dot product in fp32 (the sigma and rgb heads): no operand split."""
    a = h.abs() + E
    ref = h @ w.T + b[None]
    local = err.k @ w.abs().T
    if acc:
        local = local + (w.shape[1] + 1) * U * (a @ w.abs().T + b.abs()[None])
    terms = {s: _times(w, A) for s, A in err.terms.items()}
    delta[name] = local
    terms[name] = torch.ones_like(local)
    return ref, Err(terms, torch.zeros_like(local))


def encoding(pts, L):
    """gamma(p) in float64 of the fp32 points and the kernel's error of each column."""
    ex = O.embed(pts.double(), L)
    e = SINCOS * ex.abs() + 2.0 ** -148
    e[:, :3] = 0.0
    return ex, e


def view_encoding(vd, L, rel=0.0):
    """gamma(d) in float64 of the directions (fp32 inputs, or d / |d| in float64 in rays mode) and the kernel's error
    of each column: sincosf's 2 ulp, plus 2^k rel |d_c| when the kernel forms d / |d| (sin and cos are 1-Lipschitz)."""
    v = vd.double()
    ed = O.embed(v, L)
    ev = rel * v.abs()
    e = [ev] + [ev * 2.0 ** (k // 2) + SINCOS * ed[:, 3 + 3 * k:6 + 3 * k].abs() + 2.0 ** -148 for k in range(2 * L)]
    return ed, torch.cat(e, 1)


def _p(m, dev):
    return m.weight.detach().to(dev, torch.float64), m.bias.detach().to(dev, torch.float64)


def forward_bound(net, precision, ex, e_ex, ed, e_ed, acc=True, chunk=1024):
    """(raw reference [S, 4+C+K], its bound, trunk output reference h [S, W], its bound), float64 on ex's device, for
    the product network `net` fed the trunk input ex and gamma(d) ed that the kernel sees to within e_ex / e_ed."""
    parts = [_forward_bound(net, precision, ex[i:i + chunk], e_ex[i:i + chunk], ed[i:i + chunk], e_ed[i:i + chunk], acc)
             for i in range(0, ex.shape[0], chunk)]
    return tuple(torch.cat(t, 0) for t in zip(*parts))


def _trunk(net, precision, ex, e_ex, acc, delta):
    """The trunk's forward layers: (h, its Err, its bound E, [(pre_i, E_pre_i, H_i, E_H_i)] per layer i): the reference
    pre-activation, the bound of the kernel's pre-activation, the reference activation relu(pre_i) and the bound of
    the kernel's activation.  Registers source "x" (the trunk input's error e_ex) in delta."""
    skip, dev = len(net.pts_linears) // 2, ex.device
    delta["x"] = e_ex
    x_err = Err({"x": torch.ones_like(ex)}, torch.zeros_like(ex))
    h, err, E = ex, x_err, e_ex
    layers = []
    for i, lin in enumerate(net.pts_linears):
        W, b = _p(lin, dev)
        segs = ([(W, h, err, E)] if i != skip + 1 else
                [(W[:, :ex.shape[1]], ex, x_err, e_ex), (W[:, ex.shape[1]:], h, err, E)])
        pre, pre_err = linear(segs, b, precision, acc, delta, f"L{i}")
        E_pre = pre_err.bound(delta)
        h, err = relu(pre, pre_err, delta, E_pre)
        E = err.bound(delta)
        layers.append((pre, E_pre, h, E))
    return h, err, E, layers


def _forward_bound(net, precision, ex, e_ex, ed, e_ed, acc):
    dev = ex.device
    delta = {"d": e_ed}
    d_err = Err({"d": torch.ones_like(ed)}, torch.zeros_like(ed))
    h, err, E, _ = _trunk(net, precision, ex, e_ex, acc, delta)
    sig, sig_err = dot_head(*_p(net.alpha_linear, dev), h, err, E, acc, delta, "sigma")
    # view layer: [W_view_h W_feat | W_view_d] [h | gamma(d)] + W_view_h b_feat + b_view, the fold rounded to fp32 from
    # a double sum: 2^-24 of |W_view_h| |W_feat| for the rounding, the double sum's error far below the other 2^-24
    Wf, bf = _p(net.feature_linear, dev)
    Wv, bv = _p(net.views_linears[0], dev)
    Wvh, Wvd = Wv[:, :Wf.shape[0]], Wv[:, Wf.shape[0]:]
    fold, dfold = Wvh @ Wf, 2.0 ** -23 * (Wvh.abs() @ Wf.abs())
    bfold = Wvh @ bf + bv
    v, v_err = linear([(fold, h, err, E), (Wvd, ed, d_err, e_ed)], bfold, precision, acc, delta, "view", dW=dfold)
    delta["view"] = delta["view"] + 2.0 ** -23 * (Wvh.abs() @ bf.abs() + bv.abs())[None]   # the folded bias
    v, v_err = relu(v, v_err, delta)
    rgb, rgb_err = dot_head(*_p(net.rgb_linear, dev), v, v_err, v_err.bound(delta), acc, delta, "rgb")
    outs, bounds = [rgb, sig], [rgb_err.bound(delta), sig_err.bound(delta)]
    for name in ("semantic_linears", "instance_linears"):
        if hasattr(net, name):
            (W1, b1), (W2, b2) = (_p(m, dev) for m in getattr(net, name))
            g, g_err = relu(*linear([(W1, h, err, E)], b1, precision, acc, delta, name + "0"), delta)
            logit, l_err = linear([(W2, g, g_err, g_err.bound(delta))], b2, precision, acc, delta, name + "1")
            outs.append(logit)
            bounds.append(l_err.bound(delta))
    return torch.cat(outs, 1), torch.cat(bounds, 1), h, E


def backward_bound(net, precision, ex, e_ex, grad_h, grad_scale, masks, acc=True, chunk=1024):
    """The trunk backward (pnr_mlp_backward_trunk) pinned to the kernel's ReLU masks (masks[i] [S, W], 0 / 1: layer
    i's pattern; the last one gates grad_h).  Returns a dict of float64 tensors on ex's device:
        pre, E_pre, H, E_H: per trunk layer, the forward side (_trunk): reference pre-activation and activation, and
                            the bounds of the kernel's (what the stash's H_i slots and the masks are checked against);
        dZ, B_dZ:           per trunk layer j, the reference gradient w.r.t. its pre-activation and the bound of the
                            kernel's (the stash's dZ_j slots);
        d_in, B_in:         d(trunk input) [S, E] and its bound.
    The model: BACKWARD in the module docstring."""
    out = {}
    for i in range(0, ex.shape[0], chunk):
        sl = slice(i, i + chunk)
        part = _backward_bound(net, precision, ex[sl], e_ex[sl], grad_h[sl], grad_scale, [m[sl] for m in masks], acc)
        for k, v in part.items():
            out.setdefault(k, []).append(v)
    return {k: ([torch.cat(t, 0) for t in zip(*v)] if isinstance(v[0], list) else torch.cat(v, 0)) for k, v in out.items()}


def _masked(err, M):
    return Err({s: (A * M if A.dim() == 2 else A * M[..., None]) for s, A in err.terms.items()}, err.k * M)


def _backward_bound(net, precision, ex, e_ex, grad_h, gs, masks, acc):
    D, skip, dev = len(net.pts_linears), len(net.pts_linears) // 2, ex.device
    Ex = ex.shape[1]
    _, _, _, layers = _trunk(net, precision, ex, e_ex, acc, {})
    delta = {}
    M = [m.to(dev, torch.float64) for m in masks]
    # scaled units throughout (the kernel's operands): g_{D-1} = M_{D-1} grad_h gs, exact
    g = M[D - 1] * grad_h.to(dev, torch.float64) * gs
    err = Err({}, torch.zeros_like(g))
    E = torch.zeros_like(g)
    dZ, B = [None] * D, [None] * D
    dZ[D - 1], B[D - 1] = g / gs, E.clone()
    parts = []                       # the d(trunk input) contributions: the skip layer's first, then layer 0's
    for l in range(D - 1, -1, -1):
        W = _p(net.pts_linears[l], dev)[0]
        if l == 0 or l == skip + 1:
            parts.append(linear([(W[:, :Ex].T, g, err, E)], None, precision, acc, delta, f"g{l}x"))
        if l == 0:
            break
        ref, e = linear([(W[:, Ex:].T if l == skip + 1 else W.T, g, err, E)], None, precision, acc, delta, f"g{l}")
        g, err = ref * M[l - 1], _masked(e, M[l - 1])
        E = err.bound(delta)
        dZ[l - 1], B[l - 1] = g / gs, E / gs
    ref, err = parts[0]
    if len(parts) == 2:              # layer 0's contribution added to the skip layer's: one fp32 rounding of the sum
        ref1, err1 = parts[1]
        ref = ref + ref1
        terms = dict(err.terms)
        for s, A in err1.terms.items():
            terms[s] = terms[s] + A if s in terms else A
        err = Err(terms, err.k + err1.k)
        if acc:
            delta["sum"] = U * (ref.abs() + err.bound(delta))
            err.terms["sum"] = torch.ones_like(ref)
    return {"pre": [t[0] for t in layers], "E_pre": [t[1] for t in layers], "H": [t[2] for t in layers],
            "E_H": [t[3] for t in layers], "dZ": dZ, "B_dZ": B, "d_in": ref / gs, "B_in": err.bound(delta) / gs}


# ------------------------------------------------------------------------------------------------ pnr_wgrad
WGRAD_U = {"fp16x3": 2.0 ** -11, "bf16x3": 2.0 ** -8}    # unit roundoff of one 16-bit operand part
WGRAD_RUN_SLABS = 16                                    # slabs of 64 samples per run of pnr_wgrad's register accumulators


def wgrad_slabs_per_cta(S, No, sms):
    """(64-sample slabs per CTA, CTAs per column block) of one pnr_wgrad call on a device with `sms` SMs."""
    mh = 2 if No > 128 else 1
    slabs = -(-S // 64)
    G = max(1, min(slabs, max(sms // mh, 1)))
    return -(-slabs // G), G


def wgrad_tau(prec, S, No, sms):
    """tau of one pnr_wgrad call (tests/test_gpu_train_limits.py): the operand split, 3 products x 4 k-steps per slab
    accumulated in one run, and the round-to-nearest adds of the runs and of the CTAs' partials."""
    per_cta, G = wgrad_slabs_per_cta(S, No, sms)
    runs = -(-per_cta // WGRAD_RUN_SLABS)
    return 3 * WGRAD_U[prec] ** 2 + 12 * min(per_cta, WGRAD_RUN_SLABS) * 2.0 ** -23 + 4 * (runs + G) ** 0.5 * 2.0 ** -24


def wgrad_bound(A, ab, cx, S, No, prec, sc, sms):
    """pnr_wgrad's per-element bound of dW = dZ^T X and db = column sums of dZ, from the operands it was given:
    A = |dZ|^T |X|, ab = column sums of |dZ|, cx = column sums of |X|; sc = the dz_scale it ran with (1: none).
    dW: tau A + floor, the floor 2^-24 (cx / sc + ab) in fp16x3 where a 16-bit part can be subnormal; db: 2^-24 (S + 64) ab."""
    bW = wgrad_tau(prec, S, No, sms) * A
    if prec == "fp16x3":
        bW = bW + 2.0 ** -24 * (cx[None, :] / sc + ab[:, None])
    return bW, 2.0 ** -24 * (S + 64) * ab


# ------------------------------------------------------------------------------------------------ regimes
def twin(net, layer, k):
    """Scale trunk layer `layer`'s W and b by 2^-k and every weight column that reads its output by 2^k (the next trunk
    layer's h columns, or alpha / feature / the head hidden layers after the last).  ReLU is positively homogeneous, so
    in float64 the network computes the same function bit for bit; the kernel sees that layer's operands 2^k smaller
    (k > 0) or larger (k < 0)."""
    D, skip = len(net.pts_linears), len(net.pts_linears) // 2
    s = 2.0 ** -k
    with torch.no_grad():
        net.pts_linears[layer].weight.mul_(s)
        net.pts_linears[layer].bias.mul_(s)
        if layer < D - 1:
            nxt = net.pts_linears[layer + 1].weight
            E = nxt.shape[1] - net.pts_linears[layer].weight.shape[0]
            nxt[:, E if layer == skip else 0:].div_(s)
        else:
            for m in [net.alpha_linear, net.feature_linear] + [getattr(net, n)[0] for n in ("semantic_linears", "instance_linears")
                                                               if hasattr(net, n)]:
                m.weight.div_(s)
    return net
