"""CPU oracle for the normflows coupling-stack hot path.  TEST INFRASTRUCTURE ONLY.

This file is a numpy restatement of the reference algorithm (normflows 1.7.3,
commit c6616b1a) for the density / sampling pass over stacked coupling layers.
It exists to CHECK the CUDA product path; nothing under `normalizing-flows_b200/`
imports it.  Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s
`cpu_baseline` / `--impl reference` leg may import it.

Pinned against the real reference: `tests/golden/make_golden.py` imports the
reference package from its checkout (oracle/reference.py), dumps state_dicts + inputs + outputs
(fp64 and fp32) to `tests/golden/*.npz`, and `tests/test_oracle_golden.py`
replays every fixture through this file (fp64: rtol 1e-12, fp32: rtol 2e-5).

Every function cites the reference file:line it restates (paths relative to
the reference's normflows/ package).  The restatement is mask-free: where the reference
uses boolean-mask indexing (utils/splines.py:40-41,77-95) it evaluates every
element and selects with `where`, which is the formulation the CUDA kernels use.

A model is described by (spec, sd):
  spec = {"kind": "NormalizingFlow", "q0": {...}, "flows": [ {...}, ... ]}
  sd   = the reference `state_dict()` as {key: np.ndarray}
"""
import math

import numpy as np

MIN_BIN_WIDTH = 1e-3  # utils/splines.py:6
MIN_BIN_HEIGHT = 1e-3  # utils/splines.py:7
MIN_DERIVATIVE = 1e-3  # utils/splines.py:8


# --------------------------------------------------------------------------
# elementwise helpers (ATen semantics)
# --------------------------------------------------------------------------
def softplus(x):
    """F.softplus(beta=1, threshold=20): x if x > 20 else log1p(exp(x))."""
    x = np.asarray(x)
    safe = np.minimum(x, 20.0)
    return np.where(x > 20.0, x, np.log1p(np.exp(safe))).astype(x.dtype)


def softmax(x, axis=-1):
    m = np.max(x, axis=axis, keepdims=True)
    e = np.exp(x - m)
    return e / np.sum(e, axis=axis, keepdims=True)


def sigmoid(x):
    return (1.0 / (1.0 + np.exp(-x))).astype(x.dtype)


def leaky_relu(x, slope):
    return np.where(x >= 0, x, x * np.asarray(slope, dtype=x.dtype)).astype(x.dtype)


def linear(x, w, b=None):
    y = x @ w.T
    if b is not None:
        y = y + b
    return y


# --------------------------------------------------------------------------
# rational-quadratic spline  (utils/splines.py)
# --------------------------------------------------------------------------
def _knots(un, lo, hi, min_size):
    """softmax -> min size -> cumsum -> pad -> rescale -> pin ends -> diff.
    utils/splines.py:126-136 (widths) and :140-152 (heights)."""
    k = un.shape[-1]
    s = softmax(un, axis=-1)
    s = min_size + (1 - min_size * k) * s
    cum = np.cumsum(s, axis=-1, dtype=un.dtype)
    cum = np.concatenate([np.zeros_like(cum[..., :1]), cum], axis=-1)
    if np.ndim(lo) > 0:  # per-element bounds (:130-131, :145-148: the `lim_tensor` branch)
        lo, hi = np.asarray(lo)[..., None], np.asarray(hi)[..., None]
        cum = (hi - lo) * cum + lo
        cum[..., 0] = lo[..., 0]
        cum[..., -1] = hi[..., 0]
    else:
        cum = (hi - lo) * cum + lo
        cum[..., 0] = lo
        cum[..., -1] = hi
    size = cum[..., 1:] - cum[..., :-1]
    return cum.astype(un.dtype), size.astype(un.dtype)


def _gather(a, idx):
    return np.take_along_axis(a, idx[..., None], axis=-1)[..., 0]


def rational_quadratic_spline(x, uw, uh, ud, inverse=False, left=0.0, right=1.0,
                              bottom=0.0, top=1.0):
    """utils/splines.py:100-219.  `ud` has K+1 entries (boundary derivatives included).
    x must lie inside [left,right] (forward) / [bottom,top] (inverse)."""
    k = uw.shape[-1]
    if MIN_BIN_WIDTH * k > 1.0:
        raise ValueError("Minimal bin width too large for the number of bins")
    if MIN_BIN_HEIGHT * k > 1.0:
        raise ValueError("Minimal bin height too large for the number of bins")
    dt = x.dtype
    cumw, w = _knots(uw, left, right, MIN_BIN_WIDTH)
    cumh, h = _knots(uh, bottom, top, MIN_BIN_HEIGHT)
    d = (MIN_DERIVATIVE + softplus(ud)).astype(dt)  # :138

    # searchsorted, :11-13 -- eps is added to the LAST knot only, comparison is >=
    loc = (cumh if inverse else cumw).copy()
    loc[..., -1] += np.asarray(1e-6, dtype=dt)
    idx = np.sum(x[..., None] >= loc, axis=-1) - 1
    idx = np.clip(idx, 0, k - 1)  # only reachable for out-of-interval x, which callers mask

    in_cumw = _gather(cumw, idx)
    in_w = _gather(w, idx)
    in_cumh = _gather(cumh, idx)
    delta = h / w
    in_delta = _gather(delta, idx)
    in_d = _gather(d, idx)
    in_d1 = _gather(d[..., 1:], idx)
    in_h = _gather(h, idx)

    if inverse:  # :172-198
        t = (x - in_cumh)
        s = in_d + in_d1 - 2 * in_delta
        a = t * s + in_h * (in_delta - in_d)
        b = in_h * in_d - t * s
        c = -in_delta * t
        disc = b * b - 4 * a * c
        root = (2 * c) / (-b - np.sqrt(disc))
        out = root * in_w + in_cumw
        tomt = root * (1 - root)
        den = in_delta + s * tomt
        dnum = in_delta ** 2 * (in_d1 * root ** 2 + 2 * in_delta * tomt + in_d * (1 - root) ** 2)
        lad = np.log(dnum) - 2 * np.log(den)
        return out.astype(dt), (-lad).astype(dt)
    theta = (x - in_cumw) / in_w  # :200-219
    tomt = theta * (1 - theta)
    num = in_h * (in_delta * theta ** 2 + in_d * tomt)
    den = in_delta + (in_d + in_d1 - 2 * in_delta) * tomt
    out = in_cumh + num / den
    dnum = in_delta ** 2 * (in_d1 * theta ** 2 + 2 * in_delta * tomt + in_d * (1 - theta) ** 2)
    lad = np.log(dnum) - 2 * np.log(den)
    return out.astype(dt), lad.astype(dt)


def unconstrained_rqs(x, uw, uh, ud, inverse=False, tail_bound=1.0):
    """utils/splines.py:16-97 with tails='linear'.  `ud` has K-1 entries; the two
    boundary derivatives are the constant log(exp(1-1e-3)-1) (:35-38).  Elements
    outside [-B,B] pass through with logabsdet 0 (:40-41); NaN is 'outside'."""
    dt = x.dtype
    inside = (x >= -tail_bound) & (x <= tail_bound)
    const = np.asarray(np.log(np.exp(1 - MIN_DERIVATIVE) - 1), dtype=dt)
    pad = np.full(ud.shape[:-1] + (1,), const, dtype=dt)
    ud_full = np.concatenate([pad, ud.astype(dt), pad], axis=-1)
    xs = np.where(inside, x, np.zeros_like(x))  # any in-range value; result discarded
    with np.errstate(all="ignore"):
        y, lad = rational_quadratic_spline(xs, uw, uh, ud_full, inverse=inverse,
                                           left=-tail_bound, right=tail_bound,
                                           bottom=-tail_bound, top=tail_bound)
    y = np.where(inside, y, x).astype(dt)
    lad = np.where(inside, lad, np.zeros_like(lad)).astype(dt)
    return y, lad


# --------------------------------------------------------------------------
# conditioner nets
# --------------------------------------------------------------------------
def _num_blocks(sd, p):
    n = 0
    while f"{p}blocks.{n}.linear_layers.0.weight" in sd:
        n += 1
    return n


def residual_net(x, sd, p):
    """nets/resnet.py:92-104 with ResidualBlock :37-50 (pre-activation ReLU blocks,
    no batch-norm, dropout p=0, no context)."""
    h = linear(x, sd[p + "initial_layer.weight"], sd[p + "initial_layer.bias"])
    for n in range(_num_blocks(sd, p)):
        q = f"{p}blocks.{n}.linear_layers."
        t = np.maximum(h, 0)
        t = linear(t, sd[q + "0.weight"], sd[q + "0.bias"])
        t = np.maximum(t, 0)
        t = linear(t, sd[q + "1.weight"], sd[q + "1.bias"])
        h = h + t
    return linear(h, sd[p + "final_layer.weight"], sd[p + "final_layer.bias"])


def made(x, sd, p):
    """nets/made.py:296-304; MaskedLinear.forward :80-81 (W*mask every call);
    MaskedResidualBlock.forward :199-214."""
    def ml(v, q):
        return linear(v, sd[q + "weight"] * sd[q + "mask"].astype(v.dtype), sd[q + "bias"])
    h = ml(x, p + "initial_layer.")
    for n in range(_num_blocks(sd, p)):
        q = f"{p}blocks.{n}.linear_layers."
        t = np.maximum(h, 0)
        t = ml(t, q + "0.")
        t = np.maximum(t, 0)
        t = ml(t, q + "1.")
        h = h + t
    return ml(h, p + "final_layer.")


def mlp(x, sd, p, leaky=0.0):
    """nets/mlp.py:34-58: Linear/LeakyReLU stack, last layer linear (no output_fn)."""
    idx = sorted({int(k[len(p + "net."):].split(".")[0]) for k in sd if k.startswith(p + "net.")})
    for j, i in enumerate(idx):
        x = linear(x, sd[f"{p}net.{i}.weight"], sd[f"{p}net.{i}.bias"])
        if j + 1 < len(idx):
            x = leaky_relu(x, leaky)
    return x


def conv2d(x, w, b=None):
    """F.conv2d, stride 1, padding k//2 (nets/cnn.py:35-52).  x [B,C,H,W], w [O,C,k,k]."""
    bsz, c, hh, ww = x.shape
    o, _, k, _ = w.shape
    pd = k // 2
    xp = np.pad(x, ((0, 0), (0, 0), (pd, pd), (pd, pd)))
    cols = np.empty((bsz, c, k, k, hh, ww), dtype=x.dtype)
    for i in range(k):
        for j in range(k):
            cols[:, :, i, j] = xp[:, :, i:i + hh, j:j + ww]
    y = np.einsum("bcklhw,ockl->bohw", cols, w, optimize=True).astype(x.dtype)
    if b is not None:
        y = y + b[None, :, None, None]
    return y


def convnet2d(x, sd, p, leaky=0.0):
    """nets/cnn.py:33-63 without actnorm: conv/LeakyReLU stack, last conv linear."""
    idx = sorted({int(k[len(p + "net."):].split(".")[0]) for k in sd if k.startswith(p + "net.")})
    for j, i in enumerate(idx):
        x = conv2d(x, sd[f"{p}net.{i}.weight"], sd.get(f"{p}net.{i}.bias"))
        if j + 1 < len(idx):
            x = leaky_relu(x, leaky)
    return x


# --------------------------------------------------------------------------
# flow layers.  Every function returns (z', log_det[B]); `direction` is the
# reference method name: "inverse" = density pass (x -> z), "forward" = sampling.
# --------------------------------------------------------------------------
def _split_params(params, k, hidden):
    """neural_spline/coupling.py:330-336: [w|h|d] chunks of 3K-1; w,h divided by
    sqrt(hidden_features); d not scaled.  NOTE the autoregressive twin
    (neural_spline/autoregressive.py:105-107) guards the division with
    `hasattr(self.autoregressive_net, "hidden_features")`, and nets/made.py MADE never sets
    that attribute -- so the AR layer does NOT scale (hidden=None here).  Pinned by the goldens."""
    dt = params.dtype
    sc = np.asarray(1.0 if hidden is None else np.sqrt(hidden), dtype=dt)
    uw = params[..., :k] / sc
    uh = params[..., k:2 * k] / sc
    ud = params[..., 2 * k:]
    return uw, uh, ud


def ar_rqs(z, sd, p, L, direction):
    """flows/neural_spline/wrapper.py:238-244 (direction swap) ->
    flows/affine/autoregressive.py:24-38 -> neural_spline/autoregressive.py:94-128."""
    k, tb = L.get("num_bins", 8), float(L.get("tail_bound", 3.0))
    net = p + "mprqat.autoregressive_net."
    hidden = None  # MADE has no .hidden_features attribute -> no 1/sqrt(H) scaling (see _split_params)
    bsz, d = z.shape
    if direction == "inverse":  # wrapper.inverse -> Autoregressive.forward (one MADE pass)
        params = made(z, sd, net).reshape(bsz, d, 3 * k - 1)
        uw, uh, ud = _split_params(params, k, hidden)
        y, lad = unconstrained_rqs(z, uw, uh, ud, inverse=False, tail_bound=tb)
        return y, lad.sum(axis=1)
    out = np.zeros_like(z)  # wrapper.forward -> Autoregressive.inverse (D MADE passes)
    lad = None
    for _ in range(d):
        params = made(out, sd, net).reshape(bsz, d, 3 * k - 1)
        uw, uh, ud = _split_params(params, k, hidden)
        out, lad = unconstrained_rqs(z, uw, uh, ud, inverse=True, tail_bound=tb)
    return out, lad.sum(axis=1)


def coupled_rqs(z, sd, p, L, direction):
    """flows/neural_spline/wrapper.py:79-85 -> neural_spline/coupling.py:71-128
    (Coupling.forward / .inverse) with the unconditional CDF transform :221-253."""
    k, tb = L.get("num_bins", 8), float(L.get("tail_bound", 3.0))
    q = p + "prqct."
    idf = sd[q + "identity_features"].astype(np.int64)
    trf = sd[q + "transform_features"].astype(np.int64)
    hidden = sd[q + "transform_net.initial_layer.weight"].shape[0]
    bsz = z.shape[0]
    ident, trans = z[:, idf], z[:, trf]
    u = q + "unconditional_transform."
    bc = lambda a: np.broadcast_to(a[None], (bsz,) + a.shape).astype(z.dtype)
    uuw, uuh, uud = bc(sd[u + "unnormalized_widths"]), bc(sd[u + "unnormalized_heights"]), \
        bc(sd[u + "unnormalized_derivatives"])
    if direction == "inverse":  # prqct.forward: net sees the RAW identity split
        params = residual_net(ident, sd, q + "transform_net.").reshape(bsz, len(trf), 3 * k - 1)
        uw, uh, ud = _split_params(params, k, hidden)
        yt, lad = unconstrained_rqs(trans, uw, uh, ud, inverse=False, tail_bound=tb)
        yi, lad_i = unconstrained_rqs(ident, uuw, uuh, uud, inverse=False, tail_bound=tb)
        ld = lad.sum(axis=1) + lad_i.sum(axis=1)
    else:  # prqct.inverse: unconditional inverse FIRST, net sees the transformed identity
        yi, lad_i = unconstrained_rqs(ident, uuw, uuh, uud, inverse=True, tail_bound=tb)
        params = residual_net(yi, sd, q + "transform_net.").reshape(bsz, len(trf), 3 * k - 1)
        uw, uh, ud = _split_params(params, k, hidden)
        yt, lad = unconstrained_rqs(trans, uw, uh, ud, inverse=True, tail_bound=tb)
        ld = lad_i.sum(axis=1) + lad.sum(axis=1)
    out = np.empty_like(z)
    out[:, idf] = yi
    out[:, trf] = yt
    return out, ld


def unconstrained_rqs_tails(x, uw, uh, ud, circular, inverse=False, tail_bound=1.0):
    """utils/splines.py:16-97 with `tails` given as a list (:48-57): `ud` has K+1 entries per element; features with
    linear tails overwrite entries 0 and K with the constant of :35-38, circular features copy entry 0 into entry K.
    `circular`: bool [features]; `tail_bound`: scalar or [features] (broadcast_to, :61-66).  x: [B, features]."""
    dt = x.dtype
    tb = np.broadcast_to(np.asarray(tail_bound, dtype=dt), x.shape)
    inside = (x >= -tb) & (x <= tb)
    const = np.asarray(np.log(np.exp(1 - MIN_DERIVATIVE) - 1), dtype=dt)
    udf = ud.astype(dt).copy()
    circ = np.asarray(circular, dtype=bool)
    udf[..., ~circ, 0] = const
    udf[..., ~circ, -1] = const
    udf[..., circ, -1] = udf[..., circ, 0]
    xs = np.where(inside, x, np.zeros_like(x))
    with np.errstate(all="ignore"):
        y, lad = rational_quadratic_spline(xs, uw, uh, udf, inverse=inverse, left=-tb, right=tb, bottom=-tb, top=tb)
    # NOTE (:48-57): the list branch never copies the out-of-interval inputs into `outputs`, which therefore keeps the
    # zeros it was created with (:31) -- unlike the "linear" / "circular" string branches (:40-41, :46-47).  Restated as is.
    return np.where(inside, y, np.zeros_like(x)).astype(dt), np.where(inside, lad, np.zeros_like(lad)).astype(dt)


def periodic_features_elementwise(x, sd, p):
    """utils/nn.py:120-130 PeriodicFeaturesElementwise.forward (no bias, identity activation): features `ind` become
    w0 sin(scale f) + w1 cos(scale f), the rest pass through; order restored by inv_perm."""
    ind = sd[p + "ind"].astype(np.int64)
    ind_ = sd[p + "ind_"].astype(np.int64)
    inv = sd[p + "inv_perm"].astype(np.int64)
    w = sd[p + "weights"]
    scale = sd[p + "scale"] if p + "scale" in sd else None
    return ind, ind_, inv, w, scale


def _periodic(x, sd, p, scale_default):
    ind, ind_, inv, w, scale = periodic_features_elementwise(x, sd, p)
    sc = np.asarray(scale_default if scale is None else scale, dtype=x.dtype)
    a = sc * x[..., ind]
    per = w[:, 0].astype(x.dtype) * np.sin(a) + w[:, 1].astype(x.dtype) * np.cos(a)
    out = np.concatenate([per, x[..., ind_]], axis=-1)
    return out[..., inv]


def _tails_of(L, idx):
    circ_all = np.zeros(L["features"], dtype=bool)
    circ_all[np.asarray(L["ind_circ"], dtype=np.int64)] = True
    return circ_all[idx]


def circular_coupled_rqs(z, sd, p, L, direction):
    """flows/neural_spline/wrapper.py:88-183 (CircularCoupledRationalQuadraticSpline) -> neural_spline/coupling.py:
    71-128, 262-362 with tails as a per-feature list, PeriodicFeaturesElementwise in front of the ResidualNet
    (wrapper.py:140-147) and the unconditional CDF with the identity features' tails (coupling.py:293-303)."""
    k = L.get("num_bins", 8)
    q = p + "prqct."
    idf = sd[q + "identity_features"].astype(np.int64)
    trf = sd[q + "transform_features"].astype(np.int64)
    hidden = sd[q + "transform_net.initial_layer.weight"].shape[0]
    bsz = z.shape[0]
    tb_all = np.asarray(L.get("tail_bound", 3.0), dtype=np.float64)
    tb_tr = tb_all[trf] if tb_all.ndim else tb_all
    tb_id = tb_all[idf] if tb_all.ndim else tb_all
    circ_tr, circ_id = _tails_of(L, trf), _tails_of(L, idf)
    pre = q + "transform_net.preprocessing."
    has_pre = (pre + "weights") in sd
    # scale of the periodic features: pi / tail_bound of the circular identity features (wrapper.py:134-138)
    ind_circ_id = [i for i, f in enumerate(idf) if f in set(L["ind_circ"])]
    scale_pf = (np.pi / tb_all[idf][ind_circ_id]) if tb_all.ndim else np.pi / float(tb_all)

    def net(v):
        if has_pre:
            v = _periodic(v, sd, pre, scale_pf)
        return residual_net(v, sd, q + "transform_net.").reshape(bsz, len(trf), 3 * k + 1)

    ident, trans = z[:, idf], z[:, trf]
    u = q + "unconditional_transform."
    bc = lambda a: np.broadcast_to(a[None], (bsz,) + a.shape).astype(z.dtype)
    uuw, uuh, uud = bc(sd[u + "unnormalized_widths"]), bc(sd[u + "unnormalized_heights"]), \
        bc(sd[u + "unnormalized_derivatives"])
    if direction == "inverse":
        uw, uh, ud = _split_params(net(ident), k, hidden)
        yt, lad = unconstrained_rqs_tails(trans, uw, uh, ud, circ_tr, inverse=False, tail_bound=tb_tr)
        yi, lad_i = unconstrained_rqs_tails(ident, uuw, uuh, uud, circ_id, inverse=False, tail_bound=tb_id)
        ld = lad.sum(axis=1) + lad_i.sum(axis=1)
    else:
        yi, lad_i = unconstrained_rqs_tails(ident, uuw, uuh, uud, circ_id, inverse=True, tail_bound=tb_id)
        uw, uh, ud = _split_params(net(yi), k, hidden)
        yt, lad = unconstrained_rqs_tails(trans, uw, uh, ud, circ_tr, inverse=True, tail_bound=tb_tr)
        ld = lad_i.sum(axis=1) + lad.sum(axis=1)
    out = np.empty_like(z)
    out[:, idf] = yi
    out[:, trf] = yt
    return out, ld


def circular_ar_rqs(z, sd, p, L, direction):
    """flows/neural_spline/wrapper.py:247-311 (CircularAutoregressiveRationalQuadraticSpline) ->
    neural_spline/autoregressive.py:94-128 with tails as a per-feature list (3K+1 parameters per feature) and
    PeriodicFeaturesElementwise in front of the MADE (autoregressive.py:44-53, nets/made.py:297)."""
    k = L.get("num_bins", 8)
    net = p + "mprqat.autoregressive_net."
    bsz, d = z.shape
    tb = np.asarray(L.get("tail_bound", 3.0), dtype=np.float64)
    circ = _tails_of(L, np.arange(d))
    scale_pf = (np.pi / tb[np.asarray(L["ind_circ"], dtype=np.int64)]) if tb.ndim else np.pi / float(tb)

    def params_of(v):
        v = _periodic(v, sd, net + "preprocessing.", scale_pf)
        return _split_params(made(v, sd, net).reshape(bsz, d, 3 * k + 1), k, None)

    if direction == "inverse":
        uw, uh, ud = params_of(z)
        y, lad = unconstrained_rqs_tails(z, uw, uh, ud, circ, inverse=False, tail_bound=tb)
        return y, lad.sum(axis=1)
    out, lad = np.zeros_like(z), None
    for _ in range(d):
        uw, uh, ud = params_of(out)
        out, lad = unconstrained_rqs_tails(z, uw, uh, ud, circ, inverse=True, tail_bound=tb)
    return out, lad.sum(axis=1)


def lu_matrices(sd, p, dt):
    """flows/mixing.py:402-412 (_create_lower_upper), :514-516 (upper_diag, eps=1e-3)."""
    ud = sd[p + "linear.unconstrained_upper_diag"].astype(dt)
    n = ud.shape[0]
    lower = np.zeros((n, n), dtype=dt)
    lower[np.tril_indices(n, -1)] = sd[p + "linear.lower_entries"]
    lower[np.diag_indices(n)] = 1.0
    upper = np.zeros((n, n), dtype=dt)
    upper[np.triu_indices(n, 1)] = sd[p + "linear.upper_entries"]
    diag = (softplus(ud) + np.asarray(1e-3, dtype=dt)).astype(dt)
    upper[np.diag_indices(n)] = diag
    return lower, upper, diag


def lu_linear_permute(z, sd, p, L, direction):
    """flows/mixing.py:555-563; _Permutation :232-247; _LULinear.forward_no_cache :414-434,
    inverse_no_cache :436-473, logabsdet :518-532."""
    dt = z.dtype
    perm = sd[p + "permutation._permutation"].astype(np.int64)
    lower, upper, diag = lu_matrices(sd, p, dt)
    bias = sd[p + "linear.bias"].astype(dt)
    lad = np.sum(np.log(diag)).astype(dt)
    ones = np.ones(z.shape[0], dtype=dt)
    if direction == "inverse":  # permute, then x U^T L^T + b
        x = z[:, perm]
        x = linear(linear(x, upper), lower, bias)
        return x.astype(dt), lad * ones
    import scipy.linalg as sla
    x = (z - bias).T
    x = sla.solve_triangular(lower, x, lower=True, unit_diagonal=True)
    x = sla.solve_triangular(upper, x, lower=False)
    x = x.T.astype(dt)
    return x[:, np.argsort(perm)], -lad * ones


def masked_affine(z, sd, p, L, direction):
    """flows/affine/coupling.py:208-229.  s/t are MLPs (or absent -> zeros)."""
    b = sd[p + "b"].astype(z.dtype)
    zm = b * z
    leaky = L.get("leaky", 0.0)
    has_s = any(k.startswith(p + "s.") for k in sd)
    has_t = any(k.startswith(p + "t.") for k in sd)
    s = mlp(zm, sd, p + "s.", leaky) if has_s else np.zeros_like(z)
    t = mlp(zm, sd, p + "t.", leaky) if has_t else np.zeros_like(z)
    s = np.where(np.isfinite(s), s, np.nan).astype(z.dtype)
    t = np.where(np.isfinite(t), t, np.nan).astype(z.dtype)
    red = tuple(range(1, z.ndim))
    if direction == "forward":
        out = zm + (1 - b) * (z * np.exp(s) + t)
        return out.astype(z.dtype), np.sum((1 - b) * s, axis=red)
    out = zm + (1 - b) * (z - t) * np.exp(-s)
    return out.astype(z.dtype), -np.sum((1 - b) * s, axis=red)


def _chunk2(z):
    """torch.chunk(2, dim=1): first chunk gets ceil(C/2) channels."""
    c = z.shape[1]
    h = (c + 1) // 2
    return z[:, :h], z[:, h:]


def affine_coupling_block(z, sd, p, L, direction):
    """flows/affine/coupling.py:253-267 (Split/AffineCoupling/Merge) ->
    AffineCoupling.forward :113-147 / .inverse :149-171; reshape.py:27-31,61-65."""
    mode = L.get("split_mode", "channel")
    smap = L.get("scale_map", "exp")
    scale = L.get("scale", True)
    a, b = _chunk2(z)
    z1, z2 = (a, b) if mode == "channel" else (b, a)
    pm = p + "flows.1.param_map."
    if L.get("net", "mlp") == "mlp":
        param = mlp(z1, sd, pm, L.get("leaky", 0.0))
    else:
        param = convnet2d(z1, sd, pm, L.get("leaky", 0.0))
    red = tuple(range(1, z.ndim))
    if not scale:
        z2 = z2 + param if direction == "forward" else z2 - param
        ld = np.zeros(z.shape[0], dtype=z.dtype)
    else:
        shift, sc = param[:, 0::2], param[:, 1::2]
        if smap == "exp":
            if direction == "forward":
                z2, ld = z2 * np.exp(sc) + shift, np.sum(sc, axis=red)
            else:
                z2, ld = (z2 - shift) * np.exp(-sc), -np.sum(sc, axis=red)
        elif smap in ("sigmoid", "sigmoid_inv"):
            sg = sigmoid(sc + 2)
            lsum = np.sum(np.log(sg), axis=red)
            if direction == "forward":
                z2, ld = (z2 / sg + shift, -lsum) if smap == "sigmoid" else (z2 * sg + shift, lsum)
            else:
                z2, ld = ((z2 - shift) * sg, lsum) if smap == "sigmoid" else ((z2 - shift) / sg, -lsum)
        else:
            raise NotImplementedError("This scale map is not implemented.")
    out = np.concatenate([z1, z2] if mode == "channel" else [z2, z1], axis=1)
    return out.astype(z.dtype), ld.astype(z.dtype)


def affine_const(z, sd, p, L, direction):
    """flows/affine/coupling.py:38-54 (AffineConstFlow; ActNorm after init,
    flows/normalization.py:19-39).  log_det is a scalar broadcast over the batch."""
    s, t = sd[p + "s"].astype(z.dtype), sd[p + "t"].astype(z.dtype)
    batch_dims = [i for i, n in enumerate(s.shape) if n == 1]
    prod = int(np.prod([z.shape[i] for i in batch_dims[1:]])) if len(batch_dims) > 1 else 1
    ones = np.ones(z.shape[0], dtype=z.dtype)
    if direction == "forward":
        return (z * np.exp(s) + t).astype(z.dtype), (prod * np.sum(s)).astype(z.dtype) * ones
    return ((z - t) * np.exp(-s)).astype(z.dtype), (-prod * np.sum(s)).astype(z.dtype) * ones


def actnorm_init(z, s_shape, direction):
    """flows/normalization.py:21-28 (forward) / :33-38 (inverse): data-dependent s,t."""
    batch_dims = tuple(i for i, n in enumerate(s_shape) if n == 1)
    std = z.std(axis=batch_dims, ddof=1, keepdims=True)
    mean = z.mean(axis=batch_dims, keepdims=True)
    if direction == "forward":
        s = -np.log(std + 1e-6)
        return s.astype(z.dtype), (-mean * np.exp(s)).astype(z.dtype)
    return np.log(std + 1e-6).astype(z.dtype), mean.astype(z.dtype)


def permute(z, sd, p, L, direction):
    """flows/mixing.py:31-54."""
    c = z.shape[1]
    if L.get("mode", "shuffle") == "shuffle":
        idx = sd[p + ("perm" if direction == "forward" else "inv_perm")].astype(np.int64)
        out = z[:, idx]
    else:
        h = c // 2 if direction == "forward" else (c + 1) // 2
        out = np.concatenate([z[:, h:], z[:, :h]], axis=1)
    return out, np.zeros(z.shape[0], dtype=z.dtype)


def inv1x1(z, sd, p, L, direction):
    """flows/mixing.py:88-133.  LU: W = P L U (inverse dir) or U^-1 L^-1 P^T (forward dir,
    inverted in fp64 :94-101); log_det = +-sum(log_S) * H * W."""
    dt = z.dtype
    c = z.shape[1]
    if (p + "log_S") in sd:
        lo = np.tril(sd[p + "L"].astype(dt), -1) + np.eye(c, dtype=dt)
        up = np.triu(sd[p + "U"].astype(dt), 1) + np.diag(sd[p + "sign_S"].astype(dt)
                                                           * np.exp(sd[p + "log_S"].astype(dt)))
        pm = sd[p + "P"].astype(dt)
        if direction == "inverse":
            w, ld = pm @ lo @ up, np.sum(sd[p + "log_S"].astype(dt))
        else:
            li = np.linalg.inv(lo.astype(np.float64)).astype(dt)
            ui = np.linalg.inv(up.astype(np.float64)).astype(dt)
            w, ld = ui @ li @ pm.T, -np.sum(sd[p + "log_S"].astype(dt))
    else:
        w0 = sd[p + "W"].astype(dt)
        sl = np.linalg.slogdet(w0.astype(np.float64))[1]
        if direction == "inverse":
            w, ld = w0, sl
        else:
            w, ld = np.linalg.inv(w0.astype(np.float64)).astype(dt), -sl
    out = np.einsum("oc,bchw->bohw", w, z, optimize=True).astype(dt)
    ld = np.asarray(ld * z.shape[2] * z.shape[3], dtype=dt)
    return out, ld * np.ones(z.shape[0], dtype=dt)


def glow_block(z, sd, p, L, direction):
    """flows/affine/glow.py:72-84: [AffineCouplingBlock, Invertible1x1Conv, ActNorm]."""
    sub = [(affine_coupling_block, dict(L, net="conv", scale_map=L.get("scale_map", "sigmoid")))]
    if z.shape[1] > 1:
        sub.append((inv1x1, L))
    sub.append((affine_const, L))
    ld = np.zeros(z.shape[0], dtype=z.dtype)
    order = range(len(sub)) if direction == "forward" else range(len(sub) - 1, -1, -1)
    for i in order:
        fn, ll = sub[i]
        z, d = fn(z, sd, f"{p}flows.{i}.", ll, direction)
        ld = ld + d
    return z, ld


def squeeze(z, sd, p, L, direction):
    """flows/reshape.py:114-128."""
    s = z.shape
    if direction == "forward":
        z = z.reshape(s[0], s[1] // 4, 2, 2, s[2], s[3]).transpose(0, 1, 4, 2, 5, 3)
        z = np.ascontiguousarray(z).reshape(s[0], s[1] // 4, 2 * s[2], 2 * s[3])
    else:
        z = z.reshape(s[0], s[1], s[2] // 2, 2, s[3] // 2, 2).transpose(0, 1, 3, 5, 2, 4)
        z = np.ascontiguousarray(z).reshape(s[0], 4 * s[1], s[2] // 2, s[3] // 2)
    return z, np.zeros(s[0], dtype=z.dtype)


LAYERS = {
    "AutoregressiveRationalQuadraticSpline": ar_rqs,
    "CoupledRationalQuadraticSpline": coupled_rqs,
    "LULinearPermute": lu_linear_permute,
    "MaskedAffineFlow": masked_affine,
    "AffineCouplingBlock": affine_coupling_block,
    "AffineConstFlow": affine_const,
    "ActNorm": affine_const,
    "Permute": permute,
    "Invertible1x1Conv": inv1x1,
    "GlowBlock": glow_block,
    "Squeeze": squeeze,
    "CircularCoupledRationalQuadraticSpline": circular_coupled_rqs,
    "CircularAutoregressiveRationalQuadraticSpline": circular_ar_rqs,
}


# --------------------------------------------------------------------------
# base distributions (log_prob only -- the tail of the density pass)
# --------------------------------------------------------------------------
def diag_gaussian_log_prob(z, sd, p):
    """distributions/base.py:94-103."""
    loc, ls = sd[p + "loc"].astype(z.dtype), sd[p + "log_scale"].astype(z.dtype)
    d = int(np.prod(loc.shape[1:]))
    red = tuple(range(1, z.ndim))
    return (-0.5 * d * np.log(2 * np.pi)
            - np.sum(ls + 0.5 * ((z - loc) / np.exp(ls)) ** 2, axis=red)).astype(z.dtype)


def class_cond_diag_gaussian_log_prob(z, y, sd, p):
    """distributions/base.py:327-344 with integer class labels y[B]."""
    loc = np.moveaxis(sd[p + "loc"].astype(z.dtype)[..., y], -1, 0)
    ls = np.moveaxis(sd[p + "log_scale"].astype(z.dtype)[..., y], -1, 0)
    d = int(np.prod(loc.shape[1:]))
    red = tuple(range(1, z.ndim))
    return (-0.5 * d * np.log(2 * np.pi)
            - np.sum(ls + 0.5 * ((z - loc) / np.exp(ls)) ** 2, axis=red)).astype(z.dtype)


# --------------------------------------------------------------------------
# drivers (core.py)
# --------------------------------------------------------------------------
def glow_base_log_prob(z, sd, p, y=None, logscale_factor=3.0, temperature=None):
    """distributions/base.py:436-471 GlowBase.log_prob: per-channel mean / log-scale (times exp(*_logs * factor)), plus
    the class rows of loc_cc / log_scale_cc, plus log(temperature); z: [B, C, ...]."""
    dt = z.dtype
    loc = sd[p + "loc"].astype(dt) * np.exp(sd[p + "loc_logs"].astype(dt) * logscale_factor)
    ls = sd[p + "log_scale"].astype(dt) * np.exp(sd[p + "log_scale_logs"].astype(dt) * logscale_factor)
    c = z.shape[1]
    tail = (1,) * (z.ndim - 2)
    if p + "loc_cc" in sd:
        loc = loc + sd[p + "loc_cc"].astype(dt)[y].reshape((len(y), c) + tail)
        ls = ls + sd[p + "log_scale_cc"].astype(dt)[y].reshape((len(y), c) + tail)
    if temperature is not None:
        ls = ls + np.log(temperature)
    num_pix = int(np.prod(z.shape[2:]))
    d = int(np.prod(z.shape[1:]))
    axes = tuple(range(1, z.ndim))
    ls_b = np.broadcast_to(ls, (z.shape[0],) + ls.shape[1:])
    return (-0.5 * d * np.log(2 * np.pi) - num_pix * ls_b.sum(axis=axes)
            - 0.5 * (((z - loc) / np.exp(ls)) ** 2).sum(axis=axes))


def _cast(sd, dt):
    return {k: (v.astype(dt) if v.dtype.kind == "f" else v) for k, v in sd.items()}


def inverse_and_log_det(spec, sd, x, per_layer=False):
    """core.py:70-85: reverse loop, log_det accumulated in float32 zeros (:81) --
    here in x.dtype; the fp32/fp64 distinction is applied by the callers below."""
    sd = _cast(sd, x.dtype)
    z = x
    tot = np.zeros(x.shape[0], dtype=x.dtype)
    trace = []
    for i in range(len(spec["flows"]) - 1, -1, -1):
        L = spec["flows"][i]
        z, ld = LAYERS[L["type"]](z, sd, f"flows.{i}.", L, "inverse")
        tot = tot + ld
        if per_layer:
            trace.append((i, z.copy(), ld.copy()))
    return (z, tot, trace) if per_layer else (z, tot)


def forward_and_log_det(spec, sd, z):
    """core.py:40-55."""
    sd = _cast(sd, z.dtype)
    tot = np.zeros(z.shape[0], dtype=z.dtype)
    for i, L in enumerate(spec["flows"]):
        z, ld = LAYERS[L["type"]](z, sd, f"flows.{i}.", L, "forward")
        tot = tot + ld
    return z, tot


def log_prob(spec, sd, x, y=None):
    """core.py:182-197 (NormalizingFlow) / :588-616 (MultiscaleFlow)."""
    if spec["kind"] == "MultiscaleFlow":
        return multiscale_log_prob(spec, sd, x, y)
    z, ld = inverse_and_log_det(spec, sd, x)
    sdc = _cast(sd, x.dtype)
    return ld + diag_gaussian_log_prob(z, sdc, "q0.")


def forward_kld(spec, sd, x, y=None):
    """core.py:87-102: -mean(log_q); the reference accumulates in float32 (:96)."""
    lp = log_prob(spec, sd, x, y)
    return -np.mean(lp)


def multiscale_log_prob(spec, sd, x, y=None):
    """core.py:588-616.  spec["levels"][i] = list of layer specs; merges are channel Merge
    (flows/reshape.py:88-100), whose inverse chunks channels into (z, z_)."""
    sd = _cast(sd, x.dtype)
    z = x
    lq = np.zeros(x.shape[0], dtype=x.dtype)
    n = len(spec["levels"])
    for i in range(n - 1, -1, -1):
        fl = spec["levels"][i]
        for j in range(len(fl) - 1, -1, -1):
            z, ld = LAYERS[fl[j]["type"]](z, sd, f"flows.{i}.{j}.", fl[j], "inverse")
            lq = lq + ld
        if i > 0:
            z, z_ = _chunk2(z)
        else:
            z_ = z
        if spec.get("class_cond", True):
            lq = lq + class_cond_diag_gaussian_log_prob(z_, y, sd, f"q0.{i}.")
        else:
            lq = lq + diag_gaussian_log_prob(z_, sd, f"q0.{i}.")
    return lq


def multiscale_inverse_and_log_det(spec, sd, x):
    """core.py:527-551: x -> (list of per-level latents, log_det)."""
    sd = _cast(sd, x.dtype)
    n = len(spec["levels"])
    tot = np.zeros(x.shape[0], dtype=x.dtype)
    zs = [None] * n
    for i in range(n - 1, -1, -1):
        fl = spec["levels"][i]
        for j in range(len(fl) - 1, -1, -1):
            x, ld = LAYERS[fl[j]["type"]](x, sd, f"flows.{i}.{j}.", fl[j], "inverse")
            tot = tot + ld
        if i == 0:
            zs[i] = x
        else:
            x, zs[i] = _chunk2(x)
    return zs, tot


def multiscale_forward_and_log_det(spec, sd, zs):
    """core.py:504-525: per-level latents -> x; Merge.forward concatenates channels (flows/reshape.py:68-74)."""
    sd = _cast(sd, zs[0].dtype)
    tot = np.zeros(zs[0].shape[0], dtype=zs[0].dtype)
    z = None
    for i, fl in enumerate(spec["levels"]):
        z = zs[0] if i == 0 else np.concatenate([z, zs[i]], axis=1)
        for j in range(len(fl)):
            z, ld = LAYERS[fl[j]["type"]](z, sd, f"flows.{i}.{j}.", fl[j], "forward")
            tot = tot + ld
    return z, tot
