"""Gradient oracle: hand-written reverse mode of `NormalizingFlow.log_prob` (any per-row weighting; `forward_kld`,
core.py:87-102, is the uniform one) for neural-spline stacks, in numpy.  TEST INFRASTRUCTURE ONLY (same rules as nf_oracle.py): it is the checker the
native backward kernels (SURVEY 8f-1) will be compared with at shapes for which no golden fixture exists.

Pinned: tests/test_oracle_golden.py checks every parameter gradient and the input gradient against
`tests/golden/grads_nsf_{ar,coupled}_d5_h128_l3.npz`, which were minted from the reference's own autograd in
fp64 (tests/golden/make_golden.py grads).

Covers the density pass of: AutoregressiveRationalQuadraticSpline (MADE, nets/made.py),
CoupledRationalQuadraticSpline (ResidualNet, nets/resnet.py, + unconditional CDF), LULinearPermute
(flows/mixing.py:368-563), Permute and a DiagGaussian base (trainable or not).  Each `*_bwd` takes the upstream gradients
(g_out w.r.t. the layer output, g_ld w.r.t. its per-sample log-det) and returns the gradient w.r.t. the layer
input, adding parameter gradients into `grads` under their state_dict names.

`sampling_grads` covers the sampling direction (forward_and_log_det) of CoupledRationalQuadraticSpline /
LULinearPermute stacks, with the reparameterised DiagGaussian draw; its inverse-spline adjoint is built on rqs_bwd."""
import numpy as np

from . import nf_oracle as O


# --------------------------------------------------------------------------
# spline element: forward intermediates + adjoint (utils/splines.py:100-219, forward branch)
# --------------------------------------------------------------------------
def _softmax_knots_bwd(un, g_cum_inner, min_size, scale):
    """cum_j (j = 1..K-1) = lo + scale * sum_{t<j} (min + (1 - K min) softmax(un)_t).  g_cum_inner: [..., K-1]
    gradient w.r.t. the interior knots.  Returns the gradient w.r.t. `un`."""
    k = un.shape[-1]
    s = O.softmax(un, axis=-1)
    # g wrt widths s'_t = min + c s_t :  knot j depends on s'_0..s'_{j-1}
    g_sp = np.zeros_like(un)
    rev = np.cumsum(g_cum_inner[..., ::-1], axis=-1)[..., ::-1]  # rev[..., t] = sum_{j >= t+1} g_cum_j
    g_sp[..., :k - 1] = rev * scale
    g_s = g_sp * (1 - min_size * k)
    return s * (g_s - np.sum(g_s * s, axis=-1, keepdims=True))  # softmax Jacobian


def rqs_bwd(x, uw, uh, ud, gy, glad, tail_bound):
    """Adjoint of nf_oracle.unconstrained_rqs(inverse=False).  ud: [..., K-1].  Returns (gx, guw, guh, gud)."""
    dt = x.dtype
    k = uw.shape[-1]
    B = tail_bound
    inside = (x >= -B) & (x <= B)
    const = np.asarray(np.log(np.exp(1 - O.MIN_DERIVATIVE) - 1), dtype=dt)
    pad = np.full(ud.shape[:-1] + (1,), const, dtype=dt)
    udf = np.concatenate([pad, ud, pad], axis=-1)
    xs = np.where(inside, x, 0.0)
    cumw, w = O._knots(uw, -B, B, O.MIN_BIN_WIDTH)
    cumh, h = O._knots(uh, -B, B, O.MIN_BIN_HEIGHT)
    d = O.MIN_DERIVATIVE + O.softplus(udf)
    loc = cumw.copy()
    loc[..., -1] += 1e-6
    idx = np.clip(np.sum(xs[..., None] >= loc, axis=-1) - 1, 0, k - 1)
    g = lambda a, i: np.take_along_axis(a, i[..., None], axis=-1)[..., 0]
    l_w, r_w = g(cumw, idx), g(cumw, idx + 1)
    l_h, r_h = g(cumh, idx), g(cumh, idx + 1)
    d0, d1 = g(d, idx), g(d, idx + 1)
    ww, hh = r_w - l_w, r_h - l_h
    delta = hh / ww
    th = (xs - l_w) / ww
    omt = 1 - th
    A, Bq, C = th * th, th * omt, omt * omt
    s = d0 + d1 - 2 * delta
    den = delta + s * Bq
    P = delta * A + d0 * Bq
    num = hh * P
    Q = d1 * A + 2 * delta * Bq + d0 * C
    dnum = delta * delta * Q
    # adjoint (same derivation as csrc/nfb_spline_bwd.cuh, here in the reference's [-B,B] coordinates)
    g_out = np.where(inside, gy, 0.0)
    g_l = np.where(inside, glad, 0.0)
    g_num = g_out / den
    g_den = -g_out * num / den ** 2 - 2 * g_l / den
    g_dnum = g_l / dnum
    g_delta = g_dnum * (2 * delta * Q + delta * delta * 2 * Bq)
    g_Q = g_dnum * delta * delta
    g_d1, g_d0 = g_Q * A, g_Q * C
    g_A, g_B, g_C = g_Q * d1, g_Q * 2 * delta, g_Q * d0
    g_h = g_num * P
    g_P = g_num * hh
    g_delta = g_delta + g_P * A + g_den
    g_A = g_A + g_P * delta
    g_d0 = g_d0 + g_P * Bq
    g_B = g_B + g_P * d0 + g_den * s
    g_s = g_den * Bq
    g_d0, g_d1, g_delta = g_d0 + g_s, g_d1 + g_s, g_delta - 2 * g_s
    g_th = 2 * th * g_A + (1 - 2 * th) * g_B - 2 * omt * g_C
    g_x_in = g_th / ww
    g_lw = -g_th / ww
    g_w = -g_th * th / ww - (g_delta / ww) * delta
    g_h = g_h + g_delta / ww
    g_rw, g_lw = g_w, g_lw - g_w
    g_rh, g_lh = g_h, g_out - g_h
    gx = np.where(inside, g_x_in, gy)

    def scatter_knots(g_left, g_right):  # -> gradient w.r.t. the K-1 interior knots
        out = np.zeros(x.shape + (k + 1,), dtype=dt)
        np.put_along_axis(out, idx[..., None], g_left[..., None], axis=-1)
        tmp = np.zeros_like(out)
        np.put_along_axis(tmp, (idx + 1)[..., None], g_right[..., None], axis=-1)
        return (out + tmp)[..., 1:k]
    guw = _softmax_knots_bwd(uw, scatter_knots(g_lw, g_rw), O.MIN_BIN_WIDTH, 2 * B)
    guh = _softmax_knots_bwd(uh, scatter_knots(g_lh, g_rh), O.MIN_BIN_HEIGHT, 2 * B)
    g_df = np.zeros(x.shape + (k + 1,), dtype=dt)
    np.put_along_axis(g_df, idx[..., None], g_d0[..., None], axis=-1)
    tmp = np.zeros_like(g_df)
    np.put_along_axis(tmp, (idx + 1)[..., None], g_d1[..., None], axis=-1)
    g_df = (g_df + tmp) * O.sigmoid(udf)  # softplus' = sigmoid
    return gx, guw, guh, g_df[..., 1:k]


# --------------------------------------------------------------------------
# conditioner nets (pre-activation residual blocks; masks for MADE)
# --------------------------------------------------------------------------
def _net_fwd(x, sd, p, masked):
    W = lambda q: sd[q + "weight"] * (sd[q + "mask"].astype(x.dtype) if masked else 1.0)
    acts = {"x": x}
    h = x @ W(p + "initial_layer.").T + sd[p + "initial_layer.bias"]
    n = O._num_blocks(sd, p)
    for i in range(n):
        q = f"{p}blocks.{i}.linear_layers."
        a0 = np.maximum(h, 0)
        t = a0 @ W(q + "0.").T + sd[q + "0.bias"]
        a1 = np.maximum(t, 0)
        acts[i] = (h, a0, t, a1)
        h = h + a1 @ W(q + "1.").T + sd[q + "1.bias"]
    acts["h"] = h
    return h @ W(p + "final_layer.").T + sd[p + "final_layer.bias"], acts, n, W


def _net_bwd(g_out, acts, n, W, sd, p, masked, grads):
    def lin(q, a, g):  # y = a W^T + b
        m = sd[q + "mask"].astype(g.dtype) if masked else 1.0
        grads[q + "weight"] = grads.get(q + "weight", 0) + (g.T @ a) * m
        grads[q + "bias"] = grads.get(q + "bias", 0) + g.sum(0)
        return g @ W(q)
    g_h = lin(p + "final_layer.", acts["h"], g_out)
    for i in range(n - 1, -1, -1):
        q = f"{p}blocks.{i}.linear_layers."
        h, a0, t, a1 = acts[i]
        g_a1 = lin(q + "1.", a1, g_h)
        g_t = g_a1 * (t > 0)
        g_a0 = lin(q + "0.", a0, g_t)
        g_h = g_h + g_a0 * (h > 0)
    return lin(p + "initial_layer.", acts["x"], g_h)


# --------------------------------------------------------------------------
# layers (density direction)
# --------------------------------------------------------------------------
def ar_rqs_bwd(z, sd, p, L, g_out, g_ld, grads):
    k, tb = L.get("num_bins", 8), float(L.get("tail_bound", 3.0))
    net = p + "mprqat.autoregressive_net."
    bsz, d = z.shape
    params, acts, n, W = _net_fwd(z, sd, net, masked=True)
    pr = params.reshape(bsz, d, 3 * k - 1)
    uw, uh, ud = pr[..., :k], pr[..., k:2 * k], pr[..., 2 * k:]  # no 1/sqrt(H) in the AR layer
    gx, guw, guh, gud = rqs_bwd(z, uw, uh, ud, g_out, np.broadcast_to(g_ld[:, None], z.shape), tb)
    g_params = np.concatenate([guw, guh, gud], axis=-1).reshape(bsz, -1)
    return gx + _net_bwd(g_params, acts, n, W, sd, net, True, grads)


def coupled_rqs_bwd(z, sd, p, L, g_out, g_ld, grads):
    k, tb = L.get("num_bins", 8), float(L.get("tail_bound", 3.0))
    q = p + "prqct."
    idf = sd[q + "identity_features"].astype(np.int64)
    trf = sd[q + "transform_features"].astype(np.int64)
    hidden = sd[q + "transform_net.initial_layer.weight"].shape[0]
    sc = np.sqrt(hidden)
    bsz = z.shape[0]
    ident, trans = z[:, idf], z[:, trf]
    params, acts, n, W = _net_fwd(ident, sd, q + "transform_net.", masked=False)
    pr = params.reshape(bsz, len(trf), 3 * k - 1)
    uw, uh, ud = pr[..., :k] / sc, pr[..., k:2 * k] / sc, pr[..., 2 * k:]
    gl_t = np.broadcast_to(g_ld[:, None], trans.shape)
    gxt, guw, guh, gud = rqs_bwd(trans, uw, uh, ud, g_out[:, trf], gl_t, tb)
    g_params = np.concatenate([guw / sc, guh / sc, gud], axis=-1).reshape(bsz, -1)
    g_ident = _net_bwd(g_params, acts, n, W, sd, q + "transform_net.", False, grads)
    u = q + "unconditional_transform."
    bc = lambda a: np.broadcast_to(a[None], (bsz,) + a.shape)
    gl_i = np.broadcast_to(g_ld[:, None], ident.shape)
    gxi, g1, g2, g3 = rqs_bwd(ident, bc(sd[u + "unnormalized_widths"]), bc(sd[u + "unnormalized_heights"]),
                              bc(sd[u + "unnormalized_derivatives"]), g_out[:, idf], gl_i, tb)
    for name, gg in (("unnormalized_widths", g1), ("unnormalized_heights", g2), ("unnormalized_derivatives", g3)):
        grads[u + name] = grads.get(u + name, 0) + gg.sum(0)
    gz = np.zeros_like(z)
    gz[:, idf] = gxi + g_ident
    gz[:, trf] = gxt
    return gz


def lu_bwd(z, sd, p, L, g_out, g_ld, grads):
    """x = z[:, perm]; y = (x U^T) L^T + b; log_det = sum log(softplus(u_diag) + 1e-3) for every sample."""
    dt = z.dtype
    perm = sd[p + "permutation._permutation"].astype(np.int64)
    lower, upper, diag = O.lu_matrices(sd, p, dt)
    n = len(perm)
    x = z[:, perm]
    t = x @ upper.T
    grads[p + "linear.bias"] = grads.get(p + "linear.bias", 0) + g_out.sum(0)
    g_lower = g_out.T @ t  # y = t L^T  ->  dL = g^T t
    g_t = g_out @ lower
    g_upper = g_t.T @ x
    g_x = g_t @ upper
    grads[p + "linear.lower_entries"] = grads.get(p + "linear.lower_entries", 0) + g_lower[np.tril_indices(n, -1)]
    grads[p + "linear.upper_entries"] = grads.get(p + "linear.upper_entries", 0) + g_upper[np.triu_indices(n, 1)]
    ud = sd[p + "linear.unconstrained_upper_diag"].astype(dt)
    g_diag = np.diag(g_upper) + g_ld.sum() / diag
    grads[p + "linear.unconstrained_upper_diag"] = grads.get(p + "linear.unconstrained_upper_diag", 0) + \
        g_diag * O.sigmoid(ud)
    gz = np.zeros_like(z)
    gz[:, perm] = g_x
    return gz


def permute_bwd(z, sd, p, L, g_out, g_ld, grads):
    """Adjoint of nf_oracle.permute (density direction): the inverse gather."""
    c = z.shape[1]
    gz = np.zeros_like(g_out)
    if L.get("mode", "shuffle") == "shuffle":
        gz[:, sd[p + "inv_perm"].astype(np.int64)] = g_out
    else:
        h = (c + 1) // 2
        gz[:, h:], gz[:, :h] = g_out[:, :c - h], g_out[:, c - h:]
    return gz


_BWD = {"AutoregressiveRationalQuadraticSpline": ar_rqs_bwd, "CoupledRationalQuadraticSpline": coupled_rqs_bwd,
        "LULinearPermute": lu_bwd, "Permute": permute_bwd}


def log_prob_grads(spec, sd, x, w, trainable_base=False):
    """Gradients of sum(w * log q(x)) for per-row weights w[B]: (log q(x), {state_dict name: gradient}, d / d x) in x's
    dtype.  trainable_base: also the DiagGaussian base's q0.loc and q0.log_scale."""
    sd = O._cast(sd, x.dtype)
    flows = spec["flows"]
    zs = [x]
    z = x
    tot = np.zeros(x.shape[0], dtype=x.dtype)
    for i in range(len(flows) - 1, -1, -1):  # density pass, keeping every layer's input
        z, ld = O.LAYERS[flows[i]["type"]](z, sd, f"flows.{i}.", flows[i], "inverse")
        tot = tot + ld
        zs.append(z)
    lp = tot + O.diag_gaussian_log_prob(z, sd, "q0.")
    g_lp = np.asarray(w, dtype=x.dtype)
    loc = sd["q0.loc"].reshape(-1)
    ls = sd["q0.log_scale"].reshape(-1)
    u = (z - loc) / np.exp(2 * ls)
    g_z = g_lp[:, None] * (-u)  # d log N / d z
    grads = {}
    if trainable_base:
        grads["q0.loc"] = (g_lp[:, None] * u).sum(0).reshape(sd["q0.loc"].shape)
        grads["q0.log_scale"] = (g_lp[:, None] * ((z - loc) * u - 1)).sum(0).reshape(sd["q0.log_scale"].shape)
    for i in range(len(flows)):  # backward: layers in list order, inputs from the cache
        z_in = zs[len(flows) - 1 - i]
        g_z = _BWD[flows[i]["type"]](z_in, sd, f"flows.{i}.", flows[i], g_z, g_lp, grads)
    return lp, grads, g_z


# --------------------------------------------------------------------------
# sampling direction (forward_and_log_det): coupled spline blocks and LU maps
# --------------------------------------------------------------------------
def rqs_inv_bwd(x, uw, uh, ud, gx, g_ld, tail_bound):
    """Adjoint of nf_oracle.unconstrained_rqs(inverse=True) at its OUTPUT x = f^-1(y) (the inverse's log-det is
    -log f'(x)), through the implicit-function relation on the forward adjoint rqs_bwd: with
    lam = gx - g_ld d/dx log f'(x), g_y = lam / f'(x) and the parameters' gradient is rqs_bwd's for
    (gy = -g_y, glad = -g_ld).  Outside the tails f is the identity: g_y = gx.  Returns (gy, guw, guh, gud)."""
    zero, one = np.zeros_like(x), np.ones_like(x)
    fp = rqs_bwd(x, uw, uh, ud, one, zero, tail_bound)[0]        # f'(x) (1 outside)
    dlog = rqs_bwd(x, uw, uh, ud, zero, one, tail_bound)[0]      # d/dx log f'(x) (0 outside)
    gy = (gx - g_ld * dlog) / fp
    _, guw, guh, gud = rqs_bwd(x, uw, uh, ud, -gy, -g_ld, tail_bound)
    return gy, guw, guh, gud


def coupled_rqs_sampling_bwd(z, x, sd, p, L, g_out, g_ld, grads):
    """Coupling.inverse: x_id = the unconditional CDF's inverse at z_id, the conditioner reads x_id, x_tr = the inverse
    spline at z_tr.  The conditioner's data gradient joins g_out[id] before the identity columns' inverse adjoint."""
    k, tb = L.get("num_bins", 8), float(L.get("tail_bound", 3.0))
    q = p + "prqct."
    idf = sd[q + "identity_features"].astype(np.int64)
    trf = sd[q + "transform_features"].astype(np.int64)
    sc = np.sqrt(sd[q + "transform_net.initial_layer.weight"].shape[0])
    bsz = z.shape[0]
    xi, xt = x[:, idf], x[:, trf]
    params, acts, n, W = _net_fwd(xi, sd, q + "transform_net.", masked=False)
    pr = params.reshape(bsz, len(trf), 3 * k - 1)
    uw, uh, ud = pr[..., :k] / sc, pr[..., k:2 * k] / sc, pr[..., 2 * k:]
    gzt, guw, guh, gud = rqs_inv_bwd(xt, uw, uh, ud, g_out[:, trf], np.broadcast_to(g_ld[:, None], xt.shape), tb)
    g_params = np.concatenate([guw / sc, guh / sc, gud], axis=-1).reshape(bsz, -1)
    g_xi = g_out[:, idf] + _net_bwd(g_params, acts, n, W, sd, q + "transform_net.", False, grads)
    u = q + "unconditional_transform."
    bc = lambda a: np.broadcast_to(a[None], (bsz,) + a.shape)
    gzi, g1, g2, g3 = rqs_inv_bwd(xi, bc(sd[u + "unnormalized_widths"]), bc(sd[u + "unnormalized_heights"]),
                                  bc(sd[u + "unnormalized_derivatives"]), g_xi,
                                  np.broadcast_to(g_ld[:, None], xi.shape), tb)
    for name, gg in (("unnormalized_widths", g1), ("unnormalized_heights", g2), ("unnormalized_derivatives", g3)):
        grads[u + name] = grads.get(u + name, 0) + gg.sum(0)
    gz = np.zeros_like(z)
    gz[:, idf] = gzi
    gz[:, trf] = gzt
    return gz


def lu_sampling_bwd(z, x, sd, p, L, g_out, g_ld, grads):
    """t = W^-1 (y - b) per row (W = L U), x = t[:, inv_perm], log_det = -sum log diag U:  g_t = g_x[:, perm],
    g_y = W^-T g_t, dW = -sum_rows g_y t^T, g_b = -colsum(g_y); -sum(g_ld) is the cotangent of log|det W|."""
    perm = sd[p + "permutation._permutation"].astype(np.int64)
    lower, upper, diag = O.lu_matrices(sd, p, z.dtype)
    n = len(perm)
    t = x[:, perm]                        # x = t[:, inv_perm]
    g_t = g_out[:, perm]
    w = lower @ upper
    g_y = np.linalg.solve(w.T, g_t.T).T   # row form of W^-T g_t
    d_w = -(g_y.T @ t)
    grads[p + "linear.bias"] = grads.get(p + "linear.bias", 0) - g_y.sum(0)
    g_lower = d_w @ upper.T
    g_upper = lower.T @ d_w
    grads[p + "linear.lower_entries"] = grads.get(p + "linear.lower_entries", 0) + g_lower[np.tril_indices(n, -1)]
    grads[p + "linear.upper_entries"] = grads.get(p + "linear.upper_entries", 0) + g_upper[np.triu_indices(n, 1)]
    ud = sd[p + "linear.unconstrained_upper_diag"].astype(z.dtype)
    g_diag = np.diag(g_upper) - g_ld.sum() / diag
    grads[p + "linear.unconstrained_upper_diag"] = grads.get(p + "linear.unconstrained_upper_diag", 0) + \
        g_diag * O.sigmoid(ud)
    return g_y


_SAMPLING_BWD = {"CoupledRationalQuadraticSpline": coupled_rqs_sampling_bwd, "LULinearPermute": lu_sampling_bwd}


def sampling_grads(spec, sd, z, g_x, g_ld, trainable_base=False, g_lq0=None):
    """Gradients of sum(g_x * x) + sum(g_ld * log_det) of (x, log_det) = nf_oracle.forward_and_log_det(spec, sd, z) for
    stacks of CoupledRationalQuadraticSpline and LULinearPermute: (x, log_det, {state_dict name: gradient}, d / d z) in
    z's dtype.  trainable_base: z is the DiagGaussian base's standardised draw eps, the stack's input is
    loc + exp(log_scale) eps (the reparameterised draw), and g_lq0 [rows] (default 0) is the cotangent of the base's
    log-density of that draw; q0.loc and q0.log_scale get their gradients and d / d eps is returned."""
    sd = O._cast(sd, z.dtype)
    flows = spec["flows"]
    g_x, g_ld = np.asarray(g_x, z.dtype), np.asarray(g_ld, z.dtype)
    eps = z
    if trainable_base:
        loc, ls = sd["q0.loc"].reshape(-1), sd["q0.log_scale"].reshape(-1)
        z = loc + np.exp(ls) * eps
    zs = [z]
    tot = np.zeros(z.shape[0], dtype=z.dtype)
    for i, L in enumerate(flows):   # sampling pass, keeping every layer's input and output
        z, ld = O.LAYERS[L["type"]](z, sd, f"flows.{i}.", L, "forward")
        tot = tot + ld
        zs.append(z)
    grads = {}
    g = g_x
    for i in range(len(flows) - 1, -1, -1):
        g = _SAMPLING_BWD[flows[i]["type"]](zs[i], zs[i + 1], sd, f"flows.{i}.", flows[i], g, g_ld, grads)
    if trainable_base:
        glq = np.zeros(eps.shape[0], z.dtype) if g_lq0 is None else np.asarray(g_lq0, z.dtype)
        grads["q0.loc"] = g.sum(0).reshape(sd["q0.loc"].shape)
        grads["q0.log_scale"] = ((g * eps * np.exp(ls)).sum(0) - glq.sum()).reshape(sd["q0.log_scale"].shape)
        g = g * np.exp(ls) - glq[:, None] * eps   # log q0 = -D/2 log 2 pi - sum(log_scale + eps^2 / 2)
    return z, tot, grads, g


def forward_kld_grads(spec, sd, x):
    """loss = -mean(log q(x)); returns (loss, {state_dict name: gradient}, d loss / d x) in x's dtype."""
    bsz = x.shape[0]
    lp, grads, g_z = log_prob_grads(spec, sd, x, np.full(bsz, -1.0 / bsz, dtype=x.dtype))
    return -np.mean(lp), grads, g_z
