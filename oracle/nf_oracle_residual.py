"""numpy fp64 restatement of the residual flow's training pass (reference: normflows/flows/residual.py:144-379,
nets/lipschitz.py:14-67,221-274,642-648; distributions/base.py DiagGaussian; flows/normalization.py ActNorm).

Values and gradients of `NormalizingFlow.log_prob` for stacks of Residual(LipschitzMLP) and ActNorm layers with a
DiagGaussian base, with the random truncation n and the Hutchinson probe eps of every block call given explicitly.
The gradient of a block is the reverse mode over g pushed forward with its tangents (the algorithm of
nfb_lipschitz_mlp_dual_backward, include/nfb200.h), seeded per estimator mode exactly as the reference's autograd:
  exact   (2-D, eval or brute_force): tangents e_0, e_1, seeds g_ld[r] (I + J_r)^-T, per row;
  neumann (training, reduce_memory=True): tangent eps, seed g_ld[0] * w (w = the Neumann vector, held constant; row 0's
          cotangent scales every row, MemoryEfficientLogDetEstimator.backward :335);
  g_only  (eval, D > 2): no tangents, the estimator's value is not differentiated.
Parameter gradients are keyed like the state_dict."""
import math

import numpy as np


def _sigmoid(v):
    return 1.0 / (1.0 + np.exp(-v))


def softplus(v):
    return np.log1p(np.exp(-np.abs(v))) + np.maximum(v, 0.0)


def swish_terms(h, b):
    """sigma, sigma', sigma'', d sigma / d b, d sigma' / d b of sigma(h) = h sigmoid(b h) / 1.1"""
    s = _sigmoid(b * h)
    s1 = s * (1 - s)
    u = b * h
    q = s1 * (2 + u * (1 - 2 * s)) / 1.1
    return h * s / 1.1, (s + u * s1) / 1.1, b * q, h * h * s1 / 1.1, h * q


def mlp_params(sd, prefix, coeff, n_layers):
    """[(W~, bias, b, W, u, v, sigma, beta, factor)] per layer: W~ = W / factor, factor = max(1, u^T W v / coeff)
    (compute_weight(update=False)).  The reference forms the factor as torch.max(torch.ones(1), sigma / coeff): the
    0-dim fp64 quotient does not promote the float32 [1] tensor, so the factor (and its gradient) is float32-rounded
    even in an fp64 model; so it is here."""
    out = []
    for l in range(n_layers):
        beta = np.asarray(sd[f"{prefix}net.{2 * l}.beta"], np.float64)
        W = np.asarray(sd[f"{prefix}net.{2 * l + 1}.weight"], np.float64)
        u = np.asarray(sd[f"{prefix}net.{2 * l + 1}.u"], np.float64)
        v = np.asarray(sd[f"{prefix}net.{2 * l + 1}.v"], np.float64)
        bias = np.asarray(sd[f"{prefix}net.{2 * l + 1}.bias"], np.float64)
        sigma = float(u @ W @ v)
        factor = float(np.float32(max(1.0, sigma / coeff)))
        out.append((W / factor, bias, float(softplus(beta)[0]), W, u, v, sigma, beta, factor))
    return out


def dual_forward(layers, x, tangents):
    """g(x) and J(x) t for tangents [nt, B, D]; also the per-layer stacked inputs H (pre-activations with bias)."""
    h, t, tape = x, tangents, []
    for Wt, bias, b, *_ in layers:
        a, d1, *_ = swish_terms(h, b)
        tape.append((h, t))
        t = (d1[None] * t) @ Wt.T
        h = a @ Wt.T + bias
    return h, t, tape


def vjp(layers, x, v):
    """v^T J(x) per row (the power-series terms of the estimators)."""
    _, _, tape = dual_forward(layers, x, np.zeros((0,) + x.shape))
    for (Wt, bias, b, *_), (h, _) in zip(reversed(layers), reversed(tape)):
        v = (v @ Wt) * swish_terms(h, b)[1]
    return v


def dual_backward(layers, x, tangents, g_seed, t_seeds):
    """Reverse mode over the dual network: returns gx and per layer (gW~, gbias, gb)."""
    _, _, tape = dual_forward(layers, x, tangents)
    hbar, tbar = g_seed, t_seeds
    grads = [None] * len(layers)
    for l in range(len(layers) - 1, -1, -1):
        Wt, bias, b = layers[l][:3]
        h, t = tape[l]
        a, d1, d2, db0, db1 = swish_terms(h, b)
        ta = d1[None] * t
        gW = hbar.T @ a + sum(tbar[k].T @ ta[k] for k in range(t.shape[0]))
        gbias = hbar.sum(0)
        abar, tabar = hbar @ Wt, tbar @ Wt
        mix = (t * tabar).sum(0)
        gb = float((abar * db0).sum() + (mix * db1).sum())
        hbar, tbar = d1 * abar + d2 * mix, d1[None] * tabar
        grads[l] = (gW, gbias, gb)
    return hbar, grads


def geometric_1mcdf(p, k, offset):
    if k <= offset:
        return 1.0
    return (1 - p) ** max(k - offset - 1, 0)


def poisson_1mcdf(lamb, k, offset):
    if k <= offset:
        return 1.0
    k = k - offset
    return 1 - math.exp(-lamb) * sum(lamb ** i / math.factorial(i) for i in range(k))


def coefficients(blk, sd, prefix, n, training):
    """(n_power_series, coeff_fn) of residual.py:163-198 for the truncation draw n (array)."""
    if blk["n_dist"] == "geometric":
        p = float(_sigmoid(np.asarray(sd[prefix + "geom_p"], np.float64)))
        rcdf = lambda k, off: geometric_1mcdf(p, k, off)
    else:
        lamb = float(sd[prefix + "lamb"])
        rcdf = lambda k, off: poisson_1mcdf(lamb, k, off)
    if training and blk.get("n_power_series") is not None:
        return blk["n_power_series"], lambda k: 1.0
    off = blk.get("n_exact_terms", 2) if training else 20
    n = np.asarray(n)
    return int(n.max()) + off, lambda k: 1 / rcdf(k, off) * np.sum(n >= k - off) / len(n)


def block_mode(blk, training, d):
    if (blk.get("brute_force") or not training) and d == 2:
        return "exact"
    return "neumann" if training else "g_only"


def residual_block(blk, sd, prefix, x, training, n=None, eps=None):
    """(y = x + g, log-det [B], what the backward needs) of iResBlock.forward(x, 0) (Residual.inverse)."""
    layers = mlp_params(sd, prefix + "nnet.", blk["coeff"], blk["n_layers"])
    mode = block_mode(blk, training, x.shape[1])
    if mode == "exact":
        eye = np.zeros((2,) + x.shape)
        eye[0, :, 0] = eye[1, :, 1] = 1.0
        g, jt, _ = dual_forward(layers, x, eye)
        m00, m10, m01, m11 = jt[0, :, 0] + 1, jt[0, :, 1], jt[1, :, 0], jt[1, :, 1] + 1
        det = m00 * m11 - m01 * m10
        ld = np.log(np.abs(det))
        return x + g, ld, (mode, layers, eye, (m00, m10, m01, m11, det))
    g = dual_forward(layers, x, np.zeros((0,) + x.shape))[0]
    N, coeff = coefficients(blk, sd, prefix, n, training)
    if mode == "neumann":
        v, w = eps, eps.copy()
        for k in range(1, N + 1):
            v = vjp(layers, x, v)
            w = w + (-1) ** k * coeff(k) * v
        return x + g, (vjp(layers, x, w) * eps).sum(1), (mode, layers, eps[None], w)
    v, ld = eps, np.zeros(x.shape[0])
    for k in range(1, N + 1):
        v = vjp(layers, x, v)
        ld = ld + (-1) ** (k + 1) / k * coeff(k) * (v * eps).sum(1)
    return x + g, ld, (mode, layers, None, None)


def residual_block_backward(x, saved, gy, g_ld):
    mode, layers, tangents, extra = saved
    if mode == "exact":
        m00, m10, m01, m11, det = extra
        c = g_ld / det
        seeds = np.stack([np.stack([c * m11, -c * m01], 1), np.stack([-c * m10, c * m00], 1)])
    elif mode == "neumann":
        # MemoryEfficientLogDetEstimator: the log-det gradient is formed with unit cotangents in the forward and scaled
        # by dL = g_ld[0] in the backward; the gradient of g is a separate autograd pass (:304-352)
        gx_ld, grads_ld = dual_backward(layers, x, tangents, np.zeros_like(gy), extra[None])
        gx_g, grads_g = dual_backward(layers, x, tangents[:0], gy, tangents[:0])
        return gy + g_ld[0] * gx_ld + gx_g, layers, [(g_ld[0], grads_ld), (1.0, grads_g)]
    else:
        tangents = np.zeros((0,) + x.shape)
        seeds = np.zeros((0,) + x.shape)
    gx, grads = dual_backward(layers, x, tangents, gy, seeds)
    return gy + gx, layers, [(1.0, grads)]


def chain_params(blk, prefix, layers, parts):
    """gW~ -> weight (through W~ = W / factor, factor = sigma / c when sigma > c), gb -> beta (softplus'); bias as is.
    parts: [(scale, per-layer (gW~, gbias, gb))], one per autograd pass of the reference; each pass rounds its own
    cotangent of the factor to float32 (see mlp_params) before it is scaled."""
    out = {}
    c = blk["coeff"]
    for l, (Wt, bias, b, W, u, v, sigma, beta, f) in enumerate(layers):
        gWraw, gbias, gb = 0.0, 0.0, 0.0
        for scale, grads in parts:
            gW, gbl, gbb = grads[l]
            gw = gW / f
            if sigma / c > 1.0:
                g_factor = float(np.float32(-float((gW * W).sum()) / f ** 2))
                gw = gw + (g_factor / c) * np.outer(u, v)
            gWraw, gbias, gb = gWraw + scale * gw, gbias + scale * gbl, gb + scale * gbb
        out[f"{prefix}nnet.net.{2 * l + 1}.weight"] = gWraw
        out[f"{prefix}nnet.net.{2 * l + 1}.bias"] = gbias
        out[f"{prefix}nnet.net.{2 * l}.beta"] = np.array([gb * float(_sigmoid(beta[0]))])
    return out


def log_prob_and_grads(spec, sd, x, cot, training, draws):
    """log_prob(x) [B] of the stack and the gradients of sum_r cot[r] log_prob(x_r) w.r.t. x and every parameter.
    spec: {"flows": [{"type": "residual", "coeff", "n_layers", "n_dist", "brute_force", ...} | {"type": "actnorm"}],
    "base_trainable": bool}; draws: [(n, eps)] per estimator call, in call order (flows last to first)."""
    sd = {k: np.asarray(v, np.float64) for k, v in sd.items()}
    z, lq, saved, di = x, np.zeros(x.shape[0]), [], 0
    for i in range(len(spec["flows"]) - 1, -1, -1):
        blk, pre = spec["flows"][i], f"flows.{i}."
        if blk["type"] == "actnorm":
            s, t = sd[pre + "s"].reshape(1, -1), sd[pre + "t"].reshape(1, -1)
            saved.append((i, z))
            z, ld = (z - t) * np.exp(-s), -s.sum() * np.ones(z.shape[0])
        else:
            n, eps = (None, None)
            if block_mode(blk, training, z.shape[1]) != "exact":
                n, eps = draws[di]
                di += 1
            zin = z
            z, ld, sv = residual_block(blk, sd, pre + "iresblock.", z, training, n, eps)
            saved.append((i, (zin, sv)))
        lq = lq + ld
    loc, ls = sd["q0.loc"].reshape(1, -1), sd["q0.log_scale"].reshape(1, -1)
    r = (z - loc) * np.exp(-ls)
    lq = lq - 0.5 * x.shape[1] * np.log(2 * np.pi) - (ls + 0.5 * r ** 2).sum(1)
    grads = {}
    if spec.get("base_trainable", True):
        grads["q0.loc"] = (cot[:, None] * r * np.exp(-ls)).sum(0, keepdims=True)
        grads["q0.log_scale"] = (cot[:, None] * (r ** 2 - 1)).sum(0, keepdims=True)
    gz = -cot[:, None] * r * np.exp(-ls)
    for i, item in reversed(saved):
        blk, pre = spec["flows"][i], f"flows.{i}."
        if blk["type"] == "actnorm":
            s, t = sd[pre + "s"].reshape(1, -1), sd[pre + "t"].reshape(1, -1)
            zin = item
            grads[pre + "t"] = -(gz * np.exp(-s)).sum(0, keepdims=True)
            grads[pre + "s"] = (-(gz * (zin - t) * np.exp(-s))).sum(0, keepdims=True) - cot.sum()
            gz = gz * np.exp(-s)
        else:
            zin, sv = item
            gz, layers, g = residual_block_backward(zin, sv, gz, cot)
            grads.update(chain_params(blk, pre + "iresblock.", layers, g))
    grads["x"] = gz
    return lq, grads
