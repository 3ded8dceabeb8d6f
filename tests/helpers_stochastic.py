"""fp64 numpy restatement of the stochastic kernels (csrc/nfb_stochastic.cu): the HMC transition, its parameter
gradients in closed form, Metropolis-Hastings with a diagonal Gaussian proposal, and the HAIS chain; plus the models of
tests/golden/make_stochastic_grads.py.

A density is a list of terms (coef, loc [K, D], log_scale [K, D], weight_scores [K]) with log p = sum coef log p_i; a
DiagGaussian is the one-mode term with weight score 0.

HMC with grad log p held constant (the reference detaches it) has, for L leapfrog steps, eps = exp(log_step_size),
m = exp(log_mass) and momentum noise n:
    z_L - z = L eps n m^-1/2 + eps^2 m^-1 S,   S = L/2 g_0 + sum_{i=1}^{L-1} (L - i) g_i   (g_i = grad log p at z_i)
so with A = L eps n m^-1/2 and B = eps^2 m^-1 S, dz_L/dlog_step_size = A + 2 B and dz_L/dlog_mass = -A/2 - B."""
import numpy as np

import helpers_mixture as M


def lp_grad(z, terms):
    """log p [N] and grad log p [N, D] of the density at rows z."""
    lp = np.zeros(len(z))
    g = np.zeros_like(z)
    for c, loc, ls, ws in terms:
        lp = lp + c * M.log_prob(z, loc, ls, ws)
        g = g + c * M.log_prob_grads(z, loc, ls, ws, np.ones(len(z)))[0]
    return lp, g


def _clamp(g, mag):
    return np.clip(g, -mag, mag) if mag else g


def hmc(z, terms, steps, log_step, log_mass, mag, noise, unif):
    """One transition -> (z_out, log_det, accept, probability)."""
    eps, m = np.exp(log_step), np.exp(log_mass)
    p = noise * np.exp(0.5 * log_mass)
    lp0, g = lp_grad(z, terms)
    g = _clamp(g, mag)
    zn, pn, lp1 = z.copy(), p.copy(), lp0
    for _ in range(steps):
        pn = pn + eps / 2 * g
        zn = zn + eps * pn / m
        lp1, g = lp_grad(zn, terms)
        g = _clamp(g, mag)
        pn = pn + eps / 2 * g
    with np.errstate(over="ignore", invalid="ignore"):
        prob = np.exp(lp1 - lp0 - 0.5 * (pn ** 2 / m).sum(1) + 0.5 * (p ** 2 / m).sum(1))
    acc = unif < prob
    z_out = np.where(acc[:, None], zn, z)
    return z_out, lp0 - np.where(acc, lp1, lp0), acc, prob


def hmc_step_grads(z, terms, steps, log_step, log_mass, mag, noise, accept, G):
    """Gradients of sum <G, z_out> with respect to log_step_size and log_mass [D] (closed form above)."""
    eps, m = np.exp(log_step), np.exp(log_mass)
    zn, pn = z.copy(), noise * np.exp(0.5 * log_mass)
    S = np.zeros_like(z)
    for j in range(steps):
        g = _clamp(lp_grad(zn, terms)[1], mag)
        S += (0.5 * steps if j == 0 else steps - j) * g
        pn = pn + eps / 2 * g if j == 0 else pn + eps * g
        zn = zn + eps * pn / m
    A = steps * eps * noise / np.sqrt(m)
    B = eps ** 2 / m * S
    Ga = G * accept[:, None]
    return (Ga * (A + 2 * B)).sum(0), (Ga * (-0.5 * A - B)).sum(0)


def log_det_grads(z, z_out, moved, terms, g_ld):
    """Gradients of sum_r g_ld[r] moved[r] (log p(z_r) - log p(z_out_r)): (g_z, g_z_out, [(g_loc, g_ls, g_ws)] per
    term)."""
    g = g_ld * moved
    gz, gzo, gp = np.zeros_like(z), np.zeros_like(z), []
    for c, loc, ls, ws in terms:
        a = M.log_prob_grads(z, loc, ls, ws, c * g)
        b = M.log_prob_grads(z_out, loc, ls, ws, -c * g)
        gz += a[0]
        gzo += b[0]
        gp.append(tuple(x + y for x, y in zip(a[1:], b[1:])))
    return gz, gzo, gp


def hmc_grads(z, terms, steps, log_step, log_mass, mag, noise, unif, w_z, w_ld):
    """Every gradient of sum <w_z, z_out> + <w_ld, log_det> for one transition: (g_z, g_log_step, g_log_mass,
    [(g_loc, g_ls, g_ws)] per term)."""
    z_out, _, acc, _ = hmc(z, terms, steps, log_step, log_mass, mag, noise, unif)
    gz, gzo, gp = log_det_grads(z, z_out, acc.astype(float), terms, w_ld)
    G = w_z + gzo
    g_ls, g_lm = hmc_step_grads(z, terms, steps, log_step, log_mass, mag, noise, acc, G)
    return G + gz, g_ls, g_lm, gp


def mh(z, terms, steps, scale, noise, unif):
    """-> (z_out, log_det, moved)."""
    lp0 = lp_grad(z, terms)[0]
    ld, moved = np.zeros(len(z)), np.zeros(len(z), bool)
    for s in range(steps):
        zn = noise[s] * scale + z
        lp1 = lp_grad(zn, terms)[0]
        with np.errstate(over="ignore", invalid="ignore"):
            acc = unif[s] <= np.minimum(np.exp(lp1 - lp0), 1.0)
        z = np.where(acc[:, None], zn, z)
        ld = np.where(acc, ld + lp0 - lp1, ld)
        lp0 = np.where(acc, lp1, lp0)
        moved |= acc
    return z, ld, moved


def mh_margin(z, terms, steps, scale, noise, unif):
    """Per row, the smallest |u - min(exp(delta), 1)| / max(u, 1e-30) over the steps."""
    lp0 = lp_grad(z, terms)[0]
    out = np.full(len(z), np.inf)
    for s in range(steps):
        zn = noise[s] * scale + z
        lp1 = lp_grad(zn, terms)[0]
        P = np.minimum(np.exp(lp1 - lp0), 1.0)
        out = np.minimum(out, np.abs(unif[s] - P) / np.maximum(unif[s], 1e-30))
        acc = unif[s] <= P
        z = np.where(acc[:, None], zn, z)
        lp0 = np.where(acc, lp1, lp0)
    return out


def hais(z, log_w, target, prior, betas, steps, log_step, log_mass, noise, unif):
    """HAIS.sample after the prior draw: z [N, D], log_w = -log q0(z) -> (samples, log weights, smallest margin per
    row).  target / prior are term lists."""
    n = len(betas) - 1
    margin = np.full(len(z), np.inf)
    for t, i in enumerate(range(n - 1, 0, -1)):
        b = float(betas[i])
        terms = [(b * c, *x) for c, *x in target] + [((1 - b) * c, *x) for c, *x in prior]
        z, ld, _, prob = hmc(z, terms, steps, log_step, log_mass, 0, noise[t], unif[t])
        margin = np.minimum(margin, np.abs(unif[t] - prob) / np.maximum(np.minimum(prob, 1e300), 1e-30))
        log_w = log_w + ld
    return z, log_w + lp_grad(z, target)[0], margin


class Replay:
    """Patches torch.randn / randn_like / rand / rand_like to return stored arrays in call order (as float32 on the
    caller's device): replays the goldens' draws through the package's draw hook and its base distributions."""

    def __init__(self, arrays, device="cuda"):
        import torch
        self.torch, self.arrays, self.device = torch, list(arrays), device

    def _next(self, shape, dtype=None):
        t = self.torch
        a = self.arrays.pop(0)
        a = t.as_tensor(a if t.is_tensor(a) else np.asarray(a), dtype=dtype or t.float32, device=self.device)
        assert tuple(a.shape) == tuple(shape), (a.shape, shape)
        return a.clone()

    def __enter__(self):
        t = self.torch
        self.saved = t.randn, t.randn_like, t.rand, t.rand_like
        shape = lambda s: tuple(s[0]) if len(s) == 1 and isinstance(s[0], (tuple, list)) else tuple(s)
        t.randn = lambda *s, **k: self._next(shape(s))
        t.rand = lambda *s, **k: self._next(shape(s))
        t.randn_like = lambda x, **k: self._next(x.shape, x.dtype)
        t.rand_like = lambda x, **k: self._next(x.shape, x.dtype)
        return self

    def __exit__(self, *a):
        t = self.torch
        t.randn, t.randn_like, t.rand, t.rand_like = self.saved
        assert not self.arrays or a[0] is not None, f"{len(self.arrays)} draws not replayed"
