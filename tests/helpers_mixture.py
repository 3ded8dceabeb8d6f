"""Shared by tests/golden/make_mixture_grads.py (run against the reference) and tests/test_gaussian_mixture.py (run
against this package): the models and stored inputs of the Gaussian-mixture cases, and an fp64 numpy restatement of the
mixture's log-density and its gradients.  `nf` is whichever package is passed in; only constructor arguments the
reference and this package share are used."""
import numpy as np
import torch

CASES = ["cbd", "nsf", "loop"]
SEEDS = {"cbd": 51, "nsf": 52, "loop": 53}
DIMS = {"cbd": 2, "nsf": 5, "loop": 2}
SIGMA = {"cbd": 0.01, "nsf": 0.05, "loop": 0.05}


def cbd(nf, num_layers=32):
    """The second model of examples/change_base_distribution.ipynb as written."""
    base = nf.distributions.base.GaussianMixture(2, 2, loc=[[-2, 0], [2, 0]], scale=[[0.3, 0.3], [0.3, 0.3]])
    flows = []
    for i in range(num_layers):
        param_map = nf.nets.MLP([1, 64, 64, 2], init_zeros=True)
        flows.append(nf.flows.AffineCouplingBlock(param_map))
        flows.append(nf.flows.Permute(2, mode='swap'))
    return nf.NormalizingFlow(base, flows)


def build(nf, name):
    torch.manual_seed(SEEDS[name])
    np.random.seed(SEEDS[name])
    if name == "cbd":
        return cbd(nf)
    if name == "nsf":   # autoregressive RQ-NSF + LULinearPermute at D = 5 (the fused path), non-uniform weights
        flows = []
        for _ in range(2):
            flows += [nf.flows.AutoregressiveRationalQuadraticSpline(5, 1, 16), nf.flows.LULinearPermute(5)]
        base = nf.distributions.GaussianMixture(4, 5, weights=[0.1, 0.2, 0.3, 0.4])
        return nf.NormalizingFlow(base, flows)
    flows = []   # loop: residual.ipynb's layers (Residual + ActNorm) on a 3-mode mixture
    for _ in range(2):
        net = nf.nets.LipschitzMLP([2, 16, 16, 2], init_zeros=True, lipschitz_const=0.9)
        flows += [nf.flows.Residual(net, reduce_memory=True), nf.flows.ActNorm(2)]
    base = nf.distributions.GaussianMixture(3, 2, scale=[[0.5, 1.0], [1.0, 0.7], [0.8, 0.8]], weights=[0.5, 0.3, 0.2])
    return nf.NormalizingFlow(base, flows)


def mark_actnorm_done(model):
    for f in model.flows:
        if hasattr(f, "data_dep_init_done"):
            f.data_dep_init_done.fill_(1.0)


def data(name, n=512):
    """The stored inputs x of case `name` (float32)."""
    g = torch.Generator().manual_seed(300 + SEEDS[name])
    return 1.5 * torch.randn(n, DIMS[name], generator=g)


# value cases: constructor kwargs and z; `seed`: loc drawn with np.random.randn after np.random.seed(seed); `ws`: the
# weight_scores set after construction (-800: the reference's softmax underflows to 0 for that mode)
def value_case_model(nf, spec):
    if "seed" in spec:
        np.random.seed(spec["seed"])
    q = nf.distributions.base.GaussianMixture(**spec["kw"])
    if "ws" in spec:
        with torch.no_grad():
            q.weight_scores.copy_(torch.tensor(spec["ws"])[None])
    return q


def value_cases():
    rng = np.random.default_rng(7)
    far = rng.normal(size=(6, 3)) * 1e3
    far[0] = [1e3, -1e3, 1e3]
    return {
        "seeded": dict(seed=5, kw=dict(n_modes=4, dim=3), z=rng.normal(size=(9, 3)) * 2),
        "explicit": dict(kw=dict(n_modes=2, dim=2, loc=[[-2, 0], [2, 0]], scale=[[0.3, 0.3], [0.3, 0.3]]),
                         z=rng.normal(size=(9, 2)) * 2),
        "far": dict(seed=6, kw=dict(n_modes=3, dim=3, scale=[[0.1, 0.2, 0.1], [1, 1, 1], [0.5, 0.5, 0.5]]), z=far),
        "underflow": dict(seed=7, kw=dict(n_modes=3, dim=2), ws=[0.0, -800.0, 0.0], z=rng.normal(size=(9, 2))),
        "k1": dict(seed=8, kw=dict(n_modes=1, dim=4, scale=[[0.5, 1.5, 1.0, 2.0]]), z=rng.normal(size=(9, 4))),
    }


# ---- fp64 numpy restatement (log_softmax in place of log(softmax)) ----------------------------------------------------
def log_prob(z, loc, log_scale, weight_scores):
    """z [N, D], loc / log_scale [K, D], weight_scores [K] -> log p [N]."""
    z, loc, ls, ws = (np.asarray(v, np.float64) for v in (z, loc, log_scale, weight_scores))
    e = _exponents(z, loc, ls, ws)
    m = e.max(1, keepdims=True)
    m = np.where(np.isfinite(m), m, 0.0)
    return (m + np.log(np.exp(e - m).sum(1, keepdims=True)))[:, 0]


def _exponents(z, loc, ls, ws):
    wm = ws.max()
    lw = ws - (wm + np.log(np.exp(ws - wm).sum()))
    t = (z[:, None, :] - loc[None]) * np.exp(-ls)[None]
    return lw[None] - 0.5 * z.shape[1] * np.log(2 * np.pi) - (ls[None] + 0.5 * t * t).sum(2)


def log_prob_grads(z, loc, log_scale, weight_scores, g):
    """Gradients of sum_r g[r] log p(z_r): (g_z, g_loc, g_log_scale, g_weight_scores)."""
    z, loc, ls, ws, g = (np.asarray(v, np.float64) for v in (z, loc, log_scale, weight_scores, g))
    e = _exponents(z, loc, ls, ws)
    lp = log_prob(z, loc, ls, ws)
    a = g[:, None] * np.exp(e - lp[:, None])                         # [N, K]
    inv = np.exp(-ls)
    t = (z[:, None, :] - loc[None]) * inv[None]                     # [N, K, D]
    gz = -(a[:, :, None] * t * inv[None]).sum(1)
    gloc = (a[:, :, None] * t * inv[None]).sum(0)
    gls = (a[:, :, None] * (t * t - 1)).sum(0)
    wm = ws.max()
    sm = np.exp(ws - wm) / np.exp(ws - wm).sum()
    gws = a.sum(0) - sm * g.sum()
    return gz, gloc, gls, gws
