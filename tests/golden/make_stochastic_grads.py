"""Mint goldens of the stochastic layers and HAIS from the REAL reference (a checkout found by oracle/reference.py, no GPU
needed): fp64 autograd on stored draws.
    python tests/golden/make_stochastic_grads.py
Writes tests/golden/stochastic_<case>.npz:
    hmc_a   HamiltonianMonteCarlo(GaussianMixture(3, 4), 5 leapfrog steps), max_abs_grad=None: z_out, log_det and the
            gradients of sum <w_z, z_out> + <w_ld, log_det> w.r.t. z, log_step_size, log_mass and the mixture's parameters
    hmc_b   the same with max_abs_grad=1.5 (part of the gradients clamp)
    mh      MetropolisHastings(DiagGaussian(4), DiagGaussianProposal((4,), 0.6), 5): the same outputs and gradients
    hais    HAIS(linspace(1, 0, 20), DiagGaussian(4), GaussianMixture(3, 4), 5, 0.15, 0): samples and log weights
    snf     NormalizingFlow(DiagGaussian(4), [MaskedAffineFlow, ActNorm, HamiltonianMonteCarlo] x 2, p=GaussianMixture):
            reverse_kld and the gradient of every parameter
The draws are replayed by patching torch's samplers in the order the reference calls them.  Only rows whose every
accept test has a margin |u - P| of at least 1e-4 (relative) are kept, so a float32 run takes the same decisions."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import nf  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_stochastic as H  # noqa: E402

MARGIN = 1e-4
D, K = 4, 3


class Replay:
    """Patches torch.randn / randn_like / rand / rand_like to return the stored arrays in call order; rand_like records
    its argument (HMC's acceptance probabilities)."""

    def __init__(self, arrays):
        self.arrays, self.probs = list(arrays), []

    def _next(self, shape):
        a = torch.as_tensor(self.arrays.pop(0), dtype=torch.float64)
        assert tuple(a.shape) == tuple(shape), (a.shape, shape)
        return a.clone()

    def __enter__(self):
        self.saved = torch.randn, torch.randn_like, torch.rand, torch.rand_like
        torch.randn = lambda *s, **k: self._next(s[0] if len(s) == 1 and isinstance(s[0], (tuple, list)) else s)
        torch.randn_like = lambda t, **k: self._next(t.shape)
        torch.rand = lambda *s, **k: self._next(s[0] if len(s) == 1 and isinstance(s[0], (tuple, list)) else s)

        def rand_like(t, **k):
            self.probs.append(t.detach().clone())
            return self._next(t.shape)
        torch.rand_like = rand_like
        return self

    def __exit__(self, *a):
        torch.randn, torch.randn_like, torch.rand, torch.rand_like = self.saved


def mixture(seed):
    g = np.random.default_rng(seed)
    loc = g.normal(0, 1.5, (K, D))
    scale = np.exp(g.normal(-0.2, 0.25, (K, D)))
    w = g.uniform(0.5, 1.5, K)
    gm = nf.distributions.GaussianMixture(K, D, loc=loc, scale=scale, weights=w).double()
    return gm


def terms_of(gm):
    return [(1.0, gm.loc[0].detach().numpy(), gm.log_scale[0].detach().numpy(),
             gm.weight_scores[0].detach().numpy())]


def diag_terms(dg):
    return [(1.0, dg.loc.detach().numpy().reshape(1, -1), dg.log_scale.detach().numpy().reshape(1, -1), np.zeros(1))]


def case_hmc(mag, seed):
    g = np.random.default_rng(seed)
    gm = mixture(seed)
    ls = np.log(0.12) + g.normal(0, 0.1, D)
    lm = g.normal(0, 0.2, D)
    n = 1024
    z = g.normal(0, 1.8, (n, D))
    noise = g.normal(size=(n, D))
    unif = g.uniform(size=n)
    *_, prob = H.hmc(z, terms_of(gm), 5, ls, lm, mag, noise, unif)
    keep = (np.abs(unif - prob) / np.maximum(np.minimum(prob, 1e300), 1e-30) >= MARGIN)
    z, noise, unif = z[keep][:256], noise[keep][:256], unif[keep][:256]
    w_z, w_ld = g.normal(size=z.shape), g.normal(size=len(z))
    layer = nf.flows.HamiltonianMonteCarlo(gm, 5, torch.tensor(ls), torch.tensor(lm), max_abs_grad=mag)
    zt = torch.tensor(z, requires_grad=True)
    with Replay([noise, unif]):
        z_out, ld = layer(zt)
    loss = (torch.tensor(w_z) * z_out).sum() + (torch.tensor(w_ld) * ld).sum()
    loss.backward()
    out = dict(z=z, noise=noise, unif=unif, w_z=w_z, w_ld=w_ld, log_step_size=ls, log_mass=lm,
               loc=gm.loc[0].detach().numpy(), log_scale=gm.log_scale[0].detach().numpy(),
               weight_scores=gm.weight_scores[0].detach().numpy(), steps=np.array(5), max_abs_grad=np.array(mag or 0.0),
               z_out=z_out.detach().numpy(), log_det=ld.detach().numpy(), g_z=zt.grad.numpy(),
               g_log_step_size=layer.log_step_size.grad.numpy(), g_log_mass=layer.log_mass.grad.numpy(),
               g_loc=gm.loc.grad[0].numpy(), g_log_scale=gm.log_scale.grad[0].numpy(),
               g_weight_scores=gm.weight_scores.grad[0].numpy(),
               sd_keys=np.array(sorted(layer.state_dict().keys())))
    return out


def case_mh(seed=3):
    g = np.random.default_rng(seed)
    dg = nf.distributions.DiagGaussian(D).double()
    with torch.no_grad():
        dg.loc.copy_(torch.tensor(g.normal(0, 0.5, (1, D))))
        dg.log_scale.copy_(torch.tensor(g.normal(0, 0.3, (1, D))))
    steps, n = 5, 1024
    z = g.normal(0, 1.5, (n, D))
    noise = g.normal(size=(steps, n, D))
    unif = g.uniform(size=(steps, n))
    keep = H.mh_margin(z, diag_terms(dg), steps, 0.6, noise, unif) >= MARGIN
    z, noise, unif = z[keep][:256], noise[:, keep][:, :256], unif[:, keep][:, :256]
    w_z, w_ld = g.normal(size=z.shape), g.normal(size=len(z))
    layer = nf.flows.MetropolisHastings(dg, nf.distributions.DiagGaussianProposal((D,), 0.6), steps).double()
    zt = torch.tensor(z, requires_grad=True)
    seq = []
    for s in range(steps):
        seq += [noise[s], unif[s]]
    with Replay(seq):
        z_out, ld = layer(zt)
    loss = (torch.tensor(w_z) * z_out).sum() + (torch.tensor(w_ld) * ld).sum()
    loss.backward()
    return dict(z=z, noise=noise, unif=unif, w_z=w_z, w_ld=w_ld, scale=np.array(0.6), steps=np.array(steps),
                loc=dg.loc.detach().numpy()[0], log_scale=dg.log_scale.detach().numpy()[0],
                z_out=z_out.detach().numpy(), log_det=ld.detach().numpy(), g_z=zt.grad.numpy(),
                g_loc=dg.loc.grad.numpy()[0], g_log_scale=dg.log_scale.grad.numpy()[0],
                sd_keys=np.array(sorted(layer.state_dict().keys())),
                sd_scale=layer.state_dict()["proposal.scale"].numpy())


def case_hais(seed=4):
    g = np.random.default_rng(seed)
    gm = mixture(seed)
    prior = nf.distributions.DiagGaussian(D, trainable=False).double()
    betas = torch.linspace(1, 0, 20, dtype=torch.float64)
    T = len(betas) - 2
    n = 2048
    eps = g.normal(size=(n, D))
    noise = g.normal(size=(T, n, D))
    unif = g.uniform(size=(T, n))
    z0 = eps
    lq0 = -0.5 * D * np.log(2 * np.pi) - 0.5 * (eps ** 2).sum(1)
    *_, margin = H.hais(z0, -lq0, terms_of(gm), diag_terms(prior), betas.numpy(), 5, np.full(D, np.log(0.15)),
                        np.zeros(D), noise, unif)
    keep = margin >= MARGIN
    eps, noise, unif = eps[keep][:256], noise[:, keep][:, :256], unif[:, keep][:, :256]
    seq = [eps]
    for t in range(T):
        seq += [noise[t], unif[t]]
    h = nf.HAIS(betas, prior, gm, 5, torch.full((D,), 0.15, dtype=torch.float64), torch.zeros(D, dtype=torch.float64))
    with Replay(seq):   # (the reference's gradlogP needs grad mode)
        samples, log_w = h.sample(len(eps))
    return dict(eps=eps, noise=noise, unif=unif, betas=betas.numpy(), loc=gm.loc[0].detach().numpy(),
                log_scale=gm.log_scale[0].detach().numpy(), weight_scores=gm.weight_scores[0].detach().numpy(),
                samples=samples.detach().numpy(), log_w=log_w.detach().numpy())


def snf_model(gm, seed):
    torch.manual_seed(seed)
    flows = []
    for i in range(2):
        b = torch.tensor([(j + i) % 2 for j in range(D)], dtype=torch.float64)
        s = nf.nets.MLP([D, 16, D], init_zeros=True)
        t = nf.nets.MLP([D, 16, D], init_zeros=True)
        flows += [nf.flows.MaskedAffineFlow(b, t, s), nf.flows.ActNorm(D),
                  nf.flows.HamiltonianMonteCarlo(gm, 3, torch.full((D,), np.log(0.1)), torch.zeros(D))]
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows, p=gm).double()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.05 * torch.randn_like(p))
    for m in model.modules():
        if hasattr(m, "data_dep_init_done"):
            m.data_dep_init_done.fill_(1.0)
    return model


def case_snf(seed=5):
    g = np.random.default_rng(seed)
    gm = mixture(seed)
    n = 1024
    eps = g.normal(size=(n, D))
    draws = [g.normal(size=(n, D)), g.uniform(size=n), g.normal(size=(n, D)), g.uniform(size=n)]
    model = snf_model(gm, seed)
    rep = Replay([eps] + draws)
    with rep:
        model.reverse_kld(n)
    keep = np.ones(n, bool)
    for (pr, u) in zip(rep.probs, (draws[1], draws[3])):
        pr = pr.numpy()
        keep &= np.abs(u - pr) / np.maximum(np.minimum(pr, 1e300), 1e-30) >= MARGIN
    eps, draws = eps[keep][:256], [d[keep][:256] for d in draws]
    model = snf_model(gm, seed)
    with Replay([eps] + draws):
        loss = model.reverse_kld(len(eps))
    loss.backward()
    out = dict(eps=eps, n0=draws[0], u0=draws[1], n1=draws[2], u1=draws[3], loss=np.array(loss.item()))
    for k, v in model.state_dict().items():
        out["sd__" + k] = v.numpy()
    for k, p in model.named_parameters():
        out["g__" + k] = p.grad.numpy()
    return out


def main():
    cases = {"hmc_a": lambda: case_hmc(None, 1), "hmc_b": lambda: case_hmc(1.5, 2), "mh": case_mh,
             "hais": case_hais, "snf": case_snf}
    for name in sys.argv[1:] or cases:
        out = cases[name]()
        np.savez_compressed(os.path.join(HERE, f"stochastic_{name}.npz"), **out)
        print(name, {k: np.shape(v) for k, v in out.items() if not k.startswith("sd__")})


if __name__ == "__main__":
    main()
