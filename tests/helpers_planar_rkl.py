"""Shared by tests/golden/make_planar_rkl_grads.py (run against the reference) and tests/test_planar_radial_training.py
(run against this package): the models, targets, stored base draws and data of the planar / radial cases r-v, which
continue the lettering of helpers_affine_rkl.py.  `nf` is whichever package is passed in; only constructor arguments
the reference and this package share are used."""
import math

import torch
from torch import nn

SEEDS = {"r": 18, "s": 19, "t": 20, "u": 20, "v": 22}
DIMS = {"r": 2, "s": 2, "t": 5, "u": 5, "v": 40}


class GaussTarget(nn.Module):
    """Cases t-v: an axis-aligned Gaussian (unnormalised) with means 0.5 sin(j) and scales 1 + 0.5 cos(j) / 2."""

    def __init__(self, d):
        super().__init__()
        j = torch.arange(d, dtype=torch.float64)
        self.mean = 0.5 * torch.sin(j)
        self.std = 1 + 0.25 * torch.cos(j)

    def log_prob(self, z):
        return -0.5 * torch.sum(((z - self.mean.to(z)) / self.std.to(z)) ** 2, 1)


def notebook_targets(nf):
    """The five targets of examples/comparison_plan_rad_aff.ipynb."""
    d = nf.distributions
    return {"TwoModes": d.TwoModes(2.0, 0.2), "Sinusoidal": d.Sinusoidal(0.4, 4), "Sinusoidal_gap": d.Sinusoidal_gap(0.4, 4),
            "Sinusoidal_split": d.Sinusoidal_split(0.4, 4), "Smiley": d.Smiley(0.15)}


def build(nf, name):
    torch.manual_seed(SEEDS[name])
    if name == "r":          # examples/planar.ipynb, 8 instead of 16 layers
        flows = [nf.flows.Planar((2,)) for _ in range(8)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, nf.distributions.TwoModes(2, 0.1))
    if name == "s":
        flows = [nf.flows.Radial((2,)) for _ in range(8)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, nf.distributions.Smiley(0.15))
    if name in ("t", "u"):
        flows = [nf.flows.Planar((5,), act="leaky_relu") for _ in range(6)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows, GaussTarget(5))
    flows = []               # v: the VAE notebook's latent size
    for _ in range(10):
        flows += [nf.flows.Planar((40,)), nf.flows.Radial((40,))]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(40), flows, GaussTarget(40))


def draws(name, n=512):
    """The stored standardised base draws of case `name` (float32)."""
    g = torch.Generator().manual_seed(200 + SEEDS[name])
    return torch.randn(n, DIMS[name], generator=g)


def data(n=512):
    """Case u's data for forward_kld."""
    g = torch.Generator().manual_seed(321)
    return 0.8 * torch.randn(n, 5, generator=g) + 0.3


def loss_of(name, model, n, x=None):
    if name == "r":
        return model.reverse_kld(n, beta=0.5)
    if name == "t":
        return model.reverse_kld(n, score_fn=False)
    if name == "u":
        return model.forward_kld(x)
    return model.reverse_kld(n)


def replay_forward(q0, eps):
    """A `forward(num_samples)` for a DiagGaussian q0 that returns loc + exp(log_scale) eps and its log-density."""
    def forward(num_samples=1, context=None):
        assert num_samples == eps.shape[0]
        e = eps.to(dtype=q0.loc.dtype, device=q0.loc.device)
        ls = q0.log_scale
        return q0.loc + torch.exp(ls) * e, -0.5 * e.shape[1] * math.log(2 * math.pi) - torch.sum(ls + 0.5 * e ** 2, 1)
    return forward
