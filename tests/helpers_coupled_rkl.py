"""Shared by tests/golden/make_coupled_rkl_grads.py (run against the reference) and tests/test_coupled_rkl_training.py
(run against this package): the models, targets and stored base draws of the reverse-KL cases w-z (coupled spline +
LULinearPermute stacks).  The base's draws are replayed with helpers_rkl.replay_forward, so each loss is a deterministic
function of the parameters.  Only constructor arguments and attribute names the reference and this package share are
used."""
import torch
from torch import nn

SEEDS = {"w": 20, "x": 20, "y": 22, "z": 23}


class Target6(nn.Module):
    """Cases w / x: heavy-tailed (log-Cauchy-like in each residual, so log p - log q stays within float32's exp range
    for the draws beyond the tail bound), a linear pair (0, 1), a sine ridge (2 -> 3), a cosine coupling of (3, 5)."""

    def log_prob(self, z):
        r = torch.stack([z[:, 0], z[:, 1] - 0.6 * z[:, 0], z[:, 2], z[:, 3] - 0.5 * torch.sin(z[:, 2]), z[:, 4],
                         z[:, 5] - 0.4 * z[:, 4]], 1)
        return -torch.sum(torch.log1p(r ** 2 / 4), 1) + 0.5 * torch.cos(z[:, 5] - z[:, 3])


class Target64(nn.Module):
    """Case y: a Gaussian chain, each feature tied to its neighbour."""

    def log_prob(self, z):
        return -0.5 * torch.sum((z[:, 1:] - 0.5 * z[:, :-1]) ** 2, 1) - 0.5 * z[:, 0] ** 2


class Target5(nn.Module):
    """Case z: correlated pairs and a quartic well."""

    def log_prob(self, z):
        return (-0.5 * (z[:, 0] ** 2 + (z[:, 1] - 0.8 * z[:, 0]) ** 2 + z[:, 2] ** 2 + (z[:, 3] + 0.5 * z[:, 2]) ** 2)
                - 0.1 * z[:, 4] ** 4)


def build(nf, name):
    """The model of case `name` built with `nf` (the reference or this package), seeded construction."""
    torch.manual_seed(SEEDS[name])
    Cq, LU = nf.flows.CoupledRationalQuadraticSpline, nf.flows.LULinearPermute
    if name in ("w", "x"):
        flows = []
        for i in range(4):
            flows += [Cq(6, 2, 64, reverse_mask=bool(i % 2)), LU(6)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(6), flows, Target6())
    if name == "y":
        flows = []
        for i in range(2):
            flows += [Cq(64, 2, 256, reverse_mask=bool(i % 2)), LU(64)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(64), flows, Target64())
    flows = [Cq(5, 1, 32, reverse_mask=bool(i % 2)) for i in range(3)]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows, Target5())


def loss_of(name, model, n):
    """The case's loss on the replayed draws (model.q0.forward patched by helpers_rkl.replay_forward)."""
    if name in ("w", "y"):
        return model.reverse_kld(n)
    if name == "x":
        return model.reverse_alpha_div(n, alpha=1, dreg=True)
    return model.reverse_kld(n, score_fn=False)


def draws(name):
    """The stored standardised base draws of case `name` (float32)."""
    g = torch.Generator().manual_seed(100 + SEEDS[name])
    if name in ("w", "x"):
        eps = torch.randn(512, 6, generator=g)
        eps[:8, :] = torch.tensor([[3.4, -3.7, 4.2, -3.2, 3.9, -4.6]]) * torch.tensor([1., -1.]).repeat(4)[:, None]
        return eps
    if name == "y":   # candidates: make_coupled_rkl_grads.py keeps the first 256 rows clear of every ReLU kink
        return torch.randn(1024, 64, generator=g)
    return torch.randn(512, 5, generator=g)
