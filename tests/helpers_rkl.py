"""Shared by tests/golden/make_reverse_kld_grads.py (run against the reference) and tests/test_reverse_kld_training.py
(run against this package): the targets of the reverse-KL cases h-l and the replay of a base distribution's stored
random draws, which makes the loss a deterministic function of the parameters.  Only attribute names the reference and
this package share are used (`scale` of UniformGaussian, `loc` / `log_scale` of DiagGaussian)."""
import math

import numpy as np
import torch
from torch import nn


def gaussian_von_mises(target_base):
    """examples/paper_example_nsf.ipynb's target, subclassing `target_base` (nf.distributions.Target)."""
    class GaussianVonMises(target_base):
        def __init__(self):
            super().__init__(prop_scale=torch.tensor(2 * np.pi), prop_shift=torch.tensor(-np.pi))
            self.n_dims = 2
            self.max_log_prob = -1.99
            self.log_const = -1.5 * np.log(2 * np.pi) - np.log(np.i0(1))

        def log_prob(self, x):
            return -0.5 * x[:, 0] ** 2 + torch.cos(x[:, 1] - 3 * x[:, 0]) + self.log_const
    return GaussianVonMises()


class TorusTarget5(nn.Module):
    """Case j: circular features 1 and 3 coupled to the linear ones."""

    def log_prob(self, z):
        return (-0.5 * (z[:, 0] ** 2 + z[:, 2] ** 2 + z[:, 4] ** 2) - 0.25 * (z[:, 2] - z[:, 0]) ** 2
                + torch.cos(z[:, 1] - z[:, 0]) + 2 * torch.cos(z[:, 3]))


class TorusTarget3(nn.Module):
    """Case k: feature 1 circular."""

    def log_prob(self, z):
        return -0.5 * z[:, 0] ** 2 - 0.5 * (z[:, 2] - 0.5 * z[:, 0]) ** 2 + torch.cos(z[:, 1] - 2 * z[:, 0])


class ContextTarget(nn.Module):
    """Case l: N(context[:, :2], exp(context[:, 2:])) per row."""

    def log_prob(self, z, context=None):
        return -0.5 * torch.sum(((z - context[:, :2]) * torch.exp(-0.5 * context[:, 2:])) ** 2, 1) \
            - 0.5 * torch.sum(context[:, 2:], 1)


def replay_forward(q0, eps):
    """A `forward(num_samples, context=None)` for q0 that returns the base's sample for the stored draws eps [n, d]
    (the standardised draw: UniformGaussian z = scale * eps, DiagGaussian z = loc + exp(log_scale) * eps) and its
    log-density, with the base's own reparameterised formula."""
    def forward(num_samples=1, context=None):
        assert num_samples == eps.shape[0]
        if hasattr(q0, "inv_perm"):   # UniformGaussian
            e = eps.to(dtype=q0.scale.dtype, device=q0.scale.device)
            z = q0.scale * e
            return z, q0.log_prob(z)
        e = eps.to(dtype=q0.loc.dtype, device=q0.loc.device)
        ls = q0.log_scale
        z = q0.loc + torch.exp(ls) * e
        log_p = -0.5 * e.shape[1] * math.log(2 * math.pi) - torch.sum(ls + 0.5 * e ** 2, 1)
        return z, log_p
    return forward


def draws(name, n=512):
    """The stored standardised base draws of case `name` (float32)."""
    g = torch.Generator().manual_seed({"h": 108, "i": 108, "j": 110, "k": 111, "l": 112}[name])
    if name in ("h", "i"):   # UniformGaussian(2, [1]): feature 1 uniform on [-0.5, 0.5), feature 0 standard normal
        eps = torch.stack([torch.randn(n, generator=g), torch.rand(n, generator=g) - 0.5], 1)
        eps[:6, 0] = torch.tensor([5.3, -5.6, 6.1, -7.0, 5.05, -5.9])   # beyond the tail bound 5 of feature 0
        return eps
    d = {"j": 5, "k": 3, "l": 2}[name]
    return torch.randn(n, d, generator=g)


def context_of(n=512):
    """Case l's context [n, 4]: means in [-1, 1], log-variances in [-1, 1]."""
    return torch.rand(n, 4, generator=torch.Generator().manual_seed(113)) * 2 - 1
