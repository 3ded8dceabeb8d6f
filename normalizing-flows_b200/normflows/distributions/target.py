"""Targets (reference: normflows/distributions/target.py): the Target base class that user targets subclass
(:8-73), and the synthetic 2-D TwoMoons used to generate benchmark/test inputs (:99-129), and TwoIndependent (:76-96)."""
import numpy as np
import torch
from torch import nn


class Target(nn.Module):
    """Base class of sample target distributions (reference: distributions/target.py:8-73): `prop_scale` / `prop_shift`
    buffers of the uniform proposal, rejection sampling against exp(log_prob - max_log_prob).  A subclass sets
    `n_dims` and `max_log_prob` and implements `log_prob` (e.g. examples/paper_example_nsf.ipynb's GaussianVonMises)."""

    def __init__(self, prop_scale=torch.tensor(6.0), prop_shift=torch.tensor(-3.0)):
        super().__init__()
        self.register_buffer("prop_scale", prop_scale)
        self.register_buffer("prop_shift", prop_shift)

    def log_prob(self, z):
        raise NotImplementedError("The log probability is not implemented yet.")

    def rejection_sampling(self, num_steps=1):
        eps = torch.rand((num_steps, self.n_dims), dtype=self.prop_scale.dtype, device=self.prop_scale.device)
        z_ = self.prop_scale * eps + self.prop_shift
        prob = torch.rand(num_steps, dtype=self.prop_scale.dtype, device=self.prop_scale.device)
        prob_ = torch.exp(self.log_prob(z_) - self.max_log_prob)
        return z_[prob_ > prob, :]

    def sample(self, num_samples=1):
        z = torch.zeros((0, self.n_dims), dtype=self.prop_scale.dtype, device=self.prop_scale.device)
        while len(z) < num_samples:
            z_ = self.rejection_sampling(num_samples)
            ind = np.min([len(z_), num_samples - len(z)])
            z = torch.cat([z, z_[:ind, :]], 0)
        return z


class TwoIndependent(Target):
    """Two independent targets of equal size side by side (reference: distributions/target.py:76-96), the augmented
    target of examples/augmented_flow.ipynb: log p(z) = log p1(z1) + log p2(z2) with z1, z2 = z.chunk(2, dim=1).  Both
    targets are sub-modules (`target1`, `target2`), so a DiagGaussian target's loc / log_scale are parameters of a model
    that holds this as `p`, and its state_dict keys are the reference's."""

    def __init__(self, target1, target2):
        super().__init__()
        self.target1 = target1
        self.target2 = target2

    def log_prob(self, z):
        z1, z2 = z.chunk(2, dim=1)
        return self.target1.log_prob(z1) + self.target2.log_prob(z2)

    def sample(self, num_samples=1):
        return torch.cat([self.target1.sample(num_samples), self.target2.sample(num_samples)], 1)


class TwoMoons(nn.Module):
    def __init__(self):
        super().__init__()
        self.n_dims = 2
        self.max_log_prob = 0.0
        self.register_buffer("prop_scale", torch.tensor(6.0))
        self.register_buffer("prop_shift", torch.tensor(-3.0))

    def log_prob(self, z):
        a = torch.abs(z[:, 0])
        return (-0.5 * ((torch.norm(z, dim=1) - 2) / 0.2) ** 2 - 0.5 * ((a - 2) / 0.3) ** 2
                + torch.log(1 + torch.exp(-4 * a / 0.09)))

    def sample(self, num_samples=1):
        out = torch.zeros((0, 2), dtype=self.prop_scale.dtype, device=self.prop_scale.device)
        while len(out) < num_samples:
            eps = torch.rand((num_samples, 2), dtype=out.dtype, device=out.device)
            z = self.prop_scale * eps + self.prop_shift
            accept = torch.rand(num_samples, dtype=out.dtype, device=out.device) < \
                torch.exp(self.log_prob(z) - self.max_log_prob)
            out = torch.cat([out, z[accept]], 0)
        return out[:num_samples]
