"""Unnormalised 2-D densities used as reverse-KL targets (reference: normflows/distributions/prior.py): TwoModes, the
target of examples/real_nvp.ipynb."""
import torch


class TwoModes:
    """Two modes at z[0] = -loc and z[0] = loc on a ring of radius loc:
        log p(z) = -1/2 ((|z| - loc) / (2 scale))^2 - 1/2 ((|z_0| - |loc|) / (3 scale))^2
                   + log(1 + exp(-2 |z_0| |loc| / (3 scale)^2))
    (the last two terms are the log of a symmetric pair of Gaussians in z_0, up to a constant).  Plain tensor arithmetic
    on z's device and dtype; like the reference it holds no parameters or buffers."""

    def __init__(self, loc, scale):
        self.loc = loc
        self.scale = scale

    def log_prob(self, z):
        a = torch.abs(z[:, 0])
        eps = abs(float(self.loc))
        s2, s3 = 2 * self.scale, 3 * self.scale
        return (-0.5 * ((torch.norm(z, dim=1) - self.loc) / s2) ** 2 - 0.5 * ((a - eps) / s3) ** 2
                + torch.log(1 + torch.exp(-2 * a * eps / s3 ** 2)))
