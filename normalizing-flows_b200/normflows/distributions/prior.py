"""Unnormalised 2-D densities used as reverse-KL targets (reference: normflows/distributions/prior.py): TwoModes, the
target of examples/real_nvp.ipynb and planar.ipynb, and Sinusoidal, Sinusoidal_gap, Sinusoidal_split and Smiley, the
targets of examples/comparison_plan_rad_aff.ipynb."""
import math

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


def _features_first(z):
    """z with its last axis moved to the front: z_[0], z_[1] are the two coordinates of a batch of any shape."""
    return z.permute((z.dim() - 1,) + tuple(range(z.dim() - 1))) if z.dim() > 1 else z


def _envelope(z_, scale):
    """-1/2 (|z|_4 / (20 scale))^4: a wide quartic envelope that makes the sinusoidal densities normalisable."""
    return -0.5 * (torch.norm(z_, dim=0, p=4) / (20 * scale)) ** 4


def _sin_curve(z_, period):
    return torch.sin(2 * math.pi / period * z_[0])


def _split_pair(a, eps, scale):
    """log of a symmetric pair of Gaussians at +-eps in a (up to a constant), as TwoModes writes it."""
    return -0.5 * ((a - eps) / scale) ** 2 + torch.log(1 + torch.exp(-2 * (eps * a) / scale ** 2))


class Sinusoidal:
    """Mass along the curve z_1 = sin(2 pi z_0 / period) (examples/comparison_plan_rad_aff.ipynb):
        log p(z) = -1/2 ((z_1 - sin(2 pi z_0 / period)) / scale)^2 - 1/2 (|z|_4 / (20 scale))^4
    The last axis of z holds the two coordinates; plain tensor arithmetic on z's device and dtype."""

    def __init__(self, scale, period):
        self.scale = scale
        self.period = period

    def log_prob(self, z):
        z_ = _features_first(z)
        return -0.5 * ((z_[1] - _sin_curve(z_, self.period)) / self.scale) ** 2 + _envelope(z_, self.scale)


class Sinusoidal_gap:
    """Two copies of the sinusoidal curve, the second shifted down by w_2(z_0) = 3 exp(-1/2 ((z_0 - 1) / 0.6)^2), so that
    they part around z_0 = 1: a symmetric Gaussian pair at +-w_2 / 2 about the curve's midline, times the envelope."""

    def __init__(self, scale, period):
        self.scale = scale
        self.period = period
        self.w2_scale = 0.6
        self.w2_amp = 3.0
        self.w2_mu = 1.0

    def log_prob(self, z):
        z_ = _features_first(z)
        w2 = self.w2_amp * torch.exp(-0.5 * ((z_[0] - self.w2_mu) / self.w2_scale) ** 2)
        eps = torch.abs(w2 / 2)
        a = torch.abs(z_[1] - _sin_curve(z_, self.period) + w2 / 2)
        return _split_pair(a, eps, self.scale) + _envelope(z_, self.scale)


class Sinusoidal_split:
    """Like Sinusoidal_gap with the shift w_3(z_0) = 3 sigmoid((z_0 - 1) / 0.3): the two copies split for good past
    z_0 = 1."""

    def __init__(self, scale, period):
        self.scale = scale
        self.period = period
        self.w3_scale = 0.3
        self.w3_amp = 3.0
        self.w3_mu = 1.0

    def log_prob(self, z):
        z_ = _features_first(z)
        w3 = self.w3_amp * torch.sigmoid((z_[0] - self.w3_mu) / self.w3_scale)
        eps = torch.abs(w3 / 2)
        a = torch.abs(z_[1] - _sin_curve(z_, self.period) + w3 / 2)
        return _split_pair(a, eps, self.scale) + _envelope(z_, self.scale)


class Smiley:
    """A ring of radius 2 and a mouth: log p(z) = -1/2 ((|z| - 2) / (2 scale))^2 - 1/2 ((|z_1 + 0.8| - 1.2) / (2 scale))^2."""

    def __init__(self, scale):
        self.scale = scale
        self.loc = 2.0

    def log_prob(self, z):
        z_ = _features_first(z)
        return (-0.5 * ((torch.norm(z_, dim=0) - self.loc) / (2 * self.scale)) ** 2
                - 0.5 * ((torch.abs(z_[1] + 0.8) - 1.2) / (2 * self.scale)) ** 2)
