"""Decoders of the flow-based VAE (reference: normflows/distributions/decoder.py): the likelihood p(x | z) of
`NormalizingFlowVAE`.  Same class names, constructors and `state_dict` keys.

The likelihoods are one kernel each over the net's output, with a native backward (normflows/_vae.py).  When z holds
several samples per data row (rows b S .. b S + S - 1 belong to x[b]), x is read S times in place; the reference
materialises `x.repeat`.  Flat [batch, n] data only."""
import math

import torch
from torch import nn

from .. import _vae


class BaseDecoder(nn.Module):
    def forward(self, z):
        """Decodes z to x."""
        raise NotImplementedError

    def log_prob(self, x, z):
        """log p(x | z)."""
        raise NotImplementedError


def _net_out(net, z, who):
    out = net(z)
    if out.dim() != 2:
        raise NotImplementedError(f"{who}: image-shaped decoder outputs are not on the CUDA path")
    return out


def _repeats(x, z, who):
    """How many consecutive rows of z share one row of x."""
    if x.dim() != 2:
        raise NotImplementedError(f"{who}: flat [batch, n] data only on the CUDA path (got shape {tuple(x.shape)})")
    if len(z) > len(x):
        if len(x) == 0 or len(z) % len(x):
            raise ValueError(f"{who}: {len(z)} latent rows do not repeat {len(x)} data rows")
        return len(z) // len(x)
    if len(z) != len(x):
        raise ValueError(f"{who}: {len(z)} latent rows for {len(x)} data rows")
    return 1


class NNDiagGaussianDecoder(BaseDecoder):
    """Diagonal Gaussian whose mean (first n / 2 outputs) and log variance (the rest) are the net's output."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, z):
        mean_std = _net_out(self.net, z, "NNDiagGaussianDecoder")
        n_hidden = mean_std.size()[1] // 2
        mean = mean_std[:, :n_hidden]
        std = torch.exp(0.5 * mean_std[:, n_hidden:])
        return mean, std

    def log_prob(self, x, z):
        """The normalising constant counts the latent features, z.size()[1:], as the reference's does."""
        mean_std = _net_out(self.net, z, "NNDiagGaussianDecoder")
        rep = _repeats(x, z, "NNDiagGaussianDecoder")
        return _vae.gaussian_log_prob(x, len(z), rep, 1, math.prod(z.shape[1:]), net=mean_std)


class NNBernoulliDecoder(BaseDecoder):
    """Bernoulli distribution with mean sigmoid(net(z))."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def forward(self, z):
        return _vae.sigmoid(_net_out(self.net, z, "NNBernoulliDecoder"))

    def log_prob(self, x, z):
        score = _net_out(self.net, z, "NNBernoulliDecoder")
        return _vae.bernoulli_log_prob(score, x, _repeats(x, z, "NNBernoulliDecoder"))
