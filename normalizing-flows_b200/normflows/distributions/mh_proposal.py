"""Proposals of the Metropolis-Hastings layer (reference: distributions/mh_proposal.py): the same classes, buffer and
draws.  MetropolisHastings runs a DiagGaussianProposal inside its kernel (csrc/nfb_stochastic.cu) when the target is a
native density; these methods are the reference's, used by the generic path."""
import numpy as np
import torch
from torch import nn


class MHProposal(nn.Module):
    """Proposal distribution for the Metropolis Hastings algorithm."""

    def sample(self, z):
        raise NotImplementedError

    def log_prob(self, z_, z):
        raise NotImplementedError

    def forward(self, z):
        """-> (proposal z_, log p(z | z_) - log p(z_ | z))."""
        raise NotImplementedError


class DiagGaussianProposal(MHProposal):
    """Diagonal Gaussian centred at the previous value; `scale` (a buffer, [1] or [1, *shape]) is its standard
    deviation."""

    def __init__(self, shape, scale):
        super().__init__()
        self.shape = shape
        self.scale_cpu = torch.tensor(scale)
        self.register_buffer("scale", self.scale_cpu.unsqueeze(0))

    def sample(self, z):
        eps = torch.randn((len(z),) + self.shape, dtype=z.dtype, device=z.device)
        return eps * self.scale + z

    def log_prob(self, z_, z):
        return -0.5 * np.prod(self.shape) * np.log(2 * np.pi) - torch.sum(
            torch.log(self.scale) + 0.5 * torch.pow((z_ - z) / self.scale, 2), list(range(1, z.dim())))

    def forward(self, z):
        eps = torch.randn((len(z),) + self.shape, dtype=z.dtype, device=z.device)
        return eps * self.scale + z, torch.zeros(len(z), dtype=z.dtype, device=z.device)
