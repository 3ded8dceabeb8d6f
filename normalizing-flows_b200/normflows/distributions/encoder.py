"""Encoders of the flow-based VAE (reference: normflows/distributions/encoder.py): the base distribution q0(z | x) of
`NormalizingFlowVAE`.  Same class names, constructors and `state_dict` keys.

The reparameterised draws of ConstDiagGaussian and NNDiagGaussian run in one kernel each (mean + sd eps and log q,
csrc/nfb_vae.cu), their log_prob in one more, and each has a native backward (normflows/_vae.py).  Flat [batch, n] data
only.  Dirac and Uniform build log_q on the device of x; the reference builds it on the CPU (so its VAE fails on CUDA
with these encoders)."""
import numpy as np
import torch
from torch import nn

from .. import _vae


class BaseEncoder(nn.Module):
    """Base distribution of a flow-based variational autoencoder; its parameters depend on the conditioning x."""

    def forward(self, x, num_samples=1):
        """(z [batch, num_samples, ...], log q(z | x) [batch, num_samples])."""
        raise NotImplementedError

    def log_prob(self, z, x):
        raise NotImplementedError

    def _draw_eps(self, shape, device):
        """The standard-normal draw of a reparameterised encoder, at the point of the step where the reference draws
        it (so a seeded run draws the same noise); tests replace it to replay stored draws."""
        return torch.randn(shape, device=device)


def _flat_data(x, who):
    if x.dim() != 2:
        raise NotImplementedError(f"{who}: flat [batch, n] data only on the CUDA path (got shape {tuple(x.shape)})")


class Dirac(BaseEncoder):
    def forward(self, x, num_samples=1):
        z = x.unsqueeze(1).repeat(1, num_samples, 1)
        log_q = torch.zeros(z.size()[0:2], device=x.device)
        return z, log_q

    def log_prob(self, z, x):
        return torch.zeros(z.size()[0:2], device=z.device)


class Uniform(BaseEncoder):
    def __init__(self, zmin=0.0, zmax=1.0):
        super().__init__()
        self.zmin = zmin
        self.zmax = zmax
        self.log_q = -np.log(zmax - zmin)

    def forward(self, x, num_samples=1):
        z = x.unsqueeze(1).repeat(1, num_samples, 1).uniform_(self.zmin, self.zmax)
        log_q = torch.zeros(z.size()[0:2], device=x.device).fill_(self.log_q)
        return z, log_q

    def log_prob(self, z, x):
        return torch.zeros(z.size()[0:2], device=z.device).fill_(self.log_q)


class ConstDiagGaussian(BaseEncoder):
    def __init__(self, loc, scale):
        """Diagonal Gaussian whose parameters do not depend on x: `loc` the mean, `scale` the standard deviations (a
        scale, not a log-scale: a negative entry gives NaN, as in the reference)."""
        super().__init__()
        self.d = len(loc)
        if not torch.is_tensor(loc):
            loc = torch.tensor(loc)
        if not torch.is_tensor(scale):
            scale = torch.tensor(scale)
        if scale.numel() not in (1, self.d):
            raise ValueError(f"ConstDiagGaussian: scale has {scale.numel()} entries for {self.d} features (expected "
                             f"{self.d}, or 1 to broadcast)")
        self.loc = nn.Parameter(loc.reshape((1, 1, self.d)))
        self.scale = nn.Parameter(scale)

    def _scale(self):
        """The d standard deviations: a one-element scale broadcasts over the features, as in the reference."""
        return self.scale.reshape(-1).expand(self.d) if self.scale.numel() != self.d else self.scale

    def forward(self, x=None, num_samples=1):
        batch_size = len(x) if x is not None else 1
        device = x.device if x is not None else self.loc.device
        eps = self._draw_eps((batch_size, num_samples, self.d), device)
        return _vae.reparam_sample(eps, loc=self.loc, scale=self._scale())

    def log_prob(self, z, x):
        """log q(z) over the last dimension; z [d] and [batch, d] are read as the reference reads them ([1, 1, d],
        [1, batch, d])."""
        if z.dim() == 1:
            z = z.unsqueeze(0)
        if z.dim() == 2:
            z = z.unsqueeze(0)
        rows = z.shape[0] * z.shape[1]
        v = z.reshape(rows, z.shape[2])
        return _vae.gaussian_log_prob(v, rows, 1, max(rows, 1), self.d, loc=self.loc,
                                      scale=self._scale()).reshape(z.shape[:2])


class NNDiagGaussian(BaseEncoder):
    """Diagonal Gaussian whose mean (first n / 2 outputs) and log variance (next n / 2) are the net's output."""

    def __init__(self, net):
        super().__init__()
        self.net = net

    def _net_out(self, x):
        _flat_data(x, "NNDiagGaussian")
        out = self.net(x)
        if out.dim() != 2:
            raise NotImplementedError("NNDiagGaussian: image-shaped encoder outputs are not on the CUDA path")
        return out

    def forward(self, x, num_samples=1):
        mean_std = self._net_out(x)
        eps = self._draw_eps((len(x), num_samples, mean_std.shape[1] // 2), x.device)
        return _vae.reparam_sample(eps, net=mean_std)

    def log_prob(self, z, x):
        """log q(z | x) for z [batch, num_samples, d] (row b of z belongs to x[b]) -> [batch, num_samples]."""
        if z.dim() != 3 or z.shape[0] != len(x):
            raise NotImplementedError("NNDiagGaussian.log_prob takes z of shape [batch, num_samples, d] on the CUDA "
                                      f"path (got {tuple(z.shape)} for a batch of {len(x)})")
        mean_std = self._net_out(x)
        B, S, d = z.shape
        out = _vae.gaussian_log_prob(z.reshape(B * S, d), B * S, 1, S, d, net=mean_std)
        return out.reshape(B, S)
