"""Shared by tests/golden/make_affine_rkl_grads.py (run against the reference) and tests/test_affine_rkl_training.py
(run against this package): the models, targets and stored base draws of the Real NVP reverse-KL cases m-q.  `nf` is
whichever package is passed in; only constructor arguments the reference and this package share are used."""
import torch
from torch import nn

import helpers_rkl as R

SEEDS = {"m": 13, "n": 13, "o": 15, "p": 16, "q": 17}
DIMS = {"m": 2, "n": 2, "o": 4, "p": 5, "q": 2}


class Gauss5Target(nn.Module):
    """Case p: a correlated 5-D Gaussian (unnormalised)."""

    def log_prob(self, z):
        return (-0.5 * ((z[:, 0] - 1) ** 2 + z[:, 1] ** 2 / 4 + (z[:, 2] - 0.5 * z[:, 0]) ** 2 + z[:, 3] ** 2
                        + (z[:, 4] + z[:, 1]) ** 2 / 2))


def build(nf, name):
    torch.manual_seed(SEEDS[name])
    if name in ("m", "n"):   # examples/real_nvp.ipynb, 8 instead of 64 layer pairs
        b = torch.Tensor([1, 0])
        flows = []
        for i in range(8):
            s = nf.nets.MLP([2, 4, 2], init_zeros=True)
            t = nf.nets.MLP([2, 4, 2], init_zeros=True)
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(2)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, nf.distributions.TwoModes(2, 0.1))
    if name == "o":          # examples/augmented_flow.ipynb, 4 instead of 32 layer pairs
        b = torch.Tensor([1, 1, 0, 0])
        flows = []
        for i in range(4):
            s = nf.nets.MLP([4, 16, 4], init_zeros=True)
            t = nf.nets.MLP([4, 16, 4], init_zeros=True)
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(4)]
        target = nf.distributions.TwoIndependent(nf.distributions.TwoMoons(), nf.distributions.DiagGaussian(2))
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(4), flows, target)
    if name == "p":          # every op variant at D = 5
        b = torch.Tensor([1, 0, 1, 0, 1])
        mlp = lambda i, o: nf.nets.MLP([i, 8, o], leaky=0.2)
        flows = [nf.flows.AffineCouplingBlock(mlp(3, 4), True, "exp", "channel"),
                 nf.flows.Permute(5, "swap"),
                 nf.flows.AffineCouplingBlock(mlp(2, 6), True, "sigmoid", "channel_inv"),
                 nf.flows.MaskedAffineFlow(b, None, mlp(5, 5)),
                 nf.flows.Permute(5, "shuffle"),
                 nf.flows.AffineCouplingBlock(mlp(3, 4), True, "sigmoid_inv", "channel"),
                 nf.flows.MaskedAffineFlow(1 - b, mlp(5, 5), None),
                 nf.flows.AffineCouplingBlock(mlp(2, 3), False, "exp", "channel_inv"),
                 nf.flows.AffineConstFlow((5,), scale=False),
                 nf.flows.ActNorm(5)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows, Gauss5Target())
    b = torch.Tensor([1, 0])  # q: layer loop, a context spline layer between MaskedAffineFlow + ActNorm pairs
    flows = [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([2, 8, 2]), nf.nets.MLP([2, 8, 2])), nf.flows.ActNorm(2),
             nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 32, num_context_channels=4),
             nf.flows.MaskedAffineFlow(1 - b, nf.nets.MLP([2, 8, 2]), nf.nets.MLP([2, 8, 2])), nf.flows.ActNorm(2)]
    return nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows, R.ContextTarget())


def mark_actnorm_done(model):
    for f in model.flows:
        if hasattr(f, "data_dep_init_done"):
            f.data_dep_init_done.fill_(1.0)


def draws(name, n=512):
    """The stored standardised base draws of case `name` (float32)."""
    g = torch.Generator().manual_seed(100 + SEEDS[name])
    return torch.randn(n, DIMS[name], generator=g)


def context_of(n=512):
    return R.context_of(n)
