"""Hamiltonian annealed importance sampling (reference: sampling/hais.py)."""
import torch

from .. import _stochastic as S
from .. import distributions
from .. import flows


class HAIS:
    """HAIS from `prior` to `target` along the schedule `betas` (1 = beta_0 > ... > beta_n = 0): the same layers as the
    reference, HamiltonianMonteCarlo(LinearInterpolation(target, prior, betas[i]), num_leapfrog, log(step_size),
    log_mass) for i = n - 1 ... 1, and the same log-weight bookkeeping.

    When every layer's density is native (prior and target each a flat DiagGaussian or a GaussianMixture) and no
    gradient is wanted (torch.no_grad(), or the layers' parameters frozen), `sample` runs the whole chain in
    nfb_hmc_chain: one launch per noise chunk (normflows/_stochastic.py).  Otherwise it walks the layers, each a launch
    with its native backward on native densities, the reference's algorithm on others.  Both take the same draws, so
    they give the same samples and weights."""

    def __init__(self, betas, prior, target, num_leapfrog, step_size, log_mass):
        self.prior = prior
        self.target = target
        self.layers = []
        n = betas.shape[0] - 1
        for i in range(n - 1, 0, -1):
            intermediate_target = distributions.LinearInterpolation(self.target, self.prior, betas[i])
            self.layers += [flows.HamiltonianMonteCarlo(intermediate_target, num_leapfrog, torch.log(step_size),
                                                        log_mass)]

    def _wants_grad(self, *tensors):
        return torch.is_grad_enabled() and (any(t.requires_grad for t in tensors)
                                            or any(p.requires_grad for f in self.layers for p in f.parameters()))

    def sample(self, num_samples):
        """-> (samples, log weights) of `num_samples` HAIS runs."""
        samples, log_weights = self.prior.forward(num_samples)
        log_weights = -log_weights
        chained = None
        if self.layers and not self._wants_grad(samples, log_weights):
            log_weights = log_weights.contiguous()
            chained = S.hais_chain(self, samples, log_weights)
        if chained is not None:
            samples = chained
        elif self.layers:
            rows, dim = len(samples), samples.shape[1:].numel()
            per = S.chunk_transitions(rows, dim, len(self.layers))
            for t0 in range(0, len(self.layers), per):
                t1 = min(len(self.layers), t0 + per)
                noise, unif = S.draw(rows, dim, t1 - t0, samples.device, samples.dtype)
                for t in range(t0, t1):
                    samples, log_weights_addition = self.layers[t]._transition(samples, noise[t - t0], unif[t - t0])
                    log_weights += log_weights_addition
        log_weights += self.target.log_prob(samples)
        return samples, log_weights
