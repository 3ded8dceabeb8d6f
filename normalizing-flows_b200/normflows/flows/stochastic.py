"""Stochastic layers of stochastic normalizing flows (reference: flows/stochastic.py; Wu et al. 2020,
arXiv:2002.06707): the same constructors, parameters and semantics.

On a native target (a flat DiagGaussian, a GaussianMixture, or a LinearInterpolation of those; normflows/_stochastic.py)
fed CUDA float32 [rows, D] with D <= 64, a call is one launch of csrc/nfb_stochastic.cu, through HmcFn / MhFn under grad.
Any other target takes `_generic_transition` / `_generic_steps`: the reference's algorithm on the caller's tensors, with
grad log p by autograd (a user Target, TwoMoons, a torch.distributions object, a NormalizingFlow).  Both paths take
their random numbers from normflows._stochastic.draw (in z.dtype), except a MetropolisHastings whose proposal is not a
DiagGaussianProposal: that one calls its proposal and torch.rand step by step, as the reference does."""
import torch

from .. import _stochastic as S
from .base import Flow


class MetropolisHastings(Flow):
    """`steps` Metropolis-Hastings steps towards `target` with `proposal` (reference: flows/stochastic.py:7-48).
    log_det accumulates log p(z) - log p(z') over the accepted steps.  The native path takes a DiagGaussianProposal."""

    def __init__(self, target, proposal, steps):
        super().__init__()
        self.target = target
        self.proposal = proposal
        self.steps = steps

    def _sampling_differentiable(self, context=None):
        return True

    def forward(self, z):
        from ..distributions.mh_proposal import DiagGaussianProposal
        if type(self.proposal) is not DiagGaussianProposal:
            return self._generic_steps(z)
        noise, unif = S.draw(len(z), z.shape[1:].numel(), self.steps, z.device, z.dtype)
        terms = S.native_terms(self.target, z)
        if terms is None:
            return self._generic_steps(z, noise, unif)
        z = z.contiguous()   # the kernel reads dense rows (differentiable: a strided z gets its gradient back)
        step = S.MhStep(self, terms, z, noise, unif)
        tparams = S.term_params(terms)
        if torch.is_grad_enabled() and (z.requires_grad or any(p.requires_grad for p in tparams)):
            return S.MhFn.apply(step, z, *tparams)
        z_out, log_det, _ = step.run(z)
        return z_out, log_det

    def _generic_steps(self, z, noise=None, unif=None):
        """The reference's loop (flows/stochastic.py:23-45); with the draws given, a DiagGaussianProposal's step s
        proposes noise[s] scale + z and tests against unif[s]."""
        num_samples = len(z)
        log_det = torch.zeros(num_samples, dtype=z.dtype, device=z.device)
        log_p = self.target.log_prob(z)
        for i in range(self.steps):
            if noise is None:
                z_, log_p_diff = self.proposal(z)
            else:
                z_ = noise[i].reshape(z.shape) * self.proposal.scale + z
                log_p_diff = torch.zeros(num_samples, dtype=z.dtype, device=z.device)
            log_p_ = self.target.log_prob(z_)
            w = torch.rand(num_samples, dtype=z.dtype, device=z.device) if unif is None else unif[i]
            log_w_accept = log_p_ - log_p + log_p_diff
            w_accept = torch.clamp(torch.exp(log_w_accept), max=1)
            accept = w <= w_accept
            z = torch.where(accept.unsqueeze(1), z_, z)
            log_det_ = log_p - log_p_
            log_det = torch.where(accept, log_det + log_det_, log_det)
            log_p = torch.where(accept, log_p_, log_p)
        return z, log_det

    def inverse(self, z):
        return self.forward(z)


class HamiltonianMonteCarlo(Flow):
    """One HMC transition with `steps` leapfrog steps towards `target` (reference: flows/stochastic.py:51-115):
    momentum p = n exp(log_mass / 2), grad log p detached and clamped to +-max_abs_grad when max_abs_grad is truthy,
    accept when u < exp(delta H), log_det = log p(z) - log p(z_out) (0 on rejected rows).  Parameters log_step_size and
    log_mass, shape (dim)."""

    def __init__(self, target, steps, log_step_size, log_mass, max_abs_grad=None):
        super().__init__()
        self.target = target
        self.steps = steps
        self.register_parameter("log_step_size", torch.nn.Parameter(log_step_size))
        self.register_parameter("log_mass", torch.nn.Parameter(log_mass))
        self.max_abs_grad = max_abs_grad

    def _sampling_differentiable(self, context=None):
        return True

    def forward(self, z):
        noise, unif = S.draw(len(z), z.shape[1:].numel(), 1, z.device, z.dtype)
        return self._transition(z, noise[0], unif[0])

    def _transition(self, z, noise, unif):
        """The transition with momentum noise [rows, D] and uniforms [rows] given."""
        terms = S.native_terms(self.target, z)
        if terms is None:
            return self._generic_transition(z, noise.reshape(z.shape), unif)
        z = z.contiguous()   # the kernels read dense rows (differentiable: a strided z gets its gradient back)
        step = S.HmcStep(self, terms, z, noise, unif)
        tparams = S.term_params(terms)
        if torch.is_grad_enabled() and (z.requires_grad or self.log_step_size.requires_grad
                                        or self.log_mass.requires_grad or any(p.requires_grad for p in tparams)):
            return S.HmcFn.apply(step, z, self.log_step_size, self.log_mass, *tparams)
        z_out, log_det, _ = step.run(z)
        return z_out, log_det

    def _generic_transition(self, z, noise, unif):
        """The reference's forward (flows/stochastic.py:73-96) with its draws given."""
        p = noise * torch.exp(0.5 * self.log_mass)
        z_new = z.clone()
        p_new = p.clone()
        step_size = torch.exp(self.log_step_size)
        for i in range(self.steps):
            p_half = p_new - (step_size / 2.0) * -self.gradlogP(z_new)
            z_new = z_new + step_size * (p_half / torch.exp(self.log_mass))
            p_new = p_half - (step_size / 2.0) * -self.gradlogP(z_new)
        probabilities = torch.exp(
            self.target.log_prob(z_new)
            - self.target.log_prob(z)
            - 0.5 * torch.sum(p_new ** 2 / torch.exp(self.log_mass), 1)
            + 0.5 * torch.sum(p ** 2 / torch.exp(self.log_mass), 1)
        )
        mask = unif < probabilities
        z_out = torch.where(mask.unsqueeze(1), z_new, z)
        return z_out, self.target.log_prob(z) - self.target.log_prob(z_out)

    def inverse(self, z):
        return self.forward(z)

    def gradlogP(self, z):
        z_ = z.detach().requires_grad_()
        with torch.enable_grad():
            logp = self.target.log_prob(z_)
            grad = torch.autograd.grad(logp, z_, grad_outputs=torch.ones_like(logp))[0]
        if self.max_abs_grad:
            grad = torch.clamp(grad, max=self.max_abs_grad, min=-self.max_abs_grad)
        return grad
