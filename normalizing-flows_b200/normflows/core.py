"""NormalizingFlow driver (reference: normflows/core.py:9-213).

Same public surface: forward, forward_and_log_det, inverse, inverse_and_log_det, forward_kld, sample,
log_prob, save, load.  Where the reference loops over layers in Python and accumulates `log_q` with a
tiny kernel per layer (core.py:96-102), this class hands the whole stack to one `nfb_flow` so that
log-det accumulation happens in kernel epilogues and adjacent layers fuse
([LULinearPermute + spline block] -> one tensor-core kernel).  If any layer is not a `NativeFlow`, it
falls back to the reference's per-layer loop over whatever the layers implement."""
import torch
from torch import nn

from . import _lib as L
from ._native import FlowHandle
from .distributions.base import DiagGaussian
from .flows.base import NativeFlow


class NormalizingFlow(nn.Module):
    def __init__(self, q0, flows, p=None):
        super().__init__()
        self.q0 = q0
        self.flows = nn.ModuleList(flows)
        self.p = p

    # -- native stack -------------------------------------------------------------------------
    def _stack(self):
        if not all(isinstance(f, NativeFlow) for f in self.flows):
            return None
        h = self.__dict__.get("_nfb_stack")
        base = self.q0 if isinstance(self.q0, DiagGaussian) and self.q0.temperature is None \
            and self.q0.n_dim == 1 else None
        layers = list(self.flows)
        if (h is None or h.layers != layers or h.base is not base
                or h.use_tc != NativeFlow.use_tensor_cores):
            for f in layers:  # data-dependent inits must have happened before packing
                pass
            h = FlowHandle(layers, base, NativeFlow.use_tensor_cores)
            self.__dict__["_nfb_stack"] = h
        return h

    def repack(self):
        """Rebuild the packed device image of the weights on the next call.  Needed only after an out-of-band
        `.data` mutation (EMA swap, clipping): optimizer steps, load_state_dict, train()/eval() and ordinary
        in-place updates are picked up automatically (see _native.py)."""
        from ._native import invalidate_packed_weights
        invalidate_packed_weights()

    def train(self, mode=True):
        if mode != self.training:
            self.repack()
        return super().train(mode)

    def load_state_dict(self, *args, **kwargs):
        out = super().load_state_dict(*args, **kwargs)
        self.repack()
        return out

    def _needs_eager_init(self):
        from .flows.affine import ActNorm
        return any(isinstance(f, ActNorm) and not f._done() for f in self.flows)

    def _run_pending_inits(self, x, inverse):
        """Data-dependent initialisation (ActNorm, flows/normalization.py:19-39) happens inside the reference's
        first pass, transparently to training.  Here: if any layer still waits for it, walk the layers once
        under no_grad (each ActNorm sees exactly the input the reference would give it), then take the normal
        path -- fused stack, or DensityFn when gradients are wanted."""
        if not self._needs_eager_init():
            return
        with torch.no_grad():
            z = x.detach()
            for flow in (reversed(self.flows) if inverse else self.flows):
                z, _ = flow.inverse(z) if inverse else flow(z)

    # -- reference API ------------------------------------------------------------------------
    def forward(self, z):
        z, _ = self.forward_and_log_det(z)
        return z

    def forward_and_log_det(self, z):
        h = self._stack()
        self._run_pending_inits(z, inverse=False)
        if h is not None and z.dim() == 2:
            return h.transform(L.NFB_FORWARD, z)
        log_det = torch.zeros(len(z), device=z.device)
        for flow in self.flows:
            z, ld = flow(z)
            log_det = log_det + ld
        return z, log_det

    def inverse(self, x):
        z, _ = self.inverse_and_log_det(x)
        return z

    def inverse_and_log_det(self, x):
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and x.dim() == 2:
            return h.transform(L.NFB_INVERSE, x)
        log_det = torch.zeros(len(x), device=x.device)
        for i in range(len(self.flows) - 1, -1, -1):
            x, ld = self.flows[i].inverse(x)
            log_det = log_det + ld
        return x, log_det

    def _wants_grad(self, x):
        return torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))

    def log_prob(self, x):
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and h.base is not None and x.dim() == 2:
            if self._wants_grad(x):  # forward on the CUDA kernels, backward via _autograd (interim, SURVEY 8f-1)
                from ._autograd import DensityFn
                return DensityFn.apply(self, x, *self.parameters())
            return h.log_prob(x)
        z, log_q = self.inverse_and_log_det(x)
        return log_q + self.q0.log_prob(z)

    def forward_kld(self, x):
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and h.base is not None and x.dim() == 2 and not self._wants_grad(x):
            return h.forward_kld(x)
        return -torch.mean(self.log_prob(x))

    def sample(self, num_samples=1):
        z, log_q = self.q0(num_samples)
        x, log_det = self.forward_and_log_det(z)
        return x, log_q - log_det

    def _no_sampling_grad(self, what):
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError(
                f"{what}: gradients through the sampling direction are not on the CUDA path yet "
                "(evaluate under torch.no_grad(); forward_kld / log_prob are differentiable)")

    def reverse_kld(self, num_samples=1, beta=1.0, score_fn=True):
        """core.py:104-131.  z ~ q0 pushed through every layer's `.forward` (one persistent launch for coupling
        stacks), log_q = log q0(z0) - sum log_det; `score_fn=False` re-evaluates log_q by the density pass of the
        drawn samples (the reference does the same with parameter gradients switched off)."""
        self._no_sampling_grad("reverse_kld")
        z, log_q = self.sample(num_samples)
        if not score_fn:
            log_q = self.log_prob(z)
        log_p = self.p.log_prob(z)
        return torch.mean(log_q) - beta * torch.mean(log_p)

    def reverse_alpha_div(self, num_samples=1, alpha=1, dreg=False):
        """core.py:133-165 (value; see reverse_kld for the gradient caveat)."""
        import numpy as np
        self._no_sampling_grad("reverse_alpha_div")
        z, log_q = self.sample(num_samples)
        log_p = self.p.log_prob(z)
        if dreg:
            w_const = torch.exp(log_p - log_q).detach()
            log_q = self.log_prob(z)
            w = torch.exp(log_p - log_q)
            w_alpha = w_const ** alpha
            w_alpha = w_alpha / torch.mean(w_alpha)
            weights = (1 - alpha) * w_alpha + alpha * w_alpha ** 2
            return -alpha * torch.mean(weights * torch.log(w))
        return np.sign(alpha - 1) * torch.logsumexp(alpha * (log_p - log_q), 0)

    def save(self, path):
        torch.save(self.state_dict(), path)

    def load(self, path):
        self.load_state_dict(torch.load(path))

    # -- host-buffer entry points (C ABI `_host` functions) -------------------------------------
    def forward_kld_host(self, x_host, device=None):
        h = self._stack()
        if h is None or h.base is None:
            raise NotImplementedError("forward_kld_host needs an all-native stack with a DiagGaussian base")
        device = torch.device(device) if device is not None else next(self.parameters()).device
        return h.forward_kld_host(x_host, device)

    def log_prob_host(self, x_host, device=None):
        h = self._stack()
        if h is None or h.base is None:
            raise NotImplementedError("log_prob_host needs an all-native stack with a DiagGaussian base")
        device = torch.device(device) if device is not None else next(self.parameters()).device
        return h.log_prob_host(x_host, device)


class ConditionalNormalizingFlow(NormalizingFlow):
    """Conditional flow: the context goes to the base distribution and to every layer (reference: core.py:216-366).
    Context-conditioned spline layers run outside the fused block (their conditioners take the context through GLU
    gates): stand-alone tensor-core GEMMs + the HBM-bound spline kernel, layer by layer like the reference's loop."""

    def forward(self, z, context=None):
        for flow in self.flows:
            z, _ = flow(z, context=context)
        return z

    def forward_and_log_det(self, z, context=None):
        log_det = torch.zeros(len(z), device=z.device)
        for flow in self.flows:
            z, log_d = flow(z, context=context)
            log_det = log_det + log_d
        return z, log_det

    def inverse(self, x, context=None):
        for i in range(len(self.flows) - 1, -1, -1):
            x, _ = self.flows[i].inverse(x, context=context)
        return x

    def inverse_and_log_det(self, x, context=None):
        log_det = torch.zeros(len(x), device=x.device)
        for i in range(len(self.flows) - 1, -1, -1):
            x, log_d = self.flows[i].inverse(x, context=context)
            log_det = log_det + log_d
        return x, log_det

    def sample(self, num_samples=1, context=None):
        z, log_q = self.q0(num_samples, context=context)
        for flow in self.flows:
            z, log_det = flow(z, context=context)
            log_q = log_q - log_det
        return z, log_q

    def log_prob(self, x, context=None):
        z, log_q = self.inverse_and_log_det(x, context=context)
        return log_q + self.q0.log_prob(z, context=context)

    def forward_kld(self, x, context=None):
        return -torch.mean(self.log_prob(x, context=context))

    def reverse_kld(self, num_samples=1, context=None, beta=1.0, score_fn=True):
        self._no_sampling_grad("reverse_kld")
        z, log_q = self.sample(num_samples, context=context)
        if not score_fn:
            log_q = self.log_prob(z, context=context)
        log_p = self.p.log_prob(z, context=context)
        return torch.mean(log_q) - beta * torch.mean(log_p)


class ClassCondFlow(nn.Module):
    """Class-conditional flow: the class goes to the base distribution only (reference: core.py:368-452).  The layer
    stack itself runs through the same fused launch as NormalizingFlow (one persistent kernel for spline stacks)."""

    def __init__(self, q0, flows):
        super().__init__()
        self.q0 = q0
        self.flows = nn.ModuleList(flows)
        self._inner = None

    def _flow(self):
        # an inner NormalizingFlow that shares the layer modules (no base: only its transform paths are used)
        inner = self.__dict__.get("_nfb_inner")
        if inner is None or list(inner.flows) != list(self.flows):
            inner = NormalizingFlow(None, list(self.flows))
            self.__dict__["_nfb_inner"] = inner
        return inner

    def log_prob(self, x, y):
        z, log_q = self._flow().inverse_and_log_det(x)
        return log_q + self.q0.log_prob(z, y)

    def forward_kld(self, x, y):
        return -torch.mean(self.log_prob(x, y))

    def sample(self, num_samples=1, y=None):
        z, log_q = self.q0(num_samples, y)
        x, log_det = self._flow().forward_and_log_det(z)
        return x, log_q - log_det

    def save(self, path):
        torch.save(self.state_dict(), path)

    def load(self, path):
        self.load_state_dict(torch.load(path))


class MultiscaleFlow(nn.Module):
    """Multiscale (Glow) driver (reference: core.py:455-653)."""

    def __init__(self, q0, flows, merges, transform=None, class_cond=True):
        super().__init__()
        self.q0 = nn.ModuleList(q0)
        self.num_levels = len(self.q0)
        self.flows = nn.ModuleList([nn.ModuleList(f) for f in flows])
        self.merges = nn.ModuleList(merges)
        self.transform = transform
        self.class_cond = class_cond

    def log_prob(self, x, y=None):
        """core.py:588-616: levels last-to-first; each flow's `.inverse`; channel split between levels."""
        from .flows.glow import split_channels
        log_q = 0
        z = x
        if self.transform is not None:  # core.py:600-602
            z, log_det = self.transform.inverse(z)
            log_q = log_q + log_det
        for i in range(len(self.q0) - 1, -1, -1):
            for j in range(len(self.flows[i]) - 1, -1, -1):
                z, log_det = self.flows[i][j].inverse(z)
                log_q = log_q + log_det
            if i > 0:
                z, z_ = split_channels(z, getattr(self.merges[i - 1], "mode", "channel"))
            else:
                z_ = z
            log_q = log_q + (self.q0[i].log_prob(z_, y) if self.class_cond else self.q0[i].log_prob(z_))
        return log_q

    def forward_kld(self, x, y=None):
        return -torch.mean(self.log_prob(x, y))

    def forward(self, x, y=None):
        return -self.log_prob(x, y)

    def forward_and_log_det(self, z):
        """core.py:504-525: list of per-level latents -> x; levels first-to-last, each flow's `.forward`."""
        log_det = 0
        z_ = None
        for i in range(len(self.q0)):
            if i == 0:
                z_ = z[0]
            else:
                z_, ld = self.merges[i - 1]([z_, z[i]])
                log_det = log_det + ld
            for flow in self.flows[i]:
                z_, ld = flow(z_)
                log_det = log_det + ld
        if self.transform is not None:  # core.py:522-524
            z_, ld = self.transform(z_)
            log_det = log_det + ld
        return z_, log_det

    def inverse_and_log_det(self, x):
        """core.py:527-551: x -> list of per-level latents."""
        log_det = 0
        if self.transform is not None:  # core.py:536-538
            x, ld = self.transform.inverse(x)
            log_det = log_det + ld
        z = [None] * len(self.q0)
        for i in range(len(self.q0) - 1, -1, -1):
            for flow in reversed(self.flows[i]):
                x, ld = flow.inverse(x)
                log_det = log_det + ld
            if i == 0:
                z[i] = x
            else:
                [x, z[i]], ld = self.merges[i - 1].inverse(x)
                log_det = log_det + ld
        return z, log_det

    def sample(self, num_samples=1, y=None, temperature=None):
        """core.py:553-586: draw every level's latent from its base, push it through the stack."""
        if temperature is not None:
            self.set_temperature(temperature)
        log_q, z = None, None
        for i in range(len(self.q0)):
            z_, log_q_ = self.q0[i](num_samples, y) if self.class_cond else self.q0[i](num_samples)
            if i == 0:
                log_q, z = log_q_, z_
            else:
                log_q = log_q + log_q_
                z, ld = self.merges[i - 1]([z, z_])
                log_q = log_q - ld
            for flow in self.flows[i]:
                z, ld = flow(z)
                log_q = log_q - ld
        if self.transform is not None:  # core.py:577-579
            z, ld = self.transform(z)
            log_q = log_q - ld
        if temperature is not None:
            self.reset_temperature()
        return z, log_q

    def set_temperature(self, temperature):
        """core.py:634-647."""
        for q0 in self.q0:
            if hasattr(q0, "temperature"):
                q0.temperature = temperature
            else:
                raise NotImplementedError("One base function does not support temperature annealed sampling")

    def reset_temperature(self):
        self.set_temperature(None)

    def save(self, path):
        torch.save(self.state_dict(), path)

    def load(self, path):
        self.load_state_dict(torch.load(path))
