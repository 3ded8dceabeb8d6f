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
from ._image_autograd import wants_grad
from ._native import FlowHandle
from .distributions.base import ConditionalDiagGaussian, DiagGaussian, GaussianMixture, UniformGaussian
from .distributions.encoder import Dirac
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
        base = self.q0 if (isinstance(self.q0, DiagGaussian) and self.q0.temperature is None
                           and self.q0.n_dim == 1) or isinstance(self.q0, GaussianMixture) else None
        layers = list(self.flows)
        if (h is None or h.layers != layers or h.base is not base
                or h.use_tc != NativeFlow.use_tensor_cores):
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
            if wants_grad(self.flows, z):
                if not self._stack_sampling_backward():   # h.transform would return a result detached from the graph
                    raise NotImplementedError(_no_sampling_grad_message("forward_and_log_det") + ")")
                from ._standalone import stack_sampling   # one native backward
                return stack_sampling(h, self.flows, z, list(self.flows.parameters()))
            return h.transform(L.NFB_FORWARD, z)
        log_det = torch.zeros(len(z), device=z.device)
        for flow in self.flows:
            z, ld = flow(z)
            log_det = log_det + ld
        return z, log_det

    def inverse(self, x):
        z, _ = self.inverse_and_log_det(x)
        return z

    def _require_inverse(self):
        """Planar (tanh) and Radial layers have no density direction: raise, like the reference, before any launch."""
        for f in self.flows:
            if getattr(f, "_no_inverse", False):
                raise NotImplementedError("This flow has no algebraic inverse.")

    def inverse_and_log_det(self, x):
        self._require_inverse()
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and x.dim() == 2:
            if self._one_sampling_family() == "affine" and wants_grad(self.flows, x):   # native density backward
                from ._standalone import stack_sampling
                return stack_sampling(h, self.flows, x, list(self.flows.parameters()), L.NFB_INVERSE)
            return h.transform(L.NFB_INVERSE, x)
        log_det = torch.zeros(len(x), device=x.device)
        for i in range(len(self.flows) - 1, -1, -1):
            x, ld = self.flows[i].inverse(x)
            log_det = log_det + ld
        return x, log_det

    def log_prob(self, x):
        self._require_inverse()
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and h.base is not None and x.dim() == 2:
            if wants_grad(self, x):  # forward on the CUDA kernels, backward via _autograd (interim, SURVEY 8f-1)
                from ._autograd import DensityFn
                return DensityFn.apply(self, x, *self.parameters())
            return h.log_prob(x)
        z, log_q = self.inverse_and_log_det(x)
        return log_q + self.q0.log_prob(z)

    def forward_kld(self, x):
        self._require_inverse()
        h = self._stack()
        self._run_pending_inits(x, inverse=True)
        if h is not None and h.base is not None and x.dim() == 2 and not wants_grad(self, x):
            return h.forward_kld(x)
        return -torch.mean(self.log_prob(x))

    def sample(self, num_samples=1):
        z, log_q = self.q0(num_samples)
        x, log_det = self.forward_and_log_det(z)
        return x, log_q - log_det

    def _takes_layer_loop(self):
        return self._stack() is None

    def _one_sampling_family(self):
        """Every layer is in the affine family (MaskedAffineFlow, AffineConstFlow / ActNorm, AffineCouplingBlock,
        Permute), or every layer in the planar family (Planar, Radial): the all-native stack's sampling direction has a
        native backward (nfb_flow_sampling_backward); returns that family's name ("affine" / "planar"), else None.  Mixes
        of the two families do not."""
        fams = {f._sampling_family() if isinstance(f, NativeFlow) else None for f in self.flows}
        return fams.pop() if len(fams) == 1 else None

    def _coupled_spline_stack(self):
        """Every layer a CoupledRationalQuadraticSpline without a context and with 8 bins, or an LULinearPermute: the
        all-native stack's sampling direction has a native backward (nfb_flow_sampling_backward).  A stack-level rule:
        LULinearPermute on its own, or between layers outside the native stack, stays without one."""
        from .flows.mixing import LULinearPermute
        from .flows.neural_spline import CoupledRationalQuadraticSpline
        return len(self.flows) > 0 and all(
            type(f) is LULinearPermute or (type(f) is CoupledRationalQuadraticSpline and f.num_context_channels is None
                                            and f.num_bins == 8) for f in self.flows)

    def _stack_sampling_backward(self):
        """The all-native stack's sampling direction has a native backward: all-affine, all-planar, or coupled splines
        with LU layers."""
        return self._one_sampling_family() is not None or self._coupled_spline_stack()

    def _flows_sampling_differentiable(self, context=None, rows=True):
        """The sampling direction is differentiable where it runs.  On the all-native stack (rows: z is [rows, features],
        so forward_and_log_det takes the stack) when the stack has a native backward (_stack_sampling_backward).  In the
        layer loop (a stack with a layer that is not native, a conditional flow, or an all-one-family stack fed z of
        another shape) when every layer's is (`_sampling_differentiable`: the stand-alone spline layers, the coupled
        spline layer, the affine and planar families; not LULinearPermute)."""
        if rows and not self._takes_layer_loop():
            return self._stack_sampling_backward()
        return ((self._takes_layer_loop() or self._one_sampling_family() is not None)
                and all(hasattr(f, "_sampling_differentiable") and f._sampling_differentiable(context)
                        for f in self.flows))

    def _no_sampling_grad(self, what, context=None):
        """Gradients through the sampling direction exist when the layers' are (_flows_sampling_differentiable) and the
        base's draw is reparameterised (UniformGaussian, DiagGaussian, ConditionalDiagGaussian, GaussianMixture).
        Otherwise, under grad, raise."""
        if not (torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())):
            return
        if (isinstance(self.q0, (UniformGaussian, DiagGaussian, ConditionalDiagGaussian, GaussianMixture))
                and self._flows_sampling_differentiable(context, rows=getattr(self.q0, "n_dim", 1) == 1)):
            return
        raise NotImplementedError(_no_sampling_grad_message(what) + "; forward_kld / log_prob are differentiable)")

    def _log_q_no_param_grad(self, z, **context):
        """log q(z) by the density pass with the parameters' requires_grad switched off and back on, as the reference
        does (core.py:121-129, 149-157, 356-364): under grad, z's gradient flows, the parameters' does not."""
        from .utils import set_requires_grad
        set_requires_grad(self, False)
        log_q = self.log_prob(z, **context)
        set_requires_grad(self, True)
        return log_q

    def reverse_kld(self, num_samples=1, beta=1.0, score_fn=True):
        """core.py:104-131.  z ~ q0 pushed through every layer's `.forward` (one persistent launch for coupling
        stacks), log_q = log q0(z0) - sum log_det; `score_fn=False` re-evaluates log_q by the density pass of the
        drawn samples with parameter gradients switched off, like the reference.  Differentiable for the stacks
        _no_sampling_grad admits (the stand-alone spline layers, the affine or the planar family, coupled spline + LU
        stacks, on a reparameterised base)."""
        self._no_sampling_grad("reverse_kld")
        z, log_q = self.sample(num_samples)
        if not score_fn:
            log_q = self._log_q_no_param_grad(z)
        log_p = self.p.log_prob(z)
        return torch.mean(log_q) - beta * torch.mean(log_p)

    def reverse_alpha_div(self, num_samples=1, alpha=1, dreg=False):
        """core.py:133-165 (differentiable for the stacks reverse_kld is)."""
        import numpy as np
        self._no_sampling_grad("reverse_alpha_div")
        z, log_q = self.sample(num_samples)
        log_p = self.p.log_prob(z)
        if dreg:
            w_const = torch.exp(log_p - log_q).detach()
            log_q = self._log_q_no_param_grad(z)
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
            raise NotImplementedError("forward_kld_host needs an all-native stack with a DiagGaussian or GaussianMixture base")
        device = torch.device(device) if device is not None else next(self.parameters()).device
        return h.forward_kld_host(x_host, device)

    def log_prob_host(self, x_host, device=None):
        h = self._stack()
        if h is None or h.base is None:
            raise NotImplementedError("log_prob_host needs an all-native stack with a DiagGaussian or GaussianMixture base")
        device = torch.device(device) if device is not None else next(self.parameters()).device
        return h.log_prob_host(x_host, device)


def _no_sampling_grad_message(what):
    return (f"{what}: gradients through the sampling direction are not on the CUDA path yet "
            "(evaluate under torch.no_grad()")


def _inner_flow(owner):
    """A NormalizingFlow without a base that shares `owner.flows`' layer modules, for drivers that push samples through
    the layers (ClassCondFlow, NormalizingFlowVAE): its stack handle, data-dependent initialisation and sampling-direction
    backward are NormalizingFlow's own."""
    inner = owner.__dict__.get("_nfb_inner")
    if inner is None or list(inner.flows) != list(owner.flows):
        inner = NormalizingFlow(None, list(owner.flows))
        owner.__dict__["_nfb_inner"] = inner
    return inner


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

    def _takes_layer_loop(self):
        return True   # every call above walks the layers

    def reverse_kld(self, num_samples=1, context=None, beta=1.0, score_fn=True):
        """core.py:337-366; differentiable when every layer's sampling direction is (see NormalizingFlow)."""
        self._no_sampling_grad("reverse_kld", context)
        z, log_q = self.sample(num_samples, context=context)
        if not score_fn:
            log_q = self._log_q_no_param_grad(z, context=context)
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
        return _inner_flow(self)

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


class NormalizingFlowVAE(nn.Module):
    """VAE whose approximate posterior is an encoder q0(z | x) followed by flows (reference: core.py:656-700).

    `forward(x, num_samples)` returns z [B, S, d], log_q [B, S] and log_p [B, S]; row b S + s of the flattened samples
    belongs to x[b].  The encoder's draw, its log-density and the decoder's likelihood are kernels with a native
    backward (distributions/encoder.py, distributions/decoder.py); the flows go through one stack, as in
    NormalizingFlow.forward_and_log_det: one native backward for an all-planar, all-affine or coupled-spline / LU list,
    the layer loop otherwise.  Under grad, flows without a differentiable sampling direction (autoregressive splines,
    MAF, mixed families in a stack; LU in a layer loop) raise instead of being silently detached.  `prior` is used as given (a torch distribution stays torch)."""

    def __init__(self, prior, q0=Dirac(), flows=None, decoder=None):
        super().__init__()
        self.prior = prior
        self.decoder = decoder
        self.flows = nn.ModuleList(flows)
        self.q0 = q0

    def _flows_forward(self, z):
        if len(self.flows) == 0:
            return z, torch.zeros(len(z), device=z.device)
        inner = _inner_flow(self)
        if wants_grad(self.flows, z) and not inner._flows_sampling_differentiable(rows=z.dim() == 2):
            names = "+".join(sorted({type(f).__name__ for f in self.flows}))
            raise NotImplementedError(_no_sampling_grad_message(f"NormalizingFlowVAE with {names} flows") + ")")
        return inner.forward_and_log_det(z)

    def forward(self, x, num_samples=1):
        z, log_q = self.q0(x, num_samples=num_samples)
        z = z.reshape(-1, *z.size()[2:])
        log_q = log_q.reshape(-1, *log_q.size()[2:])
        z, log_det = self._flows_forward(z)
        log_q = log_q - log_det
        log_p = self.prior.log_prob(z)
        if self.decoder is not None:
            log_p = log_p + self.decoder.log_prob(x, z)
        z = z.view(-1, num_samples, *z.size()[1:])
        log_q = log_q.view(-1, num_samples, *log_q.size()[1:])
        log_p = log_p.view(-1, num_samples, *log_p.size()[1:])
        return z, log_q, log_p
