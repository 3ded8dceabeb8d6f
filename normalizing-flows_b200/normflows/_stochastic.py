"""Native path of the stochastic layers and of HAIS (flows/stochastic.py, sampling/hais.py): csrc/nfb_stochastic.cu.

A native density is a flat DiagGaussian without temperature, a GaussianMixture, or a LinearInterpolation of native
densities; it reaches the kernels as at most four Gaussian-mixture terms with coefficients (`density_terms`).

Random numbers are torch's, so torch.manual_seed makes runs reproducible.  `draw` is the one place they are drawn; tests
replace it to replay stored draws.  Order: for a run of T transitions on `rows` rows of `dim` features, one
torch.randn(T, rows, dim) (the momenta of HMC, the proposal noise of MH), then one torch.rand(T, rows) (the uniforms of
the accept tests).  For T = 1 that is the reference layer's own order (randn_like(z), then rand_like); a chain of T > 1
draws all its normals first.  HAIS draws in chunks of at most `CHUNK_BYTES` of noise, so two RNG launches per chunk.

Under grad, HmcFn / MhFn run the no-grad launch as their forward (values bit-identical with and without grad).  Their
backward follows the reference's graph, in which grad log p is a constant and the accept mask has no gradient:
  z_out   the identity to z on both branches;
  log_det = log p(z) - log p(z_out), masked to the rows that moved: to z, z_out and the target's parameters through the
          target's own log_prob backward (nfb_gaussian_mixture_log_prob_backward, the diagonal-Gaussian table adjoint);
  HMC's log_step_size / log_mass: nfb_hmc_backward on the total cotangent of z_out (the accepted rows' leapfrog)."""
import ctypes as C

import torch

from . import _lib as L
from ._native import require_cuda_f32

CHUNK_BYTES = 256 << 20


def draw(rows, dim, transitions, device, dtype=torch.float32):
    """-> (noise [transitions, rows, dim] standard normal, uniforms [transitions, rows] on [0, 1)), in the dtype of the
    rows they move (float32 on the native path; the generic path draws as the reference does, in z.dtype)."""
    noise = torch.randn((transitions, rows, dim), dtype=dtype, device=device)
    return noise, torch.rand((transitions, rows), dtype=dtype, device=device)


def chunk_transitions(rows, dim, transitions):
    """Transitions per noise chunk of a chain."""
    return max(1, min(transitions, CHUNK_BYTES // max(1, rows * dim * 4)))


def density_terms(dist):
    """[(coefficient, DiagGaussian or GaussianMixture), ...] with log p = sum c log p_i, or None when `dist` is not a
    native density."""
    from .distributions.base import DiagGaussian, GaussianMixture
    from .distributions.linear_interpolation import LinearInterpolation
    if (isinstance(dist, DiagGaussian) and dist.temperature is None and dist.n_dim == 1) \
            or isinstance(dist, GaussianMixture):
        return [(1.0, dist)]
    if isinstance(dist, LinearInterpolation):
        if torch.is_tensor(dist.alpha) and dist.alpha.requires_grad:
            return None   # the kernels take alpha as a number: a trainable alpha keeps the reference's graph
        a, b = density_terms(dist.dist1), density_terms(dist.dist2)
        if a is None or b is None:
            return None
        alpha = float(dist.alpha)
        out = [(alpha * c, m) for c, m in a] + [((1 - alpha) * c, m) for c, m in b]
        return out if len(out) <= L.DENSITY_MAX_TERMS else None
    return None


def native_terms(dist, z):
    """density_terms(dist) when z is CUDA float32 [rows, features] and every term's tensors are float32 on z's device,
    else None."""
    if not (isinstance(z, torch.Tensor) and z.is_cuda and z.dtype == torch.float32 and z.dim() == 2):
        return None
    terms = density_terms(dist)
    if terms is None or any(t.dtype != torch.float32 or t.device != z.device
                            for _, m in terms for t in (m.loc, m.log_scale)):
        return None
    return terms


def term_params(terms):
    """The parameters of the terms' distributions (each once): the target's leaves the backward differentiates."""
    seen, out = set(), []
    for _, m in terms:
        for p in m.parameters():
            if id(p) not in seen:
                seen.add(id(p))
                out.append(p)
    return out


class Density:
    """The nfb_density_t of a list of terms for rows of `dim` features, and the tensors it points to."""

    def __init__(self, modules, dim, device):
        from .distributions.base import DiagGaussian
        self.desc = L.DensityDesc()
        self.desc.n_terms, self.desc.dim = len(modules), dim
        self.keep = []
        for i, m in enumerate(modules):
            if isinstance(m, DiagGaussian):
                if m.d != dim:
                    raise ValueError(f"DiagGaussian of {m.d} features as the target of {dim}-feature rows")
                k, ts = 1, (m.loc, m.log_scale, torch.zeros(1, device=device))
            else:
                if m.dim != dim:
                    raise ValueError(f"GaussianMixture of dim {m.dim} as the target of {dim}-feature rows")
                k, ts = m.n_modes, (m.loc, m.log_scale, m.weight_scores)
            ts = [require_cuda_f32(t.detach(), "target parameter") for t in ts]
            self.keep += ts
            self.desc.term[i] = L.DensityTerm(k, *(t.data_ptr() for t in ts))

    def ref(self):
        return C.byref(self.desc)


def _coef(rows_of_coefs, device):
    return torch.tensor(rows_of_coefs, dtype=torch.float32, device=device)


def _per_feature(t, dim):
    return t.detach().to(torch.float32).reshape(-1).expand(dim).contiguous()


def hmc_launch(density, coef, leapfrog, max_abs_grad, log_step, log_mass, noise, unif, z, log_w, accept):
    """nfb_hmc_chain over noise.shape[0] transitions; log_step / log_mass / coef are [transitions, ...].  (A draw hook
    may hand back strided tensors: the kernel reads dense rows.)"""
    coef, log_step, log_mass, noise, unif, z = (t.contiguous() for t in (coef, log_step, log_mass, noise, unif, z))
    z_out = torch.empty_like(z)
    with torch.cuda.device(z.device):
        L.check(L.lib().nfb_hmc_chain(density.ref(), z.shape[0], noise.shape[0], leapfrog, max_abs_grad, L.ptr(coef),
                                      L.ptr(log_step), L.ptr(log_mass), L.ptr(noise), L.ptr(unif), L.ptr(z),
                                      L.ptr(z_out), L.ptr(log_w), L.ptr(accept), L.stream_ptr()))
    return z_out


def clamp_value(max_abs_grad):
    """The reference clamps when max_abs_grad is truthy; the kernel reads 0 as "no clamp"."""
    return float(max_abs_grad) if max_abs_grad else 0.0


class HmcStep:
    """One HMC transition of a layer on a native target: its launch and what its backward needs."""

    def __init__(self, layer, terms, z, noise, unif):
        self.layer, self.terms = layer, terms
        rows, dim = z.shape
        self.density = Density([m for _, m in terms], dim, z.device)
        self.coef = _coef([[c for c, _ in terms]], z.device)
        self.log_step = _per_feature(layer.log_step_size, dim)
        self.log_mass = _per_feature(layer.log_mass, dim)
        self.noise, self.unif = noise.reshape(1, rows, dim).contiguous(), unif.reshape(1, rows).contiguous()
        self.mag = clamp_value(layer.max_abs_grad)

    def run(self, z):
        log_det = torch.zeros(z.shape[0], dtype=torch.float32, device=z.device)
        accept = torch.empty((1, z.shape[0]), dtype=torch.uint8, device=z.device)
        z_out = hmc_launch(self.density, self.coef, self.layer.steps, self.mag, self.log_step, self.log_mass,
                           self.noise, self.unif, z, log_det, accept)
        return z_out, log_det, accept[0]

    def param_grads(self, z, accept, g_z_out):
        rows, dim = z.shape
        g_ls = torch.empty(dim, dtype=torch.float32, device=z.device)
        g_lm = torch.empty_like(g_ls)
        lib = L.lib()
        ws = torch.empty(max(1, lib.nfb_hmc_backward_workspace_bytes(rows, dim)), dtype=torch.uint8, device=z.device)
        with torch.cuda.device(z.device):
            L.check(lib.nfb_hmc_backward(self.density.ref(), rows, self.layer.steps, self.mag, L.ptr(self.coef),
                                         L.ptr(self.log_step), L.ptr(self.log_mass), L.ptr(self.noise),
                                         L.ptr(z.contiguous()),
                                         L.ptr(accept), L.ptr(g_z_out), L.ptr(ws), ws.numel(), L.ptr(g_ls), L.ptr(g_lm),
                                         L.stream_ptr()))
        return g_ls, g_lm


def _check_versions(ctx, who):
    if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
        raise RuntimeError(f"{who} backward: a parameter was modified in place after the forward pass")


def _log_det_adjoint(target, tparams, z, z_out, moved, g_z_out, g_ld):
    """Cotangents of log_det = moved (log p(z) - log p(z_out)) and of z_out = (moved ? z' : z) with z' - z constant
    in z: -> (g_z, g_z_out_total, {parameter: gradient})."""
    G = torch.zeros_like(z) if g_z_out is None else g_z_out.contiguous()
    if g_ld is None:
        return G, G, {}
    g_eff = g_ld * moved.to(g_ld.dtype)
    with torch.enable_grad():
        z_ = z.detach().requires_grad_()
        zo_ = z_out.detach().requires_grad_()
        val = torch.sum(g_eff * (target.log_prob(z_) - target.log_prob(zo_)))
        want = [p for p in tparams if p.requires_grad]
        gs = torch.autograd.grad(val, [z_, zo_] + want, allow_unused=True)
    G = G + gs[1] if gs[1] is not None else G
    g_z = G + gs[0] if gs[0] is not None else G
    return g_z, G, {id(p): g for p, g in zip(want, gs[2:]) if g is not None}


class HmcFn(torch.autograd.Function):
    """(z_out, log_det) of one HMC transition on a native target (HmcStep.run, the no-grad launch) and the reference
    graph's adjoint.  Refuses to run the backward after an in-place change of a parameter."""

    @staticmethod
    def forward(ctx, step, z, log_step_size, log_mass, *tparams):
        z_out, log_det, accept = step.run(z)
        ctx.step, ctx.params = step, (log_step_size, log_mass) + tparams
        ctx.versions = [p._version for p in ctx.params]
        ctx.save_for_backward(z, z_out, accept)
        ctx.mark_non_differentiable(accept)
        return z_out, log_det

    @staticmethod
    def backward(ctx, g_z_out, g_ld):
        z, z_out, accept = ctx.saved_tensors
        step = ctx.step
        _check_versions(ctx, "HamiltonianMonteCarlo")
        tparams = ctx.params[2:]
        g_z, G, gmap = _log_det_adjoint(step.layer.target, tparams, z, z_out, accept, g_z_out, g_ld)
        g_ls = g_lm = None
        if ctx.needs_input_grad[2] or ctx.needs_input_grad[3]:
            g_ls, g_lm = step.param_grads(z, accept, G.contiguous())
            g_ls = g_ls.sum_to_size(step.layer.log_step_size.shape)
            g_lm = g_lm.sum_to_size(step.layer.log_mass.shape)
        return (None, g_z if ctx.needs_input_grad[1] else None,
                g_ls if ctx.needs_input_grad[2] else None, g_lm if ctx.needs_input_grad[3] else None,
                *[gmap.get(id(p)) if p.requires_grad else None for p in tparams])


class MhStep:
    """`steps` Metropolis-Hastings steps with a DiagGaussianProposal on a native target."""

    def __init__(self, layer, terms, z, noise, unif):
        self.layer, self.terms = layer, terms
        rows, dim = z.shape
        self.density = Density([m for _, m in terms], dim, z.device)
        self.coef = _coef([c for c, _ in terms], z.device)
        self.scale = _per_feature(layer.proposal.scale, dim)
        self.noise, self.unif = noise.contiguous(), unif.contiguous()

    def run(self, z):
        rows = z.shape[0]
        z = z.contiguous()
        z_out = torch.empty_like(z)
        log_det = torch.empty(rows, dtype=torch.float32, device=z.device)
        moved = torch.empty(rows, dtype=torch.uint8, device=z.device)
        with torch.cuda.device(z.device):
            L.check(L.lib().nfb_mh_chain(self.density.ref(), rows, self.noise.shape[0], L.ptr(self.coef),
                                         L.ptr(self.scale), L.ptr(self.noise), L.ptr(self.unif), L.ptr(z),
                                         L.ptr(z_out), L.ptr(log_det), L.ptr(moved), L.stream_ptr()))
        return z_out, log_det, moved


class MhFn(torch.autograd.Function):
    """(z_out, log_det) of MetropolisHastings on a native target (MhStep.run) and the reference graph's adjoint: the
    accepted steps' log p terms telescope to log p(z) - log p(z_out) on the rows that moved."""

    @staticmethod
    def forward(ctx, step, z, *tparams):
        z_out, log_det, moved = step.run(z)
        ctx.step, ctx.params = step, tparams
        ctx.versions = [p._version for p in tparams]
        ctx.save_for_backward(z, z_out, moved)
        return z_out, log_det

    @staticmethod
    def backward(ctx, g_z_out, g_ld):
        z, z_out, moved = ctx.saved_tensors
        _check_versions(ctx, "MetropolisHastings")
        g_z, _, gmap = _log_det_adjoint(ctx.step.layer.target, ctx.params, z, z_out, moved, g_z_out, g_ld)
        return (None, g_z if ctx.needs_input_grad[1] else None,
                *[gmap.get(id(p)) if p.requires_grad else None for p in ctx.params])


def hais_chain(hais, z, log_w):
    """HAIS.sample's layers as nfb_hmc_chain launches (one per noise chunk) -> the samples, log_w [rows] incremented in
    place; None (nothing drawn or done) when a layer's target is not native, or the layers differ in their list of
    densities, leapfrog steps or clamp."""
    layers = hais.layers
    terms = [native_terms(layer.target, z) for layer in layers]
    if any(t is None for t in terms):
        return None
    mods = [m for _, m in terms[0]]
    if any([m for _, m in t] != mods or len(t) != len(mods) for t in terms):
        return None
    rows, dim = z.shape
    density = Density(mods, dim, z.device)
    coef = _coef([[c for c, _ in t] for t in terms], z.device)
    log_step = torch.stack([_per_feature(layer.log_step_size, dim) for layer in layers])
    log_mass = torch.stack([_per_feature(layer.log_mass, dim) for layer in layers])
    leapfrog = {layer.steps for layer in layers}
    mags = {clamp_value(layer.max_abs_grad) for layer in layers}
    if len(leapfrog) != 1 or len(mags) != 1:
        return None
    leapfrog, mag = leapfrog.pop(), mags.pop()
    z = require_cuda_f32(z)
    per = chunk_transitions(rows, dim, len(layers))
    for t0 in range(0, len(layers), per):
        t1 = min(len(layers), t0 + per)
        noise, unif = draw(rows, dim, t1 - t0, z.device)
        z = hmc_launch(density, coef[t0:t1], leapfrog, mag, log_step[t0:t1], log_mass[t0:t1], noise, unif, z, log_w,
                       None)
    return z
