"""Invertible residual flow (reference: normflows/flows/residual.py:12-430, after rtqichen/residual-flows).

`Residual(net)` wraps an `iResBlock`: y = x + g(x) with a Lipschitz-constrained `g` (nets.LipschitzMLP), and
log|det(I + dg/dx)| from
  * the exact 2 x 2 Jacobian for 2-D inputs in eval mode or with brute_force=True (:148-161), or
  * the (Russian-roulette) power series sum_k (-1)^(k+1)/k c_k tr(J^k) with Hutchinson's trace estimator (:163-217,
    :355-379); in training mode with neumann_grad the reference returns the Neumann-series surrogate (:368-379), and so
    does this class.
Everything numerical runs in libnfb200: g, its Jacobian-vector products (forward mode: 2 tangents for the exact path)
and its vector-Jacobian products (reverse mode: one per power-series term) are tensor-core GEMMs (csrc/nfb_gemm_tc.cu)
around the element-wise kernels of csrc/nfb_residual.cu.  Host side only draws the random truncation n (numpy, like
the reference) and the probe vector (torch.randn_like), both injectable for exact parity tests.
Training (the density direction under autograd, examples/residual.ipynb) goes through `ResidualBlockFn`: its forward
is the value path below, unchanged; its backward is ONE call of nfb_lipschitz_mlp_dual_backward, which recomputes g
pushed forward with the estimator's tangents and runs the adjoint of that dual network (csrc/nfb_residual.cu).  The
sampling direction (`Residual.forward`: the fixed-point inverse) stays value-only."""
import ctypes as C
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib as L
from .._image_autograd import wants_grad
from .._native import linear, linear_t, mul_rows, require_cuda_f32, rowdot, swish
from ..nets.lipschitz import InducedNormLinear, Swish
from .base import Flow


class Residual(Flow):
    def __init__(self, net, reverse=True, reduce_memory=True, geom_p=0.5, lamb=2.0, n_power_series=None,
                 exact_trace=False, brute_force=False, n_samples=1, n_exact_terms=2, n_dist="geometric"):
        super().__init__()
        self.reverse = reverse
        self.iresblock = iResBlock(net, n_samples=n_samples, n_exact_terms=n_exact_terms, neumann_grad=reduce_memory,
                                   grad_in_forward=reduce_memory, exact_trace=exact_trace, geom_p=geom_p, lamb=lamb,
                                   n_power_series=n_power_series, brute_force=brute_force, n_dist=n_dist)

    def forward(self, z):
        if self.reverse:
            z, log_det = self.iresblock.inverse(z, 0)
        else:
            z, log_det = self.iresblock.forward(z, 0)
        return z, -log_det.view(-1)

    def inverse(self, z):
        if self.reverse:
            z, log_det = self.iresblock.forward(z, 0)
        else:
            z, log_det = self.iresblock.inverse(z, 0)
        return z, -log_det.view(-1)


class iResBlock(nn.Module):
    def __init__(self, nnet, geom_p=0.5, lamb=2.0, n_power_series=None, exact_trace=False, brute_force=False,
                 n_samples=1, n_exact_terms=2, n_dist="geometric", neumann_grad=True, grad_in_forward=False):
        super().__init__()
        self.nnet = nnet
        self.n_dist = n_dist
        self.geom_p = nn.Parameter(torch.tensor(np.log(geom_p) - np.log(1.0 - geom_p)))
        self.lamb = nn.Parameter(torch.tensor(lamb))
        self.n_samples, self.n_power_series = n_samples, n_power_series
        self.exact_trace, self.brute_force, self.n_exact_terms = exact_trace, brute_force, n_exact_terms
        self.grad_in_forward, self.neumann_grad = grad_in_forward, neumann_grad
        self.register_buffer("last_n_samples", torch.zeros(self.n_samples))
        self.register_buffer("last_firmom", torch.zeros(1))
        self.register_buffer("last_secmom", torch.zeros(1))
        # test hooks: inject the random truncation / the probe vector of the next _logdetgrad call
        self._inject_n, self._inject_eps = None, None

    # ---- the network, split into its layers ------------------------------------------------------------
    def _layers(self):
        mods = list(self.nnet.net) if hasattr(self.nnet, "net") else None
        if not mods or len(mods) % 2 or not all(isinstance(mods[i], Swish) and isinstance(mods[i + 1], InducedNormLinear)
                                                for i in range(0, len(mods), 2)):
            raise NotImplementedError("the CUDA path of Residual takes a nets.LipschitzMLP")
        return [(mods[i], mods[i + 1]) for i in range(0, len(mods), 2)]

    @torch.no_grad()
    def _run(self, x, tangents=None, keep=False):
        """g(x); optionally pushes `tangents` [nt, B, D] forward (Jacobian-vector products) and/or keeps what the
        vector-Jacobian product needs (activation derivatives, effective weights)."""
        h, t, tape = x, tangents, []
        for sw, lin in self._layers():
            a, da = swish(h, float(F.softplus(sw.beta.detach())), want_derivative=(t is not None or keep))
            w = lin.compute_weight(update=False).contiguous()
            if t is not None:
                nt, b, width = t.shape
                t = mul_rows(t, da, nt)
                t = linear(t.reshape(nt * b, width), w).reshape(nt, b, w.shape[0])
            if keep:
                tape.append((da, w))
            h = linear(a, w, lin.bias)
        return h, t, tape

    @torch.no_grad()
    def _vjp(self, v, tape):
        """v^T J for every row (reverse mode through the taped layers)."""
        for da, w in reversed(tape):
            v = linear_t(v, w)       # (v W): cotangent w.r.t. the activation
            v = mul_rows(v[None], da, 1)[0]
        return v

    # ---- reference API ---------------------------------------------------------------------------------
    def forward(self, x, logpx=None):
        if logpx is None:
            return x + self._run(require_cuda_f32(x))[0]
        g, logdetgrad = self._logdetgrad(x)
        return x + g, logpx - logdetgrad

    def inverse(self, y, logpy=None):
        x = self._inverse_fixed_point(y)
        if logpy is None:
            return x
        return x, logpy + self._logdetgrad_values(x)[1]   # the sampling direction is value-only

    @torch.no_grad()
    def _inverse_fixed_point(self, y, atol=1e-5, rtol=1e-5):
        y = require_cuda_f32(y)
        x, x_prev = y - self._run(y)[0], y
        i = 0
        tol = atol + y.abs() * rtol
        while not torch.all((x - x_prev) ** 2 / tol < 1):
            x, x_prev = y - self._run(x)[0], x
            i += 1
            if i > 1000:
                break
        return x

    def _exact(self, x):
        return (self.brute_force or not self.training) and x.dim() == 2 and x.shape[1] == 2

    def _logdetgrad(self, x):
        """(g(x), log|det(I + dg/dx)| estimate [B, 1]); differentiable (ResidualBlockFn) when a gradient is wanted."""
        if not wants_grad(self, x):
            return self._logdetgrad_values(x)[:2]
        if self.training and not self._exact(x) and not self.neumann_grad:
            raise NotImplementedError(
                "Residual(reduce_memory=False): the gradient of the basic power-series estimator in training mode is not "
                "on the CUDA path; train with reduce_memory=True (the Neumann-series gradient, the default)")
        return ResidualBlockFn.apply(self, x, *self._grad_params())

    def _grad_params(self):
        return [p for sw, lin in self._layers() for p in (sw.beta, lin.weight, lin.bias)]

    @torch.no_grad()
    def _logdetgrad_values(self, x):
        """(g, log-det [B, 1], what the backward needs: the tangents pushed through g and their seeds' ingredients)."""
        x = require_cuda_f32(x)
        if self._exact(x):
            # exact 2 x 2 Jacobian by two forward-mode tangents (residual.py:148-161)
            b = x.shape[0]
            eye = torch.zeros(2, b, 2, device=x.device)
            eye[0, :, 0] = 1.0
            eye[1, :, 1] = 1.0
            g, jt, _ = self._run(x, tangents=eye)
            jt = jt.contiguous()
            out = torch.empty(b, device=x.device)
            if b:
                with torch.cuda.device(x.device):
                    L.check(L.lib().nfb_logabsdet_i_plus_j_2x2(L.ptr(jt), b, L.ptr(out), L.stream_ptr()))
            return g, out.view(-1, 1), {"mode": "exact", "tangents": eye, "jt": jt}
        if x.dim() != 2:
            raise NotImplementedError("the CUDA path of Residual takes [batch, features] inputs")
        if self.exact_trace:
            raise NotImplementedError("exact_trace=True is not on the CUDA path (use brute_force for 2-D inputs)")
        if self.n_dist == "geometric":
            geom_p = torch.sigmoid(self.geom_p).item()
            sample_fn = lambda m: geometric_sample(geom_p, m)
            rcdf_fn = lambda k, offset: geometric_1mcdf(geom_p, k, offset)
        elif self.n_dist == "poisson":
            lamb = self.lamb.item()
            sample_fn = lambda m: poisson_sample(lamb, m)
            rcdf_fn = lambda k, offset: poisson_1mcdf(lamb, k, offset)
        else:
            raise ValueError("unknown n_dist " + str(self.n_dist))
        draw = (lambda m: np.asarray(self._inject_n)) if self._inject_n is not None else sample_fn
        n_samples = None
        if self.training:
            if self.n_power_series is None:
                n_samples = draw(self.n_samples)
                n_power_series = max(n_samples) + self.n_exact_terms
                exact = self.n_exact_terms
                coeff_fn = lambda k: 1 / rcdf_fn(k, exact) * sum(n_samples >= k - exact) / len(n_samples)
            else:
                n_power_series = self.n_power_series
                coeff_fn = lambda k: 1.0
        else:
            n_samples = draw(self.n_samples)
            n_power_series = max(n_samples) + 20
            coeff_fn = lambda k: 1 / rcdf_fn(k, 20) * sum(n_samples >= k - 20) / len(n_samples)
        vareps = self._inject_eps if self._inject_eps is not None else torch.randn_like(x)
        vareps = require_cuda_f32(vareps)
        self._inject_n, self._inject_eps = None, None
        g, _, tape = self._run(x, keep=True)
        n_power_series = int(n_power_series)
        if self.training and self.neumann_grad:
            # neumann_logdet_estimator (:368-379): the value is the Neumann-series surrogate of the reference
            vjp, neumann = vareps, vareps.clone()
            for k in range(1, n_power_series + 1):
                vjp = self._vjp(vjp, tape)
                neumann.add_(vjp, alpha=float((-1) ** k * coeff_fn(k)))
            logdetgrad = rowdot(self._vjp(neumann, tape), vareps)
            saved = {"mode": "neumann", "tangents": vareps[None], "w": neumann}
        else:
            # basic_logdet_estimator (:355-366)
            vjp, logdetgrad = vareps, None
            for k in range(1, n_power_series + 1):
                vjp = self._vjp(vjp, tape)
                logdetgrad = rowdot(vjp, vareps, c=float((-1) ** (k + 1) / k * coeff_fn(k)), out=logdetgrad)
            saved = {"mode": "g_only"}   # eval mode: the estimator is not differentiated (:355-366, create_graph=False)
        if self.training and self.n_power_series is None:
            self.last_n_samples.copy_(torch.tensor(n_samples).to(self.last_n_samples))
            self.last_firmom.copy_(torch.mean(logdetgrad).to(self.last_firmom))
            self.last_secmom.copy_(torch.mean(logdetgrad ** 2).to(self.last_secmom))
        return g, logdetgrad.view(-1, 1), saved


class ResidualBlockFn(torch.autograd.Function):
    """(g, log-det) = iResBlock._logdetgrad(x) with gradients w.r.t. x and every beta / weight / bias of the
    LipschitzMLP (geom_p and lamb get none: the reference reads them with .item()).

    The backward differentiates the dual network g pushed forward with tangents t_0, seeded per mode:
      neumann  (training, reduce_memory=True; residual.py:282-352,368-379): t_0 = eps; the value is s = w^T J eps with
               the Neumann vector w held constant, and like MemoryEfficientLogDetEstimator.backward (:335) the
               cotangent of row 0's log-det scales the gradient of every row: tangent seed g_ld[0] * w;
      exact    (2-D, eval or brute_force; :148-161): t_0 = e_0, e_1; tangent seeds g_ld[r] (I + J_r)^-T;
      g_only   (eval, D > 2: the basic estimator without create_graph): no tangents; the log-det is not differentiable.
    W~ = compute_weight(update=False) and b = softplus(beta) are rebuilt with torch autograd and chained back."""

    @staticmethod
    def forward(ctx, block, x, *params):
        g, ld, saved = block._logdetgrad_values(x)
        ctx.block, ctx.mode, ctx.params = block, saved["mode"], params
        # the backward recomputes from the module's parameters and the spectral-norm vectors u, v
        ctx.watched = list(params) + [t for _, lin in block._layers() for t in (lin.u, lin.v)]
        ctx.versions = [t._version for t in ctx.watched]
        ctx.save_for_backward(x, saved.get("tangents"), saved.get("w"), saved.get("jt"))
        if ctx.mode == "g_only":
            ctx.mark_non_differentiable(ld)
        return g, ld

    @staticmethod
    def backward(ctx, g_g, g_ld):
        x, tangents, w, jt = ctx.saved_tensors
        if any(t._version != v for t, v in zip(ctx.watched, ctx.versions)):
            raise RuntimeError("Residual backward: a parameter or a spectral-norm vector (u, v) of the block was modified "
                               "in place after the forward pass (e.g. update_lipschitz before backward): the recompute "
                               "would differentiate other weights than the forward used")
        x = x.contiguous()
        B, dev = x.shape[0], x.device
        layers = ctx.block._layers()
        nt = 0 if tangents is None else tangents.shape[0]
        g_ld = torch.zeros(B, device=dev) if g_ld is None else g_ld.reshape(-1).float().contiguous()
        g_g = g_g.contiguous() if g_g is not None else None
        t_seeds = None
        if ctx.mode == "neumann" and B:
            t_seeds = (w * g_ld[0])[None].contiguous()   # residual.py:335: dL = grad_logdetgrad[0] for every row
        elif ctx.mode == "exact":
            t_seeds = torch.empty_like(tangents)
            if B:
                with torch.cuda.device(dev):
                    L.check(L.lib().nfb_logabsdet_i_plus_j_2x2_backward(L.ptr(jt), L.ptr(g_ld), B, L.ptr(t_seeds),
                                                                          L.stream_ptr()))
        with torch.enable_grad():
            weff = [lin.compute_weight(update=False) for _, lin in layers]
            bs = [F.softplus(sw.beta) for sw, _ in layers]
        d = L.LipschitzMlpDesc()
        d.num_layers = len(layers)
        d.widths[0] = x.shape[1]
        wd = [t.detach().contiguous() for t in weff]
        bias = [lin.bias.detach().contiguous() for _, lin in layers]
        for l, (_, lin) in enumerate(layers):
            d.widths[l + 1] = lin.out_features
            d.w[l], d.bias[l], d.b[l] = wd[l].data_ptr(), bias[l].data_ptr(), float(bs[l])
        gx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        gW = [torch.empty_like(t) for t in wd]
        gbias = [torch.empty_like(t) for t in bias]
        gb = torch.empty(len(layers), device=dev)
        VP = C.c_void_p
        gW_arr = (VP * len(layers))(*[t.data_ptr() for t in gW])
        gbias_arr = (VP * len(layers))(*[t.data_ptr() for t in gbias])
        lib = L.lib()
        nbytes = lib.nfb_lipschitz_mlp_dual_backward_workspace_bytes(C.byref(d), nt, B)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.nfb_lipschitz_mlp_dual_backward(
                C.byref(d), L.ptr(x), L.ptr(tangents), nt, L.ptr(g_g), L.ptr(t_seeds), B, L.ptr(ws), nbytes, L.ptr(gx),
                gW_arr, gbias_arr, L.ptr(gb), L.stream_ptr()))
        # W~ -> weight (spectral normalisation) and b -> beta: torch autograd over compute_weight / softplus
        outs = [t for t in weff + bs if t.requires_grad]
        cots = [c for t, c in zip(weff + bs, gW + [gb[l:l + 1] for l in range(len(layers))]) if t.requires_grad]
        src = [p for _, lin in layers for p in (lin.weight,)] + [sw.beta for sw, _ in layers]
        src = [p for p in src if p.requires_grad]
        chained = dict(zip(map(id, src), torch.autograd.grad(outs, src, cots, allow_unused=True))) if outs else {}
        for (_, lin), gbl in zip(layers, gbias):
            chained[id(lin.bias)] = gbl
        return (None, gx, *[chained.get(id(p)) if p.requires_grad else None for p in ctx.params])


def geometric_sample(p, n_samples):
    return np.random.geometric(p, n_samples)


def geometric_1mcdf(p, k, offset):
    if k <= offset:
        return 1.0
    k = k - offset
    return (1 - p) ** max(k - 1, 0)


def poisson_sample(lamb, n_samples):
    return np.random.poisson(lamb, n_samples)


def poisson_1mcdf(lamb, k, offset):
    if k <= offset:
        return 1.0
    k = k - offset
    s = 1.0
    for i in range(1, k):
        s += lamb ** i / math.factorial(i)
    return 1 - np.exp(-lamb) * s
