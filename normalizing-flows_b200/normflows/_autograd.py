"""Gradients for the density pass.

`forward_kld` / `log_prob` run on the hand-written CUDA path.  Their backward is native for stacks of spline blocks,
LULinearPermute and affine-family layers (`native_backward`: nfb_flow_log_prob_backward).  For other stacks -- INTERIM
(SURVEY 8f-1 "backward of the fused blocks" is the real fix) -- and as the A/B reference of the GPU tests
(`DensityFn.use_native_backward = False`), the autograd hook below re-materialises the same density pass in
differentiable torch ops ON THE SAME DEVICE during backward and lets autograd produce exact gradients.  The forward
value, the metric and every parity claim come from the CUDA kernels; this module is only reached from
`backward()`.  It restates (mask-free) the same reference arithmetic as the kernels:
  spline utils/splines.py:16-219, MADE nets/made.py:296-304, ResidualNet nets/resnet.py:92-104,
  LULinearPermute flows/mixing.py:402-434,514-532, affine family flows/affine/coupling.py, DiagGaussian
  distributions/base.py:94-103, GaussianMixture distributions/base.py:645-659 (with log_softmax).
"""
import math

import torch
import torch.nn.functional as F

_BOUNDARY = math.log(math.exp(1 - 1e-3) - 1)


def _knots(un, tail, k):
    s = torch.softmax(un, dim=-1)
    s = 1e-3 + (1 - 1e-3 * k) * s
    cum = F.pad(torch.cumsum(s, dim=-1), (1, 0))
    cum = 2 * tail * cum - tail
    cum = torch.cat([torch.full_like(cum[..., :1], -tail), cum[..., 1:-1], torch.full_like(cum[..., :1], tail)], -1)
    return cum, cum[..., 1:] - cum[..., :-1]


def spline_forward(x, uw, uh, ud, tail):
    """Density-direction spline (inverse=False), mask-free; returns y, logabsdet (elementwise)."""
    k = uw.shape[-1]
    inside = (x >= -tail) & (x <= tail)
    xs = torch.where(inside, x, torch.zeros_like(x))
    cumw, w = _knots(uw, tail, k)
    cumh, h = _knots(uh, tail, k)
    pad = torch.full_like(ud[..., :1], _BOUNDARY)
    d = 1e-3 + F.softplus(torch.cat([pad, ud, pad], -1))
    loc = cumw.detach().clone()
    loc[..., -1] += 1e-6
    idx = (torch.sum(xs[..., None] >= loc, dim=-1) - 1).clamp(0, k - 1)[..., None]
    g = lambda t: t.gather(-1, idx)[..., 0]
    in_cw, in_w, in_ch, in_h = g(cumw), g(w), g(cumh), g(h)
    delta = in_h / in_w
    d0, d1 = g(d), g(d[..., 1:])
    theta = (xs - in_cw) / in_w
    tomt = theta * (1 - theta)
    num = in_h * (delta * theta ** 2 + d0 * tomt)
    den = delta + (d0 + d1 - 2 * delta) * tomt
    y = in_ch + num / den
    dnum = delta ** 2 * (d1 * theta ** 2 + 2 * delta * tomt + d0 * (1 - theta) ** 2)
    lad = torch.log(dnum) - 2 * torch.log(den)
    return torch.where(inside, y, x), torch.where(inside, lad, torch.zeros_like(lad))


def _resnet(net, x, masked):
    lin = (lambda l, v: F.linear(v, l.weight * l.mask, l.bias)) if masked else (lambda l, v: F.linear(v, l.weight, l.bias))
    h = lin(net.initial_layer, x)
    for blk in net.blocks:
        t = lin(blk.linear_layers[0], torch.relu(h))
        t = lin(blk.linear_layers[1], torch.relu(t))
        h = h + t
    return lin(net.final_layer, h)


def layer_inverse(layer, z):
    """(z', log_det[B]) of `layer.inverse(z)` in differentiable torch ops."""
    from .flows import neural_spline as ns, mixing, affine, planar
    b = z.shape[0]
    if isinstance(layer, ns.AutoregressiveRationalQuadraticSpline):
        k = layer.num_bins
        p = _resnet(layer.mprqat.autoregressive_net, z, True).reshape(b, z.shape[1], 3 * k - 1)
        y, lad = spline_forward(z, p[..., :k], p[..., k:2 * k], p[..., 2 * k:], layer.tail_bound)
        return y, lad.sum(1)
    if isinstance(layer, ns.CoupledRationalQuadraticSpline):
        k, q = layer.num_bins, layer.prqct
        idf, trf = q.identity_features, q.transform_features
        ident, trans = z[:, idf], z[:, trf]
        p = _resnet(q.transform_net, ident, False).reshape(b, len(trf), 3 * k - 1)
        sc = 1.0 / math.sqrt(q.transform_net.hidden_features)
        yt, lad = spline_forward(trans, p[..., :k] * sc, p[..., k:2 * k] * sc, p[..., 2 * k:], layer.tail_bound)
        u = q.unconditional_transform
        ex = lambda t: t[None].expand(b, *t.shape)
        yi, ladi = spline_forward(ident, ex(u.unnormalized_widths), ex(u.unnormalized_heights),
                                  ex(u.unnormalized_derivatives), layer.tail_bound)
        out = torch.empty_like(z)
        out = out.index_copy(1, idf, yi).index_copy(1, trf, yt)
        return out, lad.sum(1) + ladi.sum(1)
    if isinstance(layer, mixing.LULinearPermute):
        lin, n = layer.linear, layer.linear.features
        lower = z.new_zeros(n, n)
        upper = z.new_zeros(n, n)
        il, iu = torch.tril_indices(n, n, -1, device=z.device), torch.triu_indices(n, n, 1, device=z.device)
        lower = lower.index_put((il[0], il[1]), lin.lower_entries) + torch.eye(n, device=z.device, dtype=z.dtype)
        diag = F.softplus(lin.unconstrained_upper_diag) + lin.eps
        upper = upper.index_put((iu[0], iu[1]), lin.upper_entries) + torch.diag(diag)
        x = z[:, layer.permutation._permutation]
        x = F.linear(F.linear(x, upper), lower, lin.bias)
        return x, torch.sum(torch.log(diag)) * z.new_ones(b)
    if isinstance(layer, affine.MaskedAffineFlow):
        mlp = lambda net, v: v.new_zeros(v.shape) if net is None else net.net(v)
        zm = layer.b * z
        s, t = mlp(layer.s, zm), mlp(layer.t, zm)
        nan = torch.tensor(float("nan"), dtype=z.dtype, device=z.device)
        s, t = torch.where(torch.isfinite(s), s, nan), torch.where(torch.isfinite(t), t, nan)
        return zm + (1 - layer.b) * (z - t) * torch.exp(-s), -torch.sum((1 - layer.b) * s, dim=1)
    if isinstance(layer, affine.AffineCouplingBlock):
        h = (z.shape[1] + 1) // 2
        a, c = z[:, :h], z[:, h:]
        z1, z2 = (a, c) if layer.split_mode == "channel" else (c, a)
        param = layer.flows[1].param_map.net(z1)
        if not layer.scale:
            z2, ld = z2 - param, z.new_zeros(b)
        else:
            shift, sc = param[:, 0::2], param[:, 1::2]
            if layer.scale_map == "exp":
                z2, ld = (z2 - shift) * torch.exp(-sc), -sc.sum(1)
            else:
                sg = torch.sigmoid(sc + 2)
                if layer.scale_map == "sigmoid":
                    z2, ld = (z2 - shift) * sg, torch.log(sg).sum(1)
                else:
                    z2, ld = (z2 - shift) / sg, -torch.log(sg).sum(1)
        return torch.cat([z1, z2] if layer.split_mode == "channel" else [z2, z1], 1), ld
    if isinstance(layer, affine.AffineConstFlow):  # includes ActNorm (after init)
        s, t = layer.s.reshape(1, -1), layer.t.reshape(1, -1)
        return (z - t) * torch.exp(-s), -torch.sum(s) * z.new_ones(b)
    if isinstance(layer, planar.Planar):   # leaky-ReLU layers only (flows/planar.py:66-81)
        if layer._no_inverse:
            raise NotImplementedError("This flow has no algebraic inverse.")
        w, u = layer.w.reshape(1, -1), layer.u.reshape(1, -1)
        lin = torch.sum(w * z, 1) + layer.b
        a = (lin < 0) * (layer.h.negative_slope - 1.0) + 1.0
        inner = torch.sum(w * u)
        u = u + (torch.log(1 + torch.exp(inner)) - 1 - inner) * w / torch.sum(w ** 2)
        u = a.reshape(-1, 1) * u
        inner_ = torch.sum(w * u, 1)
        return z - u * (lin / (1 + inner_)).reshape(-1, 1), -torch.log(torch.abs(1 + inner_))
    if isinstance(layer, mixing.Permute):
        _, inv = layer._index_lists()
        return z[:, torch.tensor(inv, device=z.device)], z.new_zeros(b)
    raise NotImplementedError(f"no differentiable restatement for {type(layer).__name__}")


def log_prob(model, x):
    z, lq = x, x.new_zeros(x.shape[0])
    for layer in reversed(list(model.flows)):
        z, ld = layer_inverse(layer, z)
        lq = lq + ld
    from .distributions.base import GaussianMixture
    q0 = model.q0
    if isinstance(q0, GaussianMixture):
        ls, loc = q0.log_scale, q0.loc
        e = (torch.log_softmax(q0.weight_scores, 1) - 0.5 * q0.dim * math.log(2 * math.pi)
             - torch.sum(ls + 0.5 * ((z[:, None, :] - loc) / torch.exp(ls)) ** 2, 2))
        return lq + torch.logsumexp(e, 1)
    ls = q0.log_scale.reshape(1, -1)
    lq = lq - 0.5 * q0.d * math.log(2 * math.pi) - torch.sum(ls + 0.5 * ((z - q0.loc.reshape(1, -1)) / torch.exp(ls)) ** 2, 1)
    return lq


def _net_slots(net):
    ps = [net.initial_layer.weight, net.initial_layer.bias]
    for blk in net.blocks:
        for lin in blk.linear_layers:
            ps += [lin.weight, lin.bias]
    return ps + [net.final_layer.weight, net.final_layer.bias]


def grad_slot_tensors(model):
    """Parameters in the order of the C ABI's gradient slots (include/nfb200.h nfb_flow_log_prob_backward), or None
    if a layer has no native backward.  An affine-family layer's slots are those of the sampling backward; a buffer
    behind a slot (AffineConstFlow(scale=False)) gets no buffer."""
    from .flows import neural_spline as ns, mixing
    from ._standalone import sampling_slot_tensors
    out = []
    for layer in model.flows:
        if getattr(layer, "_affine_family", False) or isinstance(layer, (ns.CoupledRationalQuadraticSpline,
                                                                          mixing.LULinearPermute)):
            out += sampling_slot_tensors([layer])
        elif isinstance(layer, ns.AutoregressiveRationalQuadraticSpline):
            out += _net_slots(layer.mprqat.autoregressive_net)
        else:
            return None
    return out + model.q0._native_tensors()


def native_backward(model, x, grad_out, need_x):
    """Gradients from libnfb200.so (csrc/nfb_api.cu nfb_flow_log_prob_backward: tensor-core dgrad/wgrad + analytic
    spline adjoint, the affine family's per-row adjoint kernel).  Returns (gx | None, {id(param): grad}) or None when
    the stack is not covered."""
    import ctypes as C
    from . import _lib as L
    from ._standalone import sum_slot_grads
    slots = grad_slot_tensors(model)
    h = model._stack()
    if slots is None or h is None or h.base is None or x.dim() != 2:
        return None
    handle = h.ensure(x.shape[1], x.device)
    lib = L.lib()
    n = lib.nfb_flow_num_grad_slots(handle)
    if n < 0:
        return None
    if n != len(slots):
        raise RuntimeError(f"gradient slot mismatch: library {n}, python {len(slots)}")
    bufs = []
    for i, p in enumerate(slots):
        want = isinstance(p, torch.nn.Parameter) and p.requires_grad
        if want and lib.nfb_flow_grad_slot_numel(handle, i) != p.numel():
            raise RuntimeError(f"gradient slot {i}: size mismatch")
        bufs.append(torch.empty_like(p) if want else None)
    arr = (C.c_void_p * n)(*[b.data_ptr() if b is not None else None for b in bufs])
    g = grad_out.detach().to(torch.float32).contiguous()
    xx = x.detach().contiguous()
    gx = torch.empty_like(xx) if need_x else None
    with torch.cuda.device(x.device):
        L.check(lib.nfb_flow_log_prob_backward(handle, L.ptr(xx), L.ptr(g), xx.shape[0], None, L.ptr(gx), arr,
                                               L.stream_ptr()))
    return gx, sum_slot_grads(slots, bufs)


class DensityFn(torch.autograd.Function):
    """log_prob(x) on the CUDA path.  backward: native kernels (dgrad / wgrad on the tensor core, analytic spline
    adjoint, the affine family's per-row adjoint kernel) for stacks of spline blocks, LULinearPermute and affine-family
    layers; other stacks re-materialise a torch graph (interim)."""
    use_native_backward = True

    @staticmethod
    def forward(ctx, model, x, *params):
        ctx.model = model
        ctx.save_for_backward(x)
        with torch.no_grad():
            return model._stack().log_prob(x)

    @staticmethod
    def backward(ctx, grad_out):
        (x,) = ctx.saved_tensors
        model = ctx.model
        need_x = ctx.needs_input_grad[1]
        if DensityFn.use_native_backward:
            res = native_backward(model, x, grad_out, need_x)
            if res is not None:
                gx, gmap = res
                return (None, gx, *[gmap.get(id(p)) if p.requires_grad else None for p in model.parameters()])
        with torch.enable_grad():
            xx = x.detach().requires_grad_(need_x)
            lq = log_prob(model, xx)
            params = [p for p in model.parameters() if p.requires_grad]
            wrt = ([xx] if need_x else []) + params
            grads = torch.autograd.grad(lq, wrt, grad_out, allow_unused=True) if wrt else []
        gx = grads[0] if need_x else None
        gp = list(grads[1:] if need_x else grads)
        it = iter(gp)
        out = [next(it) if p.requires_grad else None for p in model.parameters()]
        return (None, gx, *out)


class LayerInverseFn(torch.autograd.Function):
    """(z', log_det) = layer.inverse(z) of ONE NativeFlow called on its own (a layer of a stack that also holds non-native
    layers, e.g. the ActNorms between Residual blocks).  The forward is the layer's kernel (FlowHandle.layer_apply).  The
    backward of an affine-family layer is nfb_flow_density_backward on the layer's own handle; other layers
    (LULinearPermute, leaky Planar) re-materialise the layer with `layer_inverse` above (interim, like DensityFn's torch
    path)."""

    @staticmethod
    def forward(ctx, layer, z, *params):
        from . import _lib as L
        out, ld = layer._single().layer_apply(0, L.NFB_INVERSE, z)
        ctx.layer, ctx.params = layer, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(z)
        return out, ld

    @staticmethod
    def backward(ctx, g_out, g_ld):
        (z,) = ctx.saved_tensors
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError(f"{type(ctx.layer).__name__} backward: a parameter was modified in place after the forward pass")
        need_z = ctx.needs_input_grad[1]
        if getattr(ctx.layer, "_affine_family", False):
            from . import _lib as L
            from ._standalone import stack_backward
            gz, gmap = stack_backward(ctx.layer._single(), [ctx.layer], L.NFB_INVERSE, z.contiguous(), g_out, g_ld,
                                      need_z)
            return (None, gz, *[gmap.get(id(p)) if p.requires_grad else None for p in ctx.params])
        params = [p for p in ctx.params if p.requires_grad]
        with torch.enable_grad():
            zz = z.detach().requires_grad_(need_z)
            out, ld = layer_inverse(ctx.layer, zz)
            pairs = [(t, g) for t, g in ((out, g_out), (ld, g_ld)) if g is not None and t.requires_grad]
            wrt = ([zz] if need_z else []) + params
            grads = torch.autograd.grad([t for t, _ in pairs], wrt, [g for _, g in pairs], allow_unused=True) \
                if pairs and wrt else [None] * len(wrt)
        gz = grads[0] if need_z else None
        it = iter(grads[1:] if need_z else grads)
        return (None, gz, *[next(it) if p.requires_grad else None for p in ctx.params])
