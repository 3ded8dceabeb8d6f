"""Gradients of the stand-alone layers: the context-conditioned and circular spline layers, and the conditioner nets
(ResidualNet, MADE, MLP, PeriodicFeaturesElementwise) called as modules.  Density direction only.

A module that supports this defines
  `_value(x, context, keep)`  its kernel forward (the module's no-grad path; `keep`, when not None, is a dict in which
                              it may leave tensors for the backward, e.g. the conditioner output of a spline layer), and
  `_adjoint(x, context, keep, grads, need_x, need_ctx)` -> (g_x, g_context, {parameter: gradient})
and `apply_module` routes a call through `ModuleFn` when a gradient is wanted.  The backward is the C ABI's adjoints:
nfb_rqs_spline(_tails)_backward -> nfb_resnet_backward / nfb_mlp_backward (one call per conditioner) ->
nfb_periodic_features_backward.

The sampling direction (`forward` of the autoregressive and coupling spline layers, which reverse_kld differentiates)
goes the same way through `SamplingFn`: a module defines `_sampling_value(z, context, keep)` (its unchanged sampling
code) and `_sampling_adjoint(z, x, context, keep, g_x, g_ld, need_z, need_ctx)`, built on the inverse-spline adjoints
nfb_rqs_spline(_tails)_inverse_backward and the fixed-point adjoint nfb_ar_rqs_sampling_backward."""
import ctypes as C

import torch

from . import _lib as L
from ._image_autograd import wants_grad
from ._native import mlp_desc, require_cuda_f32, resnet_desc


def _vp(ts):
    return (C.c_void_p * max(1, len(ts)))(*[t.data_ptr() if t is not None else None for t in ts])


def _grad_like(p):
    return torch.empty_like(p) if p.requires_grad else None


def _workspace(nbytes, device):
    if nbytes < 0:
        raise RuntimeError("native backward: bad descriptor or shape")
    return torch.empty(max(1, int(nbytes)), dtype=torch.uint8, device=device)


class ModuleFn(torch.autograd.Function):
    """out = module._value(x, context) with the module's native adjoint as the backward.  Refuses to run the backward if a
    parameter was modified in place after the forward (the saved activations would no longer match)."""

    @staticmethod
    def forward(ctx, module, x, context, *params):
        keep = {}
        out = module._value(x, context, keep)
        ctx.module, ctx.keep, ctx.params = module, keep, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(x, context)
        return out

    @staticmethod
    def backward(ctx, *grads):
        x, context = ctx.saved_tensors
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError(f"{type(ctx.module).__name__} backward: a parameter was modified in place after the "
                               "forward pass")
        grads = [g.contiguous() if g is not None else None for g in grads]
        gx, gctx, gmap = ctx.module._adjoint(x, context, ctx.keep, grads, ctx.needs_input_grad[1],
                                             ctx.needs_input_grad[2])
        return (None, gx if ctx.needs_input_grad[1] else None, gctx if ctx.needs_input_grad[2] else None,
                *[gmap.get(p) if p.requires_grad else None for p in ctx.params])


def apply_module(module, x, context=None):
    x = require_cuda_f32(x)
    if context is not None:
        context = require_cuda_f32(context, "context")
    if wants_grad(module, x, context):
        return ModuleFn.apply(module, x, context, *module.parameters())
    return module._value(x, context, None)


class SamplingFn(torch.autograd.Function):
    """(x, log_det) = module._sampling_value(z, context): the layer's sampling code under no_grad, so values are
    bit-identical with and without grad; the backward is the module's `_sampling_adjoint`.  Refuses to run the backward
    if a parameter was modified in place after the forward."""

    @staticmethod
    def forward(ctx, module, z, context, *params):
        keep = {}
        x, ld = module._sampling_value(z, context, keep)
        ctx.module, ctx.keep, ctx.params = module, keep, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(z, x, context)
        return x, ld

    @staticmethod
    def backward(ctx, g_x, g_ld):
        z, x, context = ctx.saved_tensors
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError(f"{type(ctx.module).__name__} backward: a parameter was modified in place after the "
                               "forward pass")
        need_z, need_ctx = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gz, gctx, gmap = ctx.module._sampling_adjoint(z, x, context, ctx.keep,
                                                      g_x.contiguous() if g_x is not None else None,
                                                      g_ld.contiguous() if g_ld is not None else None, need_z, need_ctx)
        return (None, gz if need_z else None, gctx if need_ctx else None,
                *[gmap.get(p) if p.requires_grad else None for p in ctx.params])


def apply_sampling(module, z, context=None):
    z = require_cuda_f32(z)
    if context is not None:
        context = require_cuda_f32(context, "context")
    if wants_grad(module, z, context):
        return SamplingFn.apply(module, z, context, *module.parameters())
    return module._sampling_value(z, context, None)


def sampling_slot_tensors(layers):
    """The tensors behind the gradient slots of an affine-family, planar-family or coupled-spline / LU stack
    (include/nfb200.h nfb_flow_grad_slot_numel): an affine or planar layer's parameters in registration order (an
    AffineConstFlow s / t registered as a buffer keeps its slot); a coupled spline's conditioner Linears (weight, bias)
    then its unconditional widths, heights, derivatives; an LULinearPermute's lower, upper, diagonal, bias."""
    from ._autograd import _net_slots
    from .flows import affine, mixing, neural_spline, planar, radial
    out = []
    for layer in layers:
        if isinstance(layer, neural_spline.CoupledRationalQuadraticSpline):
            u = layer.prqct.unconditional_transform
            out += _net_slots(layer.prqct.transform_net)
            out += [u.unnormalized_widths, u.unnormalized_heights, u.unnormalized_derivatives]
        elif isinstance(layer, mixing.LULinearPermute):
            lin = layer.linear
            out += [lin.lower_entries, lin.upper_entries, lin.unconstrained_upper_diag, lin.bias]
        elif isinstance(layer, planar.Planar):
            out += [layer.u, layer.w, layer.b]
        elif isinstance(layer, radial.Radial):
            out += [layer.beta, layer.alpha, layer.z_0]
        elif isinstance(layer, affine.MaskedAffineFlow):
            for net in (layer.s, layer.t):
                if net is not None:
                    out += [p for lin in net.linear_layers() for p in (lin.weight, lin.bias)]
        elif isinstance(layer, affine.AffineConstFlow):
            out += [layer.s, layer.t]
        elif isinstance(layer, affine.AffineCouplingBlock):
            out += [p for lin in layer.flows[1].param_map.linear_layers() for p in (lin.weight, lin.bias)]
        elif not isinstance(layer, mixing.Permute):
            raise NotImplementedError(f"{type(layer).__name__} has no native sampling-direction backward")
    return out


affine_slot_tensors = sampling_slot_tensors   # (the name callers of the affine-only version use)


def sum_slot_grads(slots, bufs):
    """{id(parameter): gradient} from per-slot gradient buffers: a parameter behind several slots (a net or layer used
    twice) gets the sum, as autograd would give."""
    gmap = {}
    for p, b in zip(slots, bufs):
        if b is not None:
            gmap[id(p)] = gmap[id(p)] + b if id(p) in gmap else b
    return gmap


def stack_backward(handle, layers, direction, z, g_out, g_ld, need_z):
    """(g_z | None, {id(parameter): gradient}) of (out, log_det) = handle.transform(direction, z) through
    nfb_flow_sampling_backward (NFB_FORWARD: all-affine, all-planar or coupled-spline / LU stacks) or
    nfb_flow_density_backward (NFB_INVERSE:
    all-affine stacks); g_out / g_ld are the cotangents of out / log_det (None: zero)."""
    slots = sampling_slot_tensors(layers)
    bufs = [torch.empty_like(p) if isinstance(p, torch.nn.Parameter) and p.requires_grad else None for p in slots]
    gz = torch.empty_like(z) if need_z else None
    g_out = g_out.to(torch.float32).contiguous() if g_out is not None else None
    g_ld = g_ld.to(torch.float32).contiguous() if g_ld is not None else None
    lib = L.lib()
    h = handle.ensure(z.shape[1], z.device)
    if lib.nfb_flow_num_grad_slots(h) < len(slots):
        raise RuntimeError("native backward: gradient slot mismatch")
    if direction == L.NFB_FORWARD:
        ws_bytes, call = lib.nfb_flow_sampling_backward_workspace_bytes, lib.nfb_flow_sampling_backward
    else:
        ws_bytes, call = lib.nfb_flow_density_backward_workspace_bytes, lib.nfb_flow_density_backward
    ws = _workspace(ws_bytes(h, z.shape[0]), z.device)
    arr = _vp(bufs)
    with torch.cuda.device(z.device):
        L.check(call(h, L.ptr(z), L.ptr(g_out), L.ptr(g_ld), z.shape[0], L.ptr(ws), ws.numel(), L.ptr(gz),
                     C.cast(arr, C.POINTER(C.c_void_p)), L.stream_ptr()))
    return gz, sum_slot_grads(slots, bufs)


class StackSamplingFn(torch.autograd.Function):
    """(out, log_det) = handle.transform(direction, z) of an all-affine stack (MaskedAffineFlow, AffineConstFlow /
    ActNorm, AffineCouplingBlock, Permute), or in the sampling direction of an all-planar one (Planar, Radial) or of a
    coupled-spline / LU one (CoupledRationalQuadraticSpline, LULinearPermute): the unchanged forward, so values are
    bit-identical with and without grad.  The backward is one nfb_flow_sampling_backward / nfb_flow_density_backward
    call (recompute + walk back through the layers).  Refuses to run the backward if a parameter was modified in place
    after the forward."""

    @staticmethod
    def forward(ctx, handle, layers, direction, z, *params):
        x, ld = handle.transform(direction, z)
        ctx.handle, ctx.layers, ctx.direction, ctx.params = handle, layers, direction, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(require_cuda_f32(z))
        return x, ld

    @staticmethod
    def backward(ctx, g_x, g_ld):
        (z,) = ctx.saved_tensors
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            names = "+".join(sorted({type(l).__name__ for l in ctx.layers}))
            raise RuntimeError(f"{names} backward: a parameter was modified in place after the forward pass")
        gz, gmap = stack_backward(ctx.handle, ctx.layers, ctx.direction, z, g_x, g_ld, ctx.needs_input_grad[3])
        return (None, None, None, gz, *[gmap.get(id(p)) if p.requires_grad else None for p in ctx.params])


def stack_sampling(handle, layers, z, params, direction=L.NFB_FORWARD):
    return StackSamplingFn.apply(handle, list(layers), direction, z, *params)


# ---- element adjoints ------------------------------------------------------------------------------------------
def spline_backward(x, params, shared, num_bins, gy, g_ld, wh_scale, tail_bound=None, num_derivatives=None,
                    tails=None, circular=None, want_params=True):
    """(g_x, g_params) of nfb_rqs_spline (tails=None: scalar tail_bound, linear tails) or nfb_rqs_spline_tails
    (tails = float32 [feats] bounds, circular = int32 [feats] flags).  shared: params is one [feats, P] table."""
    rows, feats = x.shape
    nd = num_bins - 1 if num_derivatives is None else num_derivatives
    P = 2 * num_bins + nd
    gx = torch.empty_like(x)
    gp = torch.empty(params.shape, dtype=torch.float32, device=x.device) if want_params else None
    stride = 0 if shared else feats * P
    with torch.cuda.device(x.device):
        if tails is None:
            L.check(L.lib().nfb_rqs_spline_backward(L.ptr(x), L.ptr(params), stride, L.ptr(gy), L.ptr(g_ld), L.ptr(gx),
                                                    L.ptr(gp), rows, feats, num_bins, C.c_float(tail_bound),
                                                    C.c_float(wh_scale), L.stream_ptr()))
        else:
            L.check(L.lib().nfb_rqs_spline_tails_backward(L.ptr(x), L.ptr(params), stride, L.ptr(gy), L.ptr(g_ld),
                                                          L.ptr(gx), L.ptr(gp), rows, feats, num_bins, nd, L.ptr(tails),
                                                          L.ptr(circular), C.c_float(wh_scale), L.stream_ptr()))
    return gx, gp


def spline_inverse_backward(z, params, shared, num_bins, gx, g_ld, wh_scale, tail_bound=None, num_derivatives=None,
                            tails=None, circular=None, need_z=True):
    """(g_z | None, g_params) of the inverse spline x = g(z) (nfb_rqs_spline(_tails) with inverse = 1) through
    nfb_rqs_spline(_tails)_inverse_backward; arguments as in spline_backward, gx the cotangent of x."""
    rows, feats = z.shape
    gz = torch.empty_like(z) if need_z else None
    gp = torch.empty(params.shape, dtype=torch.float32, device=z.device)
    stride = 0 if shared else feats * (2 * num_bins + (num_bins - 1 if num_derivatives is None else num_derivatives))
    if rows == 0:
        return gz, gp.zero_()
    with torch.cuda.device(z.device):
        if tails is None:
            L.check(L.lib().nfb_rqs_spline_inverse_backward(L.ptr(z), L.ptr(params), stride, L.ptr(gx), L.ptr(g_ld),
                                                            L.ptr(gz), L.ptr(gp), rows, feats, num_bins,
                                                            C.c_float(tail_bound), C.c_float(wh_scale), L.stream_ptr()))
        else:
            L.check(L.lib().nfb_rqs_spline_tails_inverse_backward(L.ptr(z), L.ptr(params), stride, L.ptr(gx),
                                                                  L.ptr(g_ld), L.ptr(gz), L.ptr(gp), rows, feats,
                                                                  num_bins, num_derivatives, L.ptr(tails),
                                                                  L.ptr(circular), C.c_float(wh_scale), L.stream_ptr()))
    return gz, gp


def _resnet_grad_call(net, masked, context):
    """The nfb_resnet_ctx_desc_t of a ResidualNet / MADE and its parameter-gradient outputs, in the slot order of
    nfb_resnet_backward / nfb_maf_inverse_backward: (desc, keepalive, gradient arrays (g_w, g_b, g_w_context,
    g_b_context) as C pointer arrays, {parameter: gradient} of the parameters that require grad)."""
    d = L.ResnetCtxDesc()
    d.net, keep = resnet_desc(net, masked)
    blocks = list(net.blocks)
    nb = len(blocks)
    lin_w = [net.initial_layer.weight] + [l.weight for b in blocks for l in b.linear_layers] + [net.final_layer.weight]
    lin_b = [net.initial_layer.bias] + [l.bias for b in blocks for l in b.linear_layers] + [net.final_layer.bias]
    ctx_w, ctx_b = [], []
    if context is not None:
        own = getattr(net, "context_layer", None)   # MADE: context_layer(context) added to the initial layer
        ctx_w = [own.weight if own is not None else None] + [b.context_layer.weight for b in blocks]
        ctx_b = [own.bias if own is not None else None] + [b.context_layer.bias for b in blocks]
        d.context_features = context.shape[1]
        d.w_context = ctx_w[0].data_ptr() if own is not None else None
        d.b_context = ctx_b[0].data_ptr() if own is not None else None
        wbc, bbc = _vp(ctx_w[1:]), _vp(ctx_b[1:])
        d.w_block_context = C.cast(wbc, C.POINTER(C.c_void_p))
        d.b_block_context = C.cast(bbc, C.POINTER(C.c_void_p))
        keep = (keep, wbc, bbc)
    gw = [_grad_like(p) for p in lin_w]
    gb = [_grad_like(p) for p in lin_b]
    gwc = [_grad_like(p) if p is not None else None for p in ctx_w]
    gbc = [_grad_like(p) if p is not None else None for p in ctx_b]
    arrays = [_vp(gw), _vp(gb), _vp(gwc), _vp(gbc)]
    gmap = {p: g for p, g in zip(lin_w + lin_b + ctx_w + ctx_b, gw + gb + gwc + gbc) if g is not None}
    return d, (keep, arrays), [C.cast(a, C.POINTER(C.c_void_p)) for a in arrays], gmap


def resnet_backward(net, masked, x, context, g_out, need_x=True, need_ctx=True):
    """(g_x, g_context | None, {parameter: gradient}) of a ResidualNet / MADE through nfb_resnet_backward."""
    d, keep, arrays, gmap = _resnet_grad_call(net, masked, context)
    rows = x.shape[0]
    gx = torch.empty_like(x) if need_x else None
    gctx = torch.empty_like(context) if context is not None and need_ctx else None
    lib = L.lib()
    ws = _workspace(lib.nfb_resnet_backward_workspace_bytes(C.byref(d), rows), x.device)
    with torch.cuda.device(x.device):
        L.check(lib.nfb_resnet_backward(C.byref(d), L.ptr(x), L.ptr(context), L.ptr(g_out), rows, L.ptr(ws), ws.numel(),
                                        L.ptr(gx), L.ptr(gctx), *arrays, L.stream_ptr()))
    del keep
    return gx, gctx, gmap


def maf_inverse_backward(made, features, x, y, context, g_y, g_ld, need_x=True, need_ctx=True):
    """(g_x, g_context | None, {parameter: gradient}) of MaskedAffineAutoregressive's density pass y = inverse(x)
    through nfb_maf_inverse_backward (the fixed-point adjoint of the D-pass loop; made = its autoregressive_net)."""
    d, keep, arrays, gmap = _resnet_grad_call(made, True, context)
    rows = x.shape[0]
    gx = torch.empty_like(x) if need_x else None
    gctx = torch.empty_like(context) if context is not None and need_ctx else None
    lib = L.lib()
    ws = _workspace(lib.nfb_maf_inverse_backward_workspace_bytes(C.byref(d), features, rows), x.device)
    with torch.cuda.device(x.device):
        L.check(lib.nfb_maf_inverse_backward(C.byref(d), features, L.ptr(x), L.ptr(y), L.ptr(context), L.ptr(g_y),
                                             L.ptr(g_ld), rows, L.ptr(ws), ws.numel(), L.ptr(gx), L.ptr(gctx), *arrays,
                                             L.stream_ptr()))
    del keep
    return gx, gctx, gmap


def ar_rqs_sampling_backward(made, features, num_bins, num_derivatives, tail_bound, tails, circular, z, x, context,
                             g_x, g_ld, need_z=True, need_ctx=True):
    """(g_z | None, g_context | None, {parameter: gradient}) of an autoregressive spline layer's sampling direction
    x = forward(z, context) through nfb_ar_rqs_sampling_backward (the fixed-point adjoint of the D-pass loop; made = its
    autoregressive_net, whose PeriodicFeaturesElementwise preprocessing, if any, is differentiated in the same call).
    tails / circular None: linear tails with the scalar tail_bound."""
    from .utils.nn import PeriodicFeaturesElementwise
    d, keep, arrays, gmap = _resnet_grad_call(made, True, context)
    rows = z.shape[0]
    pre = made.preprocessing
    if pre is not None and not isinstance(pre, PeriodicFeaturesElementwise):
        raise NotImplementedError("the sampling backward of an autoregressive spline takes PeriodicFeaturesElementwise "
                                  "as its only preprocessing")
    slot = w = scale = bias = g_pw = g_pb = None
    n_periodic = 0
    if pre is not None:
        slot, w, scale, bias = pre._tables(z.device)
        n_periodic = len(pre.ind)
        g_pw = _grad_like(pre.weights)
        g_pb = _grad_like(pre.bias) if pre.apply_bias else None
        gmap.update({p: g for p, g in ((pre.weights, g_pw), (getattr(pre, "bias", None), g_pb)) if g is not None})
    gz = torch.empty_like(z) if need_z else None
    gctx = torch.empty_like(context) if context is not None and need_ctx else None
    lib = L.lib()
    ws = _workspace(lib.nfb_ar_rqs_sampling_backward_workspace_bytes(C.byref(d), features, num_bins, num_derivatives,
                                                                     rows), z.device)
    with torch.cuda.device(z.device):
        L.check(lib.nfb_ar_rqs_sampling_backward(C.byref(d), features, num_bins, num_derivatives,
                                                 C.c_float(tail_bound if tails is None else 0.0), L.ptr(tails),
                                                 L.ptr(circular), L.ptr(slot), L.ptr(w), L.ptr(scale), L.ptr(bias),
                                                 n_periodic, L.ptr(z), L.ptr(x), L.ptr(context), L.ptr(g_x), L.ptr(g_ld),
                                                 rows, L.ptr(ws), ws.numel(), L.ptr(gz), L.ptr(gctx), *arrays, L.ptr(g_pw),
                                                 L.ptr(g_pb), L.stream_ptr()))
    del keep
    return gz, gctx, gmap


def mlp_backward(mlp, x, g_out, need_x=True):
    d = mlp_desc(mlp)
    lins = mlp.linear_layers()
    gw = [_grad_like(l.weight) for l in lins]
    gb = [_grad_like(l.bias) for l in lins]
    gx = torch.empty_like(x) if need_x else None
    lib = L.lib()
    ws = _workspace(lib.nfb_mlp_backward_workspace_bytes(C.byref(d), x.shape[0]), x.device)
    pw, pb = _vp(gw), _vp(gb)
    with torch.cuda.device(x.device):
        L.check(lib.nfb_mlp_backward(C.byref(d), L.ptr(x), L.ptr(g_out), x.shape[0], L.ptr(ws), ws.numel(), L.ptr(gx),
                                     C.cast(pw, C.POINTER(C.c_void_p)), C.cast(pb, C.POINTER(C.c_void_p)),
                                     L.stream_ptr()))
    ps = [l.weight for l in lins] + [l.bias for l in lins]
    return gx, {p: g for p, g in zip(ps, gw + gb) if g is not None}


def periodic_backward(pf, x, g_y):
    slot, w, scale, bias = pf._tables(x.device)
    gx = torch.empty_like(x)
    gw = torch.empty_like(pf.weights)
    gb = torch.empty_like(pf.bias) if pf.apply_bias else None
    with torch.cuda.device(x.device):
        L.check(L.lib().nfb_periodic_features_backward(L.ptr(x), L.ptr(g_y), x.shape[0], x.shape[1], L.ptr(slot),
                                                       L.ptr(w), L.ptr(scale), len(pf.ind), L.ptr(gx), L.ptr(gw),
                                                       L.ptr(gb), L.stream_ptr()))
    gmap = {pf.weights: gw}
    if gb is not None:
        gmap[pf.bias] = gb
    return gx, gmap


def conditioner_backward(net, masked, x, context, g_out, need_x=True, need_ctx=True):
    """ResidualNet / MADE with its optional preprocessing module in front: PeriodicFeaturesElementwise through its
    adjoint kernel, any other module differentiated by torch autograd."""
    from .nets.resnet import _preprocess
    from .utils.nn import PeriodicFeaturesElementwise
    pre = net.preprocessing
    xin = _preprocess(pre, x) if pre is not None else x
    need_in = need_x or (pre is not None and any(p.requires_grad for p in pre.parameters()))
    gx, gctx, gmap = resnet_backward(net, masked, require_cuda_f32(xin), context, g_out, need_in, need_ctx)
    if gx is None:
        return gx, gctx, gmap
    if isinstance(pre, PeriodicFeaturesElementwise):
        gx, gm = periodic_backward(pre, x, gx)
        gmap.update(gm)
    elif pre is not None:
        params = [p for p in pre.parameters() if p.requires_grad]
        with torch.enable_grad():
            xx = x.detach().requires_grad_(True)
            grads = torch.autograd.grad(pre(xx), [xx] + params, gx, allow_unused=True)
        gx = grads[0]
        gmap.update({p: g for p, g in zip(params, grads[1:]) if g is not None})
    return gx, gctx, gmap


class UnitGaussianFn(torch.autograd.Function):
    """log N(u; 0, I) per row (nfb_diag_gaussian_log_prob with zero tables) and its adjoint
    (nfb_gaussian_table_log_prob_backward): the density of ConditionalDiagGaussian on the standardised residual."""

    @staticmethod
    def forward(ctx, u):
        zeros = torch.zeros(u.shape[1], device=u.device)
        out = torch.empty(u.shape[0], dtype=torch.float32, device=u.device)
        if u.shape[0]:
            with torch.cuda.device(u.device):
                L.check(L.lib().nfb_diag_gaussian_log_prob(L.ptr(u), L.ptr(zeros), L.ptr(zeros), L.ptr(out), u.shape[0],
                                                           u.shape[1], 0, L.stream_ptr()))
        ctx.save_for_backward(u)
        return out

    @staticmethod
    def backward(ctx, g):
        (u,) = ctx.saved_tensors
        zeros = torch.zeros(u.shape[1], device=u.device)
        gu = torch.empty_like(u)
        if u.shape[0]:
            with torch.cuda.device(u.device):
                L.check(L.lib().nfb_gaussian_table_log_prob_backward(L.ptr(u), None, L.ptr(zeros), L.ptr(zeros),
                                                                     L.ptr(g.contiguous()), L.ptr(gu), None, None,
                                                                     u.shape[0], u.shape[1], 1, 1, L.stream_ptr()))
        return gu


class MixtureLogProbFn(torch.autograd.Function):
    """GaussianMixture.log_prob(z) per row (nfb_gaussian_mixture_log_prob) and its adjoint to z, loc, log_scale and
    weight_scores (nfb_gaussian_mixture_log_prob_backward: deterministic, two launches)."""

    @staticmethod
    def forward(ctx, z, loc, log_scale, weight_scores):
        K, D = weight_scores.shape[-1], z.shape[1]
        out = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        if z.shape[0]:
            with torch.cuda.device(z.device):
                L.check(L.lib().nfb_gaussian_mixture_log_prob(L.ptr(z), L.ptr(loc), L.ptr(log_scale),
                                                              L.ptr(weight_scores), L.ptr(out), z.shape[0], K, D, 0,
                                                              L.stream_ptr()))
        ctx.save_for_backward(z, loc, log_scale, weight_scores)
        return out

    @staticmethod
    def backward(ctx, g):
        z, loc, log_scale, weight_scores = ctx.saved_tensors
        K, D, rows = weight_scores.shape[-1], z.shape[1], z.shape[0]
        lib = L.lib()
        outs = [torch.empty_like(t) if need else None
                for t, need in zip((z, loc, log_scale, weight_scores), ctx.needs_input_grad)]
        ws = torch.empty(max(1, lib.nfb_gaussian_mixture_log_prob_backward_workspace_bytes(rows, K, D)),
                         dtype=torch.uint8, device=z.device)
        with torch.cuda.device(z.device):
            L.check(lib.nfb_gaussian_mixture_log_prob_backward(
                L.ptr(z), L.ptr(loc), L.ptr(log_scale), L.ptr(weight_scores), L.ptr(g.contiguous()), rows, K, D,
                L.ptr(ws), ws.numel(), *[L.ptr(o) for o in outs], L.stream_ptr()))
        return tuple(outs)
