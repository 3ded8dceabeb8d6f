"""Training pass of the image path (Glow, `MultiscaleFlow.forward_kld(x, y).backward()`, examples/glow.ipynb cell 4).

One `autograd.Function` per call the library already makes -- GlowBlock.inverse, Squeeze, the channel split, the base
densities and the Logit transform -- so that MultiscaleFlow.log_prob composes them unchanged.  Each forward runs exactly
the no-grad code path (same kernels, bit-identical values); each backward runs the adjoint kernels of the C ABI
(include/nfb200.h "training pass of the image path").  Activations are recomputed in backward, not stored: a Glow
block keeps only its input.  The small C x C parameter preparations (the folded ActNorm + Invertible1x1Conv, the folded
ActNorm of ConvNet2d(actnorm=True), the GlowBase tables) are mapped back to the parameters with torch autograd over a
differentiable restatement of the fold."""
import torch

from . import _lib as L


def wants_grad(module, *tensors):
    """Grad enabled, and an input or a parameter of the module requires grad: the module's call goes through its
    autograd.Function (NormalizingFlow.log_prob uses the same test)."""
    if not torch.is_grad_enabled():
        return False
    return any(t is not None and t.requires_grad for t in tensors) or any(p.requires_grad for p in module.parameters())


def _zeros_if_none(g, like):
    return torch.zeros_like(like) if g is None else g.contiguous()


def _param_grads(params, grads):
    return [grads.get(id(p)) if p.requires_grad else None for p in params]


class GlowBlockInverseFn(torch.autograd.Function):
    """(z_out, log_det) = block.inverse(z); backward: GlowBlock._inverse_backward (recompute + adjoint kernels)."""

    @staticmethod
    def forward(ctx, block, z, *params):
        out, ld = block._inverse_native(z)   # (a pending ActNorm init changes parameters here, before the versions)
        ctx.block, ctx.params = block, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(z)
        return out, ld

    @staticmethod
    def backward(ctx, g_out, g_ld):
        (z,) = ctx.saved_tensors
        # backward recomputes from the module's parameters: like torch's saved-tensor check, refuse if they changed
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError("GlowBlock backward: a parameter of the block was modified in place after the forward pass "
                               "(the recompute would differentiate other weights than the forward used)")
        g_out = _zeros_if_none(g_out, z)
        g_ld = _zeros_if_none(g_ld, z.new_empty(z.shape[0]))
        gz, grads = ctx.block._inverse_backward(z, g_out, g_ld)
        return (None, gz, *_param_grads(ctx.params, grads))


class SqueezeFn(torch.autograd.Function):
    """Squeeze is a permutation: its adjoint is nfb_squeeze in the other direction."""

    @staticmethod
    def forward(ctx, layer, z, direction):
        ctx.layer, ctx.direction = layer, direction
        out, _ = layer._run(z, direction)
        return out

    @staticmethod
    def backward(ctx, g):
        other = L.NFB_FORWARD if ctx.direction == L.NFB_INVERSE else L.NFB_INVERSE
        gz, _ = ctx.layer._run(g.contiguous(), other)
        return None, gz, None


class SplitChannelsFn(torch.autograd.Function):
    """split_channels: the adjoint pastes both chunks back (nfb_paste_channels)."""

    @staticmethod
    def forward(ctx, z, mode):
        from .flows.glow import split_channels
        ctx.mode, ctx.shape = mode, z.shape
        return split_channels(z, mode)

    @staticmethod
    def backward(ctx, g1, g2):
        from .flows.glow import merge_channels
        B, C, H, W = ctx.shape
        h = (C + 1) // 2
        a, b = (h, C - h) if ctx.mode == "channel" else (C - h, h)   # channel counts of the returned pair
        dev = g1.device if g1 is not None else g2.device
        g1 = g1.contiguous() if g1 is not None else torch.zeros(B, a, H, W, device=dev)
        g2 = g2.contiguous() if g2 is not None else torch.zeros(B, b, H, W, device=dev)
        return merge_channels(g1, g2, ctx.mode), None


class GaussianTableFn(torch.autograd.Function):
    """gaussian_table_log_prob with gradients: the forward runs the no-grad path on the same tables; backward is
    nfb_gaussian_table_log_prob_backward.  y: empty = one table column."""

    @staticmethod
    def forward(ctx, z, loc, log_scale, y, group):
        out = gaussian_table_log_prob(z, loc, log_scale, y if y.numel() else None, group)
        ctx.group = group
        ctx.save_for_backward(z, loc, log_scale, y)
        return out

    @staticmethod
    def backward(ctx, g):
        z, loc, ls, y = ctx.saved_tensors
        B = z.shape[0]
        dim = z.numel() // max(B, 1)
        ncls = loc.shape[1]
        gz = torch.empty_like(z) if ctx.needs_input_grad[0] else None
        gl = torch.empty(loc.shape, device=z.device) if ctx.needs_input_grad[1] else None   # contiguous [E, K]
        gs = torch.empty(ls.shape, device=z.device) if ctx.needs_input_grad[2] else None
        # contiguous copies held by name: a temporary freed inside the call could hand its memory to the next one
        loc, ls, g = loc.contiguous(), ls.contiguous(), g.contiguous().float()
        with torch.cuda.device(z.device):
            L.check(L.lib().nfb_gaussian_table_log_prob_backward(
                L.ptr(z), L.ptr(y if y.numel() else None), L.ptr(loc), L.ptr(ls), L.ptr(g), L.ptr(gz), L.ptr(gl),
                L.ptr(gs), B, dim, ctx.group, ncls, L.stream_ptr()))
        return gz, gl, gs, None, None


def gaussian_table_log_prob(z, loc, log_scale, y, group):
    """log_q[b] of a diagonal Gaussian whose element i of a sample uses entry i // group of the tables
    loc / log_scale [E, K], column y[b] (y None: K = 1).  The density kernel (nfb_diag_gaussian_log_prob for K = 1,
    nfb_class_cond_diag_gaussian_log_prob otherwise) reads one entry per element, so tables with group > 1 are expanded
    first; through GaussianTableFn when a gradient is wanted."""
    if torch.is_grad_enabled() and any(t.requires_grad for t in (z, loc, log_scale)) and z.shape[0]:
        yy = y if y is not None else torch.empty(0, dtype=torch.int64, device=z.device)
        return GaussianTableFn.apply(z, loc, log_scale, yy, group)
    B, K = z.shape[0], loc.shape[1]
    if group > 1:
        loc, log_scale = loc.repeat_interleave(group, dim=0), log_scale.repeat_interleave(group, dim=0)
    loc, log_scale = loc.detach().contiguous(), log_scale.detach().contiguous()   # held by name until the kernel has run
    out = torch.empty(B, dtype=torch.float32, device=z.device)
    if B:
        with torch.cuda.device(z.device):
            if K == 1:
                L.check(L.lib().nfb_diag_gaussian_log_prob(L.ptr(z), L.ptr(loc), L.ptr(log_scale), L.ptr(out), B,
                                                           loc.shape[0], 0, L.stream_ptr()))
            else:
                L.check(L.lib().nfb_class_cond_diag_gaussian_log_prob(L.ptr(z), L.ptr(y), L.ptr(loc), L.ptr(log_scale),
                                                                      L.ptr(out), B, loc.shape[0], K, 0, L.stream_ptr()))
    return out


class LogitInverseFn(torch.autograd.Function):
    """(y, log_det) = Logit.inverse(x); backward: nfb_logit_transform_backward."""

    @staticmethod
    def forward(ctx, layer, x):
        ctx.alpha = float(layer.alpha)
        ctx.save_for_backward(x)
        return layer._run(x, L.NFB_INVERSE)

    @staticmethod
    def backward(ctx, g_out, g_ld):
        (x,) = ctx.saved_tensors
        gx = torch.empty_like(x)
        B = x.shape[0]
        g_out = g_out.contiguous() if g_out is not None else None   # held by name until the kernel has run
        g_ld = g_ld.contiguous() if g_ld is not None else None
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_logit_transform_backward(L.ptr(x), L.ptr(g_out), L.ptr(g_ld), L.ptr(gx), B,
                                                         x.numel() // max(B, 1), ctx.alpha, L.stream_ptr()))
        return None, gx
