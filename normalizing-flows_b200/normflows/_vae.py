"""Gradients of the flow-VAE's encoders and decoders (distributions/encoder.py, distributions/decoder.py): one
autograd.Function per kernel pair of csrc/nfb_vae.cu.

Each forward is the call the no-grad path makes (values are bit-identical with and without grad); each backward is one
adjoint launch with fixed-order sums, so two runs give identical gradients.  The inputs the backward reads are saved
with save_for_backward, so an in-place change to one of them (an optimizer step on ConstDiagGaussian's loc / scale, a
write into a net output) between forward and backward makes autograd refuse the backward.

A diagonal Gaussian's parameters come either from a net output [rows, n] (mean in columns [0, n // 2), log variance in
[n // 2, 2 (n // 2)): NNDiagGaussian, NNDiagGaussianDecoder), read in place with row stride n, or from broadcast
`loc` / `scale` parameters (ConstDiagGaussian), read with row stride 0."""
import torch

from . import _lib as L
from ._native import require_cuda_f32


def _params(net, loc, scale):
    """(mean view, scale-column view, row stride, d, scale kind) of a net output or of (loc, scale)."""
    if net is not None:
        d = net.shape[1] // 2
        return net, net[:, d:], net.shape[1], d, L.NFB_VAE_LOGVAR
    return loc, scale, 0, loc.numel(), L.NFB_VAE_SCALE


def _param_grads(net, loc, scale, need):
    """Gradient buffers in the parameters' layout, and the (mean, scale column) views the kernels write."""
    if net is not None:
        if not need[0]:
            return (None, None, None), (None, None)
        g = torch.zeros_like(net) if net.shape[1] % 2 else torch.empty_like(net)
        return (g, None, None), (g, g[:, net.shape[1] // 2:])
    gl = torch.empty_like(loc) if need[1] else None
    gs = torch.empty_like(scale) if need[2] else None
    return (None, gl, gs), (gl, gs)


def _width(net, loc, scale):
    """The feature count d of the Gaussian's parameter rows (checked: the kernels take it as the row stride of the data
    they pair with those rows)."""
    if net is not None:
        if net.dim() != 2 or net.shape[1] < 2:
            raise ValueError(f"net output of shape {tuple(net.shape)}: expected [rows, 2 d] with d >= 1")
        return net.shape[1] // 2
    if loc.numel() != scale.numel() or loc.numel() < 1:
        raise ValueError(f"loc has {loc.numel()} entries and scale {scale.numel()}: expected the same d >= 1")
    return loc.numel()


def _check_rows(what, t, rows, div):
    """t holds one row per `div` consecutive rows of the `rows` the kernel walks."""
    need = -(-rows // div)
    if t.shape[0] != need:
        raise ValueError(f"{what} has {t.shape[0]} rows; {rows} rows in groups of {div} need {need}")


def _inputs(net, loc, scale):
    if net is not None:
        return require_cuda_f32(net, "encoder / decoder net output"), None, None
    return None, require_cuda_f32(loc, "loc"), require_cuda_f32(scale, "scale")


class ReparamFn(torch.autograd.Function):
    """(z [B, S, d], log_q [B, S]) of the reparameterised draw z = mean[b] + sd[b] eps[b, s] (nfb_vae_reparam_sample)
    and its adjoint to the net output or to loc / scale (nfb_vae_reparam_sample_backward: sums over S, or over B S for
    the shared loc / scale)."""

    @staticmethod
    def forward(ctx, eps, net, loc, scale):
        ctx.set_materialize_grads(False)
        mean, sc, stride, d, kind = _params(net, loc, scale)
        B, S = eps.shape[0], eps.shape[1]
        z = torch.empty(B, S, d, dtype=torch.float32, device=eps.device)
        log_q = torch.empty(B, S, dtype=torch.float32, device=eps.device)
        with torch.cuda.device(eps.device):
            L.check(L.lib().nfb_vae_reparam_sample(L.ptr(mean), L.ptr(sc), stride, kind, L.ptr(eps), B, S, d, L.ptr(z),
                                                   L.ptr(log_q), L.stream_ptr()))
        ctx.save_for_backward(eps, net, loc, scale)
        return z, log_q

    @staticmethod
    def backward(ctx, g_z, g_lq):
        eps, net, loc, scale = ctx.saved_tensors
        mean, sc, stride, d, kind = _params(net, loc, scale)
        outs, (gm, gs) = _param_grads(net, loc, scale, ctx.needs_input_grad[1:])
        B, S = eps.shape[0], eps.shape[1]
        g_z = g_z.contiguous() if g_z is not None else None
        g_lq = g_lq.contiguous() if g_lq is not None else None
        if gm is not None or gs is not None:
            with torch.cuda.device(eps.device):
                L.check(L.lib().nfb_vae_reparam_sample_backward(L.ptr(mean), L.ptr(sc), stride, kind, L.ptr(eps),
                                                                L.ptr(g_z), L.ptr(g_lq), B, S, d, L.ptr(gm), L.ptr(gs),
                                                                L.stream_ptr()))
        return (None, *outs)


def reparam_sample(eps, net=None, loc=None, scale=None):
    d = _width(net, loc, scale)
    if eps.dim() != 3 or eps.shape[2] != d:
        raise ValueError(f"eps of shape {tuple(eps.shape)} for {d} latent features: expected [B, S, {d}]")
    if net is not None:
        _check_rows("the net output", net, eps.shape[0], 1)
    eps = require_cuda_f32(eps, "eps")
    return ReparamFn.apply(eps, *_inputs(net, loc, scale))


class GaussianLogProbFn(torch.autograd.Function):
    """out[r] = log N(v[r // v_div]; mean[r // p_div], sd[r // p_div]^2) with the normalising constant of `norm_dim`
    features (nfb_vae_gaussian_log_prob), and its adjoint (nfb_vae_gaussian_log_prob_backward: g_v summed over the rows
    that share a value row, the parameters' gradient summed over the rows that share a parameter row)."""

    @staticmethod
    def forward(ctx, rows, v_div, p_div, norm_dim, v, net, loc, scale):
        mean, sc, stride, d, kind = _params(net, loc, scale)
        out = torch.empty(rows, dtype=torch.float32, device=v.device)
        with torch.cuda.device(v.device):
            L.check(L.lib().nfb_vae_gaussian_log_prob(L.ptr(v), L.ptr(mean), L.ptr(sc), stride, kind, rows, d, v_div,
                                                      p_div, float(norm_dim), L.ptr(out), L.stream_ptr()))
        ctx.shape = (rows, v_div, p_div)
        ctx.save_for_backward(v, net, loc, scale)
        return out

    @staticmethod
    def backward(ctx, g):
        v, net, loc, scale = ctx.saved_tensors
        rows, v_div, p_div = ctx.shape
        mean, sc, stride, d, kind = _params(net, loc, scale)
        outs, (gm, gs) = _param_grads(net, loc, scale, ctx.needs_input_grad[5:])
        gv = torch.empty_like(v) if ctx.needs_input_grad[4] else None
        with torch.cuda.device(v.device):
            L.check(L.lib().nfb_vae_gaussian_log_prob_backward(L.ptr(v), L.ptr(mean), L.ptr(sc), stride, kind,
                                                               L.ptr(g.contiguous()), rows, d, v_div, p_div, L.ptr(gv),
                                                               L.ptr(gm), L.ptr(gs), L.stream_ptr()))
        return (None, None, None, None, gv, *outs)


def gaussian_log_prob(v, rows, v_div, p_div, norm_dim, net=None, loc=None, scale=None):
    d = _width(net, loc, scale)
    if v.dim() != 2 or v.shape[1] != d:
        raise ValueError(f"values of shape {tuple(v.shape)} for a Gaussian over {d} features: expected [rows, {d}]")
    _check_rows("the value tensor", v, rows, v_div)
    if net is not None:
        _check_rows("the net output", net, rows, p_div)
    v = require_cuda_f32(v)
    return GaussianLogProbFn.apply(rows, v_div, p_div, norm_dim, v, *_inputs(net, loc, scale))


class BernoulliLogProbFn(torch.autograd.Function):
    """out[r] = sum_j x log_sig(s) + (1 - x) log_sig(-s) with x row r // x_div (nfb_bernoulli_log_prob), and its adjoint
    to the scores and, when x requires grad, to x summed over the rows that share it."""

    @staticmethod
    def forward(ctx, score, x, x_div):
        out = torch.empty(score.shape[0], dtype=torch.float32, device=score.device)
        with torch.cuda.device(score.device):
            L.check(L.lib().nfb_bernoulli_log_prob(L.ptr(score), L.ptr(x), score.shape[0], score.shape[1], x_div,
                                                   L.ptr(out), L.stream_ptr()))
        ctx.x_div = x_div
        ctx.save_for_backward(score, x)
        return out

    @staticmethod
    def backward(ctx, g):
        score, x = ctx.saved_tensors
        gs = torch.empty_like(score) if ctx.needs_input_grad[0] else None
        gx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        if score.shape[0] == 0 and gx is not None:
            gx.zero_()
        with torch.cuda.device(score.device):
            L.check(L.lib().nfb_bernoulli_log_prob_backward(L.ptr(score), L.ptr(x), L.ptr(g.contiguous()),
                                                            score.shape[0], score.shape[1], ctx.x_div, L.ptr(gs),
                                                            L.ptr(gx), L.stream_ptr()))
        return gs, gx, None


def bernoulli_log_prob(score, x, x_div):
    if score.dim() != 2 or x.dim() != 2 or x.shape[1] != score.shape[1]:
        raise ValueError(f"data of shape {tuple(x.shape)} for scores of shape {tuple(score.shape)}: the widths differ")
    _check_rows("the data", x, score.shape[0], x_div)
    return BernoulliLogProbFn.apply(require_cuda_f32(score, "score"), require_cuda_f32(x, "x"), x_div)


class SigmoidFn(torch.autograd.Function):
    """sigmoid elementwise (nfb_sigmoid) and its adjoint g y (1 - y) (nfb_sigmoid_backward)."""

    @staticmethod
    def forward(ctx, s):
        y = torch.empty_like(s)
        with torch.cuda.device(s.device):
            L.check(L.lib().nfb_sigmoid(L.ptr(s), L.ptr(y), s.numel(), L.stream_ptr()))
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, g):
        (y,) = ctx.saved_tensors
        gs = torch.empty_like(y)
        with torch.cuda.device(y.device):
            L.check(L.lib().nfb_sigmoid_backward(L.ptr(y), L.ptr(g.contiguous()), L.ptr(gs), y.numel(),
                                                 L.stream_ptr()))
        return gs


def sigmoid(s):
    return SigmoidFn.apply(require_cuda_f32(s))
