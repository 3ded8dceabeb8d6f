"""Glow building blocks on NCHW tensors (reference: normflows/flows/affine/glow.py:11-84,
flows/mixing.py:57-133 Invertible1x1Conv, flows/reshape.py:9-128 Split/Merge/Squeeze).

Both directions run on the CUDA path: ActNorm and Invertible1x1Conv are folded into one 1x1 convolution
(density: W then exp(-s); sampling: the double-precision inverse of W, then exp(s)), the ConvNet2d conditioner
runs on the tensor core (csrc/nfb_conv_tc.cu) and the coupling epilogue, Squeeze and channel split/merge are
kernels in csrc/nfb_glow.cu."""
import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .._image_autograd import GlowBlockInverseFn, SplitChannelsFn, SqueezeFn, wants_grad
from .._native import cached, require_cuda_f32
from ..nets.cnn import ConvNet2d
from .affine import _MAPS, ActNorm, AffineCoupling, Merge, Split
from .base import Flow


def _pointwise(x, w, b, out):
    """out = w x + b at every pixel of the NCHW tensor x: the folded 1x1 convolution, C -> C channels."""
    B, C, H, W = x.shape
    L.check(L.lib().nfb_conv2d(L.ptr(x), C, 0, L.ptr(w), L.ptr(b), L.ptr(out), B, C, H, W, C, 1, -1.0, L.stream_ptr()))


class Invertible1x1Conv(Flow):
    """Same parameters/buffers as the reference (mixing.py:63-86), both parameterisations: LU (P, L, U, sign_S, log_S)
    or the plain matrix W (`use_lu=False`, :85-86).  The 1x1 convolution itself runs in csrc/nfb_glow.cu; the small
    C x C parameter preparation (assembling W, the double-precision inverse of :94-101 / :110-114, slogdet of
    :117,129) is folded once per parameter version."""

    def __init__(self, num_channels, use_lu=False):
        super().__init__()
        self.num_channels, self.use_lu = num_channels, use_lu
        Q, _ = torch.linalg.qr(torch.randn(num_channels, num_channels))
        if use_lu:
            P, Lm, U = torch.linalg.lu(Q)
            self.register_buffer("P", P)
            self.L = nn.Parameter(Lm)
            S = U.diag()
            self.register_buffer("sign_S", torch.sign(S))
            self.log_S = nn.Parameter(torch.log(torch.abs(S)))
            self.U = nn.Parameter(torch.triu(U, diagonal=1))
            self.register_buffer("eye", torch.diag(torch.ones(num_channels)))
        else:
            self.W = nn.Parameter(Q)

    def _sources(self):
        return (self.P, self.L, self.U, self.sign_S, self.log_S) if self.use_lu else (self.W,)

    def folded(self, direction, s, t, hw, dev):
        """(w [C, C], b [C], logdet constant) of this layer fused with an ActNorm(s, t) on the channel axis:
        density (NFB_INVERSE): ActNorm.inverse then conv with W;  sampling: conv with W^-1 then ActNorm.forward."""
        C = self.num_channels
        if self.use_lu:
            fn = (L.lib().nfb_glow_fold_actnorm_conv1x1 if direction == L.NFB_INVERSE
                  else L.lib().nfb_glow_fold_conv1x1_actnorm_forward)
            w, b, ldc = torch.empty(C, C, device=dev), torch.empty(C, device=dev), torch.empty((), device=dev)
            with torch.cuda.device(dev):
                L.check(fn(L.ptr(self.P), L.ptr(self.L), L.ptr(self.U), L.ptr(self.sign_S), L.ptr(self.log_S),
                           L.ptr(s), L.ptr(t), C, hw, L.ptr(w), L.ptr(b), L.ptr(ldc), L.stream_ptr()))
            return w, b, ldc
        with torch.no_grad():  # plain-matrix parameterisation: C x C parameter preparation in torch (like the reference)
            W = self.W.detach()
            sv, tv = s.detach().reshape(-1), t.detach().reshape(-1)
            logabsdet = torch.linalg.slogdet(W.double())[1]
            if direction == L.NFB_INVERSE:
                w = (W * torch.exp(-sv)[None, :]).contiguous()
                b = -(w @ tv)
                ldc = (hw * (logabsdet - sv.double().sum())).float()
            else:
                w = (torch.exp(sv)[:, None] * torch.inverse(W.double()).float()).contiguous()
                b = tv.clone()
                ldc = (hw * (sv.double().sum() - logabsdet)).float()
        return w, b.contiguous(), ldc

    def folded_torch(self, s, t, hw):
        """Differentiable restatement of `folded(NFB_INVERSE, s, t, hw)` (the gradient chain of the training pass)."""
        sv, tv = s.reshape(-1), t.reshape(-1)
        if self.use_lu:
            lo = torch.tril(self.L, -1) + self.eye
            up = torch.triu(self.U, 1) + torch.diag(self.sign_S * torch.exp(self.log_S))
            Wm, logabsdet = self.P @ lo @ up, self.log_S.sum()
        else:
            Wm, logabsdet = self.W, torch.linalg.slogdet(self.W)[1]
        w = Wm * torch.exp(-sv)[None, :]
        return w, -(w @ tv), hw * (logabsdet - sv.sum())

    def _conv1x1(self, z, direction):
        z = require_cuda_f32(z)
        if z.dim() != 4 or z.shape[1] != self.num_channels:
            raise ValueError("Expected an NCHW tensor with {} channels.".format(self.num_channels))
        B, C, H, W = z.shape
        zero = torch.zeros(C, device=z.device)
        w, b, ldc = self.folded(direction, zero, zero, H * W, z.device)
        out = torch.empty_like(z)
        if B:
            with torch.cuda.device(z.device):
                _pointwise(z, w, b, out)
        return out, ldc  # 0-dim log-det like the reference (broadcasts in log_q += log_det)

    def forward(self, z):
        return self._conv1x1(z, L.NFB_FORWARD)

    def inverse(self, z):
        return self._conv1x1(z, L.NFB_INVERSE)


class Squeeze(Flow):
    def _run(self, z, direction):
        z = require_cuda_f32(z)
        B, C, H, W = z.shape
        if direction == L.NFB_INVERSE:
            out = torch.empty(B, 4 * C, H // 2, W // 2, device=z.device, dtype=z.dtype)
            big = (C, H, W)
        else:
            out = torch.empty(B, C // 4, 2 * H, 2 * W, device=z.device, dtype=z.dtype)
            big = (C // 4, 2 * H, 2 * W)
        if z.numel():
            with torch.cuda.device(z.device):
                L.check(L.lib().nfb_squeeze(L.ptr(z), L.ptr(out), B, big[0], big[1], big[2], direction,
                                            L.stream_ptr()))
        return out, 0

    def forward(self, z):
        return self._run(z, L.NFB_FORWARD)

    def inverse(self, z):
        if wants_grad(self, z):
            return SqueezeFn.apply(self, z, L.NFB_INVERSE), 0
        return self._run(z, L.NFB_INVERSE)


def split_channels(z, mode="channel"):
    """Split.forward (reshape.py:27-31): contiguous copies of the two channel chunks."""
    if torch.is_grad_enabled() and z.requires_grad:
        return SplitChannelsFn.apply(z, mode)
    z = require_cuda_f32(z)
    B, C, H, W = z.shape
    h = (C + 1) // 2
    a = torch.empty(B, h, H, W, device=z.device, dtype=z.dtype)
    b = torch.empty(B, C - h, H, W, device=z.device, dtype=z.dtype)
    if z.numel():
        with torch.cuda.device(z.device):
            L.check(L.lib().nfb_copy_channels(L.ptr(z), L.ptr(a), B, C, 0, h, H * W, L.stream_ptr()))
            L.check(L.lib().nfb_copy_channels(L.ptr(z), L.ptr(b), B, C, h, C - h, H * W, L.stream_ptr()))
    return (a, b) if mode == "channel" else (b, a)


def merge_channels(z1, z2, mode="channel"):
    """Merge.forward (reshape.py:68-74): concatenate two channel chunks."""
    z1, z2 = require_cuda_f32(z1), require_cuda_f32(z2)
    a, b = (z1, z2) if mode == "channel" else (z2, z1)
    B, ca, H, W = a.shape
    cb = b.shape[1]
    out = torch.empty(B, ca + cb, H, W, device=a.device, dtype=a.dtype)
    if out.numel():
        with torch.cuda.device(a.device):
            L.check(L.lib().nfb_paste_channels(L.ptr(a), L.ptr(out), B, ca + cb, 0, ca, H * W, L.stream_ptr()))
            L.check(L.lib().nfb_paste_channels(L.ptr(b), L.ptr(out), B, ca + cb, ca, cb, H * W, L.stream_ptr()))
    return out


class ImageMerge(Merge):
    """Merge for the multiscale driver: `inverse` splits channels (core.py:607-609), `forward` joins them."""

    def forward(self, z):
        z1, z2 = z
        return merge_channels(z1, z2, self.mode), 0

    def inverse(self, z):
        z1, z2 = split_channels(z, self.mode)
        return [z1, z2], 0


class GlowBlock(Flow):
    """[AffineCouplingBlock(ConvNet2d), Invertible1x1Conv(LU), ActNorm] -- module tree as in the reference
    (glow.py:48-70) so checkpoints load verbatim."""

    def __init__(self, channels, hidden_channels, scale=True, scale_map="sigmoid", split_mode="channel",
                 leaky=0.0, init_zeros=True, use_lu=True, net_actnorm=False):
        super().__init__()
        if scale_map not in _MAPS:
            raise NotImplementedError("This scale map is not implemented.")
        if split_mode not in ("channel", "channel_inv"):
            raise NotImplementedError("Mode " + split_mode + " is not implemented.")
        if channels < 2:
            raise NotImplementedError("GlowBlock with a single channel is not on the CUDA path")
        h = (channels + 1) // 2
        # the conditioner reads channels [c0, c0 + cin); the coupling transforms the other ones
        self._c0, self._cin = (0, h) if split_mode == "channel" else (h, channels - h)
        param_map = ConvNet2d((self._cin, hidden_channels, hidden_channels, (2 if scale else 1) * (channels - self._cin)),
                              (3, 1, 3), leaky, init_zeros, actnorm=net_actnorm)
        block = Flow()
        block.flows = nn.ModuleList([Split(split_mode), AffineCoupling(param_map, scale, scale_map),
                                     Merge(split_mode)])
        self.flows = nn.ModuleList([block, Invertible1x1Conv(channels, use_lu), ActNorm((channels, 1, 1))])
        self.channels, self.scale, self.scale_map, self.split_mode = channels, scale, scale_map, split_mode
        # (scale, scale map, split mode) enums of the coupling kernels
        self._modes = (int(bool(scale)), _MAPS[scale_map], 0 if split_mode == "channel" else 1)

    def _param_map(self):
        return self.flows[0].flows[1].param_map

    def _folded(self, direction, hw, dev):
        """Folded 1x1 convolution (weights, bias, per-sample log-det constant) of ActNorm + Invertible1x1Conv for
        one direction, rebuilt when one of the parameters changes, not on every call."""
        conv, an = self.flows[1], self.flows[2]
        return cached(self, "_nfb_fold_fwd" if direction == L.NFB_FORWARD else "_nfb_fold",
                      conv._sources() + (an.s, an.t), (hw, dev), lambda: conv.folded(direction, an.s, an.t, hw, dev))

    def _one_call(self, z, out, scratch, ld, w, b, ldc, direction):
        """The whole block through nfb_glow_block (one C-ABI call: folded 1x1 convolution, fused conditioner, tap-form
        coupling) when the conditioner has the Glow shape and the sample fits the tap-form coupling; False = not
        applicable, the caller takes the step-by-step path."""
        B, C, H, W = z.shape
        pm = self._param_map()
        if not (pm.glow_shape(self._cin) and L.lib().nfb_affine_coupling_image_taps_supported(C, H, W, self._modes[0])):
            return False
        c1, c2, c3 = pm.conv_layers()
        with torch.cuda.device(z.device):
            packed = pm._packed_conditioner(self._cin)
            yt = torch.empty(B, 9 * c3.out_channels, H, W, device=z.device, dtype=torch.float32)
            L.check(L.lib().nfb_glow_block(L.ptr(z), L.ptr(out), L.ptr(scratch), L.ptr(yt), L.ptr(ld), L.ptr(w), L.ptr(b),
                                           L.ptr(ldc), L.ptr(packed), L.ptr(c1.bias), L.ptr(c2.bias), L.ptr(c3.bias),
                                           B, C, H, W, c1.out_channels, *self._modes, float(pm.leaky), direction,
                                           L.stream_ptr()))
        return True

    def _coupling(self, z, param, ld, ldc, direction):
        """nfb_affine_coupling_image in place on the transformed half of z, given the conditioner's output param;
        ld / ldc None: no log-det."""
        B, C, H, W = z.shape
        L.check(L.lib().nfb_affine_coupling_image(L.ptr(z), L.ptr(param), L.ptr(ld), L.ptr(ldc), B, C, H * W,
                                                  *self._modes, direction, 0, L.stream_ptr()))

    def _check(self, z):
        z = require_cuda_f32(z)
        if z.dim() != 4 or z.shape[1] != self.channels:
            raise ValueError("Expected an NCHW tensor with {} channels.".format(self.channels))
        return z

    def forward(self, z):
        """Sampling direction (glow.py:72-77): coupling block, then Invertible1x1Conv.forward, then ActNorm.forward."""
        z = self._check(z)
        an = self.flows[2]
        B, C, H, W = z.shape
        dev = z.device
        out = torch.empty_like(z)
        ld = torch.empty(B, device=dev)
        if B == 0:
            return out, ld
        if an._done():
            w, b, ldc = self._folded(L.NFB_FORWARD, H * W, dev)
            if self._one_call(z, out, torch.empty_like(z), ld, w, b, ldc, L.NFB_FORWARD):
                return out, ld
        mid = z.clone()  # the coupling kernel works in place on the transformed half
        with torch.cuda.device(dev):
            param = self._param_map().apply_native(z, self._c0, self._cin)
            if not an._done():
                # data-dependent init in the sampling direction sees the output of the 1x1 convolution
                # (normalization.py:19-29): run the first two layers on a copy, initialise, then fold again
                w0, b0, _ = self._folded(L.NFB_FORWARD, H * W, dev)
                tmp = mid.clone()
                self._coupling(tmp, param, None, None, L.NFB_FORWARD)
                pre = torch.empty_like(z)
                _pointwise(tmp, w0, b0, pre)
                an._data_init(pre, "forward")
            w, b, ldc = self._folded(L.NFB_FORWARD, H * W, dev)
            self._coupling(mid, param, ld, ldc, L.NFB_FORWARD)
            _pointwise(mid, w, b, out)
        return out, ld

    def inverse(self, z):
        if wants_grad(self, z):
            return GlowBlockInverseFn.apply(self, z, *self.parameters())
        return self._inverse_native(z)

    def _inverse_native(self, z):
        z = self._check(z)
        an = self.flows[2]
        if not an._done():
            an._data_init(z, "inverse")
        B, C, H, W = z.shape
        out = torch.empty_like(z)
        ld = torch.empty(B, device=z.device)
        if B == 0:
            return out, ld
        w, b, ldc = self._folded(L.NFB_INVERSE, H * W, z.device)
        if self._one_call(z, out, None, ld, w, b, ldc, L.NFB_INVERSE):
            return out, ld
        with torch.cuda.device(z.device):
            _pointwise(z, w, b, out)
            param = self._param_map().apply_native(out, self._c0, self._cin)
            self._coupling(out, param, ld, ldc, L.NFB_INVERSE)
        return out, ld

    def _inverse_backward(self, z, g_out, g_ld):
        """Adjoint of the density direction: recompute the folded 1x1 output and the conditioner's activations, then
        coupling adjoint -> conditioner dgrad / wgrad -> 1x1 dgrad / wgrad (all CUDA), and the gradients of the folded
        w [C, C], b [C] and log-det constant mapped to Invertible1x1Conv / ActNorm parameters by torch autograd over the
        fold.  Returns (g_z, {id(parameter): gradient})."""
        lib = L.lib()
        conv, an = self.flows[1], self.flows[2]
        pm = self._param_map()
        B, C, H, W = z.shape
        HW, dev = H * W, z.device
        c0, cin = self._c0, self._cin
        grads = {}
        with torch.cuda.device(dev):
            st = L.stream_ptr()
            w, b, _ = self._folded(L.NFB_INVERSE, HW, dev)
            mid = torch.empty_like(z)
            _pointwise(z, w, b, mid)
            acts = pm.native_activations(mid, c0, cin)
            param = acts[-1]
            g_mid = torch.empty_like(z)
            g_param = torch.empty_like(param)
            L.check(lib.nfb_affine_coupling_image_backward(
                L.ptr(mid), L.ptr(param), L.ptr(g_out), L.ptr(g_ld), L.ptr(g_mid), L.ptr(g_param), B, C, HW,
                *self._modes, st))
            g_z1 = torch.empty(B, cin, H, W, device=dev)   # z1 passes through the coupling and feeds the conditioner
            L.check(lib.nfb_copy_channels(L.ptr(g_out), L.ptr(g_z1), B, C, c0, cin, HW, st))
            grads.update(pm.native_backward(mid, c0, cin, acts, g_param, g_z1))
            L.check(lib.nfb_paste_channels(L.ptr(g_z1), L.ptr(g_mid), B, C, c0, cin, HW, st))
            gz = torch.empty_like(z)
            L.check(lib.nfb_conv2d_dgrad(L.ptr(g_mid), L.ptr(w), L.ptr(gz), B, C, H, W, C, 1, None, 0.0, 0, st))
            gw, gb = torch.empty(C, C, device=dev), torch.empty(C, device=dev)
            L.check(lib.nfb_conv2d_wgrad(L.ptr(z), C, 0, L.ptr(g_mid), L.ptr(gw), L.ptr(gb), B, C, H, W, C, 1, 0, st))
        srcs = [p for p in conv._sources() + (an.s, an.t) if isinstance(p, nn.Parameter) and p.requires_grad]
        if srcs:
            with torch.enable_grad():
                outs = [(o, g) for o, g in zip(conv.folded_torch(an.s, an.t, HW), (gw, gb, g_ld.sum())) if o.requires_grad]
                gs = torch.autograd.grad([o for o, _ in outs], srcs, [g for _, g in outs], allow_unused=True)
            grads.update({id(p): g for p, g in zip(srcs, gs)})
        return gz, grads
