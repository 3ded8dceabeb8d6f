"""ConvNet2d parameter container (reference: normflows/nets/cnn.py:5-63): Conv2d / LeakyReLU stack with
`padding = k // 2`, last conv optionally zero-initialised; same `net.<i>` state_dict keys.  The convolutions
run in csrc/nfb_glow.cu (`nfb_conv2d`)."""
import torch
from torch import nn

from .. import _lib as L
from .._native import cached


class ConvNet2d(nn.Module):
    def __init__(self, channels, kernel_size, leaky=0.0, init_zeros=True, actnorm=False, weight_std=None):
        super().__init__()
        from ..utils.nn import ActNorm
        mods = []
        for i in range(len(kernel_size) - 1):
            conv = nn.Conv2d(channels[i], channels[i + 1], kernel_size[i], padding=kernel_size[i] // 2,
                             bias=(not actnorm))
            if weight_std is not None:
                conv.weight.data.normal_(mean=0.0, std=weight_std)
            mods.append(conv)
            if actnorm:  # nets/cnn.py:45-46: activation normalisation after every conv but the last
                mods.append(ActNorm((channels[i + 1],) + (1, 1)))
            mods.append(nn.LeakyReLU(leaky))
        i = len(kernel_size)
        mods.append(nn.Conv2d(channels[i - 1], channels[i], kernel_size[i - 1], padding=kernel_size[i - 1] // 2))
        if init_zeros:
            nn.init.zeros_(mods[-1].weight)
            nn.init.zeros_(mods[-1].bias)
        self.net = nn.Sequential(*mods)
        self.leaky = leaky

    def conv_layers(self):
        return [m for m in self.net if isinstance(m, nn.Conv2d)]

    def glow_shape(self, cin):
        """True when the net on `cin` input channels is the Glow conditioner that csrc/nfb_glow_fused.cu runs as one
        kernel: 3x3, 1x1 and 3x3 convolutions with no ActNorm, a LeakyReLU slope >= 0, and channel counts the library
        accepts (nfb_glow_conditioner_packed_bytes >= 0).  Fixed for a module and cin, so it is worked out once."""
        known = self.__dict__.setdefault("_nfb_glow_shape", {})
        if cin not in known:
            cv = self.conv_layers()
            known[cin] = (len(self.net) == 5 and [c.kernel_size[0] for c in cv] == [3, 1, 3]   # 5 modules: no ActNorm
                          and cv[0].out_channels == cv[1].in_channels == cv[1].out_channels and self.leaky >= 0.0
                          and L.lib().nfb_glow_conditioner_packed_bytes(cin, cv[0].out_channels, cv[2].out_channels) >= 0)
        return known[cin]

    def apply_native(self, x, c0, cin):
        """y = net(x[:, c0:c0+cin]) for a contiguous CUDA NCHW tensor x; returns [B, out, H, W].  An ActNorm still
        waiting for its data-dependent init (flows/normalization.py:19-29) gets it from its conv's raw output."""
        B, ctot, H, W = x.shape
        dev = x.device
        with torch.cuda.device(dev):
            if self.glow_shape(cin):
                # ONE fused tensor-core kernel (csrc/nfb_glow_fused.cu) leaves the last 3x3 convolution as nine stacked
                # 1x1 products; the shifted tap sum adds them up
                c1, c2, c3 = self.conv_layers()
                yt = torch.empty(B, 9 * c3.out_channels, H, W, device=dev)
                out = torch.empty(B, c3.out_channels, H, W, device=dev)
                L.check(L.lib().nfb_glow_conditioner_packed(L.ptr(x), ctot, c0, cin, L.ptr(self._packed_conditioner(cin)),
                                                            L.ptr(c1.bias), L.ptr(c2.bias), L.ptr(yt), B, H, W,
                                                            c1.out_channels, c3.out_channels, float(self.leaky),
                                                            L.stream_ptr()))
                L.check(L.lib().nfb_tap_shift_add(L.ptr(yt), L.ptr(c3.bias), L.ptr(out), B, c3.out_channels, H, W, 3,
                                                  L.stream_ptr()))
                return out
            cur, cur_tot, cur_c0 = x, ctot, c0
            for conv, an, act in self._layers():
                y = torch.empty(B, conv.out_channels, H, W, device=dev)
                k, ci, co = conv.kernel_size[0], conv.in_channels, conv.out_channels
                if an is not None and not an._done():
                    L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(conv.weight), None, L.ptr(y), B, ci,
                                               H, W, co, k, -1.0, L.stream_ptr()))
                    an._data_init(y, "forward")
                w, b = self._fold(conv, an)
                if conv is self.net[-1] and k > 1 and ci >= 128 and k * k * co <= 256 and co <= 64:
                    # last k x k conv with few outputs: k*k stacked 1x1 products on the tensor core + a shifted sum
                    # (csrc/nfb_glow.cu tap_shift_add_kernel) instead of an im2col GEMM with K = k*k*cin
                    yt = torch.empty(B, k * k * co, H, W, device=dev)
                    L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(self._tap_weights(conv)), None,
                                               L.ptr(yt), B, ci, H, W, k * k * co, 1, -1.0, L.stream_ptr()))
                    L.check(L.lib().nfb_tap_shift_add(L.ptr(yt), L.ptr(b), L.ptr(y), B, co, H, W, k, L.stream_ptr()))
                else:
                    L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(w), L.ptr(b), L.ptr(y), B, ci, H, W,
                                               co, k, act, L.stream_ptr()))
                cur, cur_tot, cur_c0 = y, co, 0
        return cur

    def _layers(self):
        """[(conv, the ActNorm that follows it or None, act)] per convolution; act = LeakyReLU slope, or -1.0 for the
        last layer."""
        from ..utils.nn import ActNorm
        mods = list(self.net)
        return [(conv, mods[j + 1].actNorm if j + 1 < len(mods) and isinstance(mods[j + 1], ActNorm) else None,
                 -1.0 if conv is mods[-1] else float(self.leaky))
                for j, conv in enumerate(mods) if isinstance(conv, nn.Conv2d)]

    @staticmethod
    def _fold(conv, an, differentiable=False):
        """(w, b) of conv with the ActNorm after it folded in (w * exp(s), b = t).  differentiable=True: w / b keep
        autograd history to the parameters (the gradient chain of the training pass)."""
        w, b = conv.weight, conv.bias
        if an is not None:
            w = conv.weight * torch.exp(an.s.reshape(-1))[:, None, None, None]
            b = an.t.reshape(-1)
        if not differentiable:
            w, b = w.detach().contiguous(), b.detach().contiguous()
        return w, b

    def _folded_layers(self, differentiable=False):
        """[(conv, w, b, act)] per convolution, as apply_native runs them (see _layers and _fold)."""
        return [(conv, *self._fold(conv, an, differentiable), act) for conv, an, act in self._layers()]

    def native_activations(self, x, c0, cin):
        """Training-pass recompute of the conditioner on x[:, c0:c0+cin] layer by layer (nfb_conv2d): the list of every
        layer's output (post-activation); the last one is the parameter tensor.  ActNorm must be initialised.  For the
        Glow shape the forward ran the fused kernel and the tap sum instead: the recomputed activations and parameter
        tensor are the same sums rounded in a different order (~1e-5 relative), so the adjoint is taken at values within
        that of the forward's; a ReLU whose input lies that close to 0 may take the other branch."""
        B, ctot, H, W = x.shape
        acts, cur, cur_tot, cur_c0 = [], x, ctot, c0
        for conv, w, b, act in self._folded_layers():
            y = torch.empty(B, conv.out_channels, H, W, device=x.device, dtype=torch.float32)
            L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(w), L.ptr(b), L.ptr(y), B, conv.in_channels,
                                       H, W, conv.out_channels, conv.kernel_size[0], act, L.stream_ptr()))
            acts.append(y)
            cur, cur_tot, cur_c0 = y, conv.out_channels, 0
        return acts

    def native_backward(self, x, c0, cin, acts, g_out, g_x):
        """Adjoint of native_activations: g_out = gradient of the last output; the input gradient is ACCUMULATED into
        g_x [B, cin, H, W].  LeakyReLU' comes from the stored post-activation tensors.  Returns {id(parameter): grad};
        folded ActNorm gradients go back to (weight, s, t) by torch autograd over the fold."""
        lib = L.lib()
        B, ctot, H, W = x.shape
        layers = self._folded_layers()
        geff = [None] * len(layers)
        g = g_out
        for i in range(len(layers) - 1, -1, -1):
            conv, w, b, _ = layers[i]
            k, ci, co = conv.kernel_size[0], conv.in_channels, conv.out_channels
            inp, itot, ic0 = (x, ctot, c0) if i == 0 else (acts[i - 1], acts[i - 1].shape[1], 0)
            gw, gb = torch.empty_like(w), torch.empty(co, device=x.device)
            L.check(lib.nfb_conv2d_wgrad(L.ptr(inp), itot, ic0, L.ptr(g), L.ptr(gw), L.ptr(gb), B, ci, H, W, co, k, 0,
                                         L.stream_ptr()))
            geff[i] = (gw, gb)
            if i > 0:
                gi = torch.empty_like(acts[i - 1])
                L.check(lib.nfb_conv2d_dgrad(L.ptr(g), L.ptr(w), L.ptr(gi), B, ci, H, W, co, k, L.ptr(acts[i - 1]),
                                             float(self.leaky), 0, L.stream_ptr()))
                g = gi
            else:
                L.check(lib.nfb_conv2d_dgrad(L.ptr(g), L.ptr(w), L.ptr(g_x), B, ci, H, W, co, k, None, 0.0, 1,
                                             L.stream_ptr()))
        params = [p for p in self.parameters() if p.requires_grad]
        if not params:
            return {}
        with torch.enable_grad():
            outs, gs = [], []
            for (conv, w, b, _), (gw, gb) in zip(self._folded_layers(differentiable=True), geff):
                for t, gt in ((w, gw), (b, gb)):
                    if t.requires_grad:
                        outs.append(t)
                        gs.append(gt)
            got = torch.autograd.grad(outs, params, gs, allow_unused=True)
        return {id(p): gp for p, gp in zip(params, got)}

    def _packed_conditioner(self, cin):
        """bf16 hi | lo records of the three convolutions in the fused kernel's layout (csrc/nfb_glow_fused.cu), once per
        parameter version: re-packing them on every call cost 5.5 % of a Glow pass."""
        c1, c2, c3 = self.conv_layers()

        def pack():
            hid, cout = c1.out_channels, c3.out_channels
            buf = torch.empty(int(L.lib().nfb_glow_conditioner_packed_bytes(cin, hid, cout)), dtype=torch.uint8,
                              device=c1.weight.device)
            L.check(L.lib().nfb_glow_conditioner_pack(L.ptr(c1.weight), L.ptr(c2.weight), L.ptr(self._tap_weights(c3)),
                                                      cin, hid, cout, L.ptr(buf), L.stream_ptr()))
            return buf
        return cached(self, "_nfb_packed", (c1.weight, c2.weight, c3.weight), (), pack)

    def _tap_weights(self, conv):
        """[cout, cin, k, k] -> [k*k*cout, cin, 1, 1] with row (kh*k + kw)*cout + n = W[n, :, kh, kw]; once per
        parameter version."""
        def permute():
            with torch.no_grad():
                w = conv.weight.detach()
                return w.permute(2, 3, 0, 1).reshape(-1, w.shape[1], 1, 1).contiguous()
        return cached(self, "_nfb_tapw", (conv.weight,), (), permute)

    def forward(self, x):
        from .._native import require_cuda_f32
        x = require_cuda_f32(x)
        return self.apply_native(x, 0, x.shape[1])
