"""ConvNet2d parameter container (reference: normflows/nets/cnn.py:5-63): Conv2d / LeakyReLU stack with
`padding = k // 2`, last conv optionally zero-initialised; same `net.<i>` state_dict keys.  The convolutions
run in csrc/nfb_glow.cu (`nfb_conv2d`)."""
from torch import nn

from .. import _lib as L


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

    def _glow_shape(self, cin):
        mods = list(self.net)
        convs = self.conv_layers()
        return (len(convs) == 3 and len(mods) == 5 and [cv.kernel_size[0] for cv in convs] == [3, 1, 3]
                and convs[0].out_channels == convs[1].out_channels == convs[1].in_channels
                and convs[0].out_channels % 64 == 0 and convs[0].out_channels <= 256
                and 9 * cin <= 256 and 9 * convs[2].out_channels <= 512 and self.leaky >= 0.0)

    def apply_native_taps(self, x, c0, cin):
        """The Glow conditioner shape only: returns (y_taps [B, 9 * out, H, W], bias [out]) -- the last 3x3 convolution
        left as nine stacked 1x1 products for nfb_affine_coupling_image_taps to sum on the fly -- or None."""
        import torch
        if not self._glow_shape(cin):
            return None
        B, ctot, H, W = x.shape
        c1, c2, c3 = self.conv_layers()
        cout, hid = c3.out_channels, c1.out_channels
        yt = torch.empty(B, 9 * cout, H, W, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            packed = self._packed_conditioner(c1, c2, c3, cin, hid, cout)
            L.check(L.lib().nfb_glow_conditioner_packed(L.ptr(x), ctot, c0, cin, L.ptr(packed), L.ptr(c1.bias),
                                                        L.ptr(c2.bias), L.ptr(yt), B, H, W, hid, cout,
                                                        float(self.leaky), L.stream_ptr()))
        return yt, c3.bias

    def apply_native(self, x, c0, cin):
        """y = net(x[:, c0:c0+cin]) for a contiguous CUDA NCHW tensor x; returns [B, out, H, W]."""
        import torch
        B, ctot, H, W = x.shape
        from ..utils.nn import ActNorm
        mods = list(self.net)
        convs = self.conv_layers()
        if self._glow_shape(cin):
            # the Glow conditioner shape: ONE fused tensor-core kernel (csrc/nfb_glow_fused.cu) + the shifted tap sum
            c1, c2, c3 = convs
            cout, hid = c3.out_channels, c1.out_channels
            yt = torch.empty(B, 9 * cout, H, W, device=x.device, dtype=torch.float32)
            out = torch.empty(B, cout, H, W, device=x.device, dtype=torch.float32)
            with torch.cuda.device(x.device):
                packed = self._packed_conditioner(c1, c2, c3, cin, hid, cout)   # once per parameter version
                L.check(L.lib().nfb_glow_conditioner_packed(L.ptr(x), ctot, c0, cin, L.ptr(packed), L.ptr(c1.bias),
                                                            L.ptr(c2.bias), L.ptr(yt), B, H, W, hid, cout,
                                                            float(self.leaky), L.stream_ptr()))
                L.check(L.lib().nfb_tap_shift_add(L.ptr(yt), L.ptr(c3.bias), L.ptr(out), B, cout, H, W, 3, L.stream_ptr()))
            return out
        cur, cur_tot, cur_c0 = x, ctot, c0
        with torch.cuda.device(x.device):
            for j, conv in enumerate(mods):
                if not isinstance(conv, nn.Conv2d):
                    continue
                last = conv is mods[-1]
                an = mods[j + 1].actNorm if j + 1 < len(mods) and isinstance(mods[j + 1], ActNorm) else None
                w, b = conv.weight, conv.bias
                y = torch.empty(B, conv.out_channels, H, W, device=x.device, dtype=torch.float32)

                def run(wt, bt, act):
                    L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(wt), L.ptr(bt), L.ptr(y), B,
                                               conv.in_channels, H, W, conv.out_channels, conv.kernel_size[0], act,
                                               L.stream_ptr()))
                if an is not None:
                    # ActNorm after the conv = per-channel affine: folded into the conv's weights and bias.  First
                    # call: raw conv output -> data-dependent init (flows/normalization.py:19-29), then the fold.
                    if not an._done():
                        run(w, None, -1.0)
                        an._data_init(y, "forward")
                    with torch.no_grad():
                        e = torch.exp(an.s.detach().reshape(-1))
                        w = (conv.weight.detach() * e[:, None, None, None]).contiguous()
                        b = an.t.detach().reshape(-1).contiguous()
                k = conv.kernel_size[0]
                if (last and an is None and k > 1 and conv.in_channels >= 128 and k * k * conv.out_channels <= 256
                        and conv.out_channels <= 64):
                    # k x k conv with few outputs: k*k stacked 1x1 products on the tensor core + a shifted sum
                    # (csrc/nfb_glow.cu tap_shift_add_kernel) instead of an im2col GEMM with K = k*k*cin
                    wt = self._tap_weights(conv)
                    yt = torch.empty(B, k * k * conv.out_channels, H, W, device=x.device, dtype=torch.float32)
                    L.check(L.lib().nfb_conv2d(L.ptr(cur), cur_tot, cur_c0, L.ptr(wt), None, L.ptr(yt), B,
                                               conv.in_channels, H, W, k * k * conv.out_channels, 1, -1.0, L.stream_ptr()))
                    L.check(L.lib().nfb_tap_shift_add(L.ptr(yt), L.ptr(b), L.ptr(y), B, conv.out_channels, H, W, k,
                                                      L.stream_ptr()))
                else:
                    run(w, b, -1.0 if last else float(self.leaky))
                cur, cur_tot, cur_c0 = y, conv.out_channels, 0
        return cur

    def _folded_layers(self, differentiable=False):
        """[(conv, w, b, act)] per convolution with a following ActNorm folded in (w * exp(s), b = t), as apply_native
        runs them; act = LeakyReLU slope, or -1.0 for the last layer.  differentiable=True: w / b keep autograd history
        to the parameters (the gradient chain of the training pass)."""
        import torch
        from ..utils.nn import ActNorm
        mods = list(self.net)
        out = []
        for j, conv in enumerate(mods):
            if not isinstance(conv, nn.Conv2d):
                continue
            an = mods[j + 1].actNorm if j + 1 < len(mods) and isinstance(mods[j + 1], ActNorm) else None
            w, b = conv.weight, conv.bias
            if an is not None:
                w = conv.weight * torch.exp(an.s.reshape(-1))[:, None, None, None]
                b = an.t.reshape(-1)
            if not differentiable:
                w, b = w.detach().contiguous(), b.detach().contiguous()
            out.append((conv, w, b, -1.0 if conv is mods[-1] else float(self.leaky)))
        return out

    def native_activations(self, x, c0, cin):
        """Training-pass recompute of the conditioner on x[:, c0:c0+cin] layer by layer (nfb_conv2d): the list of every
        layer's output (post-activation); the last one is the parameter tensor.  ActNorm must be initialised.  For the
        Glow shape the forward ran the fused kernel with the tap-form coupling instead: the recomputed activations and
        parameter tensor are the same sums rounded in a different order (~1e-5 relative), so the adjoint is taken at
        values within that of the forward's; a ReLU whose input lies that close to 0 may take the other branch."""
        import torch
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
        import torch
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

    def _packed_conditioner(self, c1, c2, c3, cin, hid, cout):
        """bf16 hi | lo records of the three convolutions in the fused kernel's layout (csrc/nfb_glow_fused.cu), cached per
        parameter version (and packed-weight generation): round 2a re-packed them on every call (5.5 % of a Glow pass)."""
        import torch
        from .._native import generation
        ws = (c1.weight, c2.weight, c3.weight)
        sig = tuple((t.data_ptr(), t._version) for t in ws) + (generation(),)
        cache = self.__dict__.get("_nfb_packed")
        if cache is None or cache[0] != sig:
            nbytes = int(L.lib().nfb_glow_conditioner_packed_bytes(cin, hid, cout))
            buf = torch.empty(nbytes, dtype=torch.uint8, device=c1.weight.device)
            L.check(L.lib().nfb_glow_conditioner_pack(L.ptr(c1.weight), L.ptr(c2.weight), L.ptr(self._tap_weights(c3)),
                                                      cin, hid, cout, L.ptr(buf), L.stream_ptr()))
            cache = (sig, buf)
            self.__dict__["_nfb_packed"] = cache
        return cache[1]

    def _tap_weights(self, conv):
        """[cout, cin, k, k] -> [k*k*cout, cin, 1, 1] with row (kh*k + kw)*cout + n = W[n, :, kh, kw]; cached per
        parameter version (and packed-weight generation)."""
        import torch
        from .._native import generation
        sig = (conv.weight.data_ptr(), conv.weight._version, generation())
        cache = self.__dict__.get("_nfb_tapw")
        if cache is None or cache[0] != sig:
            with torch.no_grad():
                w = conv.weight.detach()
                wt = w.permute(2, 3, 0, 1).reshape(-1, w.shape[1], 1, 1).contiguous()
            cache = (sig, wt)
            self.__dict__["_nfb_tapw"] = cache
        return cache[1]

    def forward(self, x):
        from .._native import require_cuda_f32
        x = require_cuda_f32(x)
        return self.apply_native(x, 0, x.shape[1])
