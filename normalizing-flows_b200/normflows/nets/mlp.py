"""MLP parameter container (reference: normflows/nets/mlp.py:5-58).

Same constructor and `state_dict` keys (`net.<i>.weight|bias`).  Inside a flow the arithmetic runs in the
affine-stack kernel (csrc/nfb_affine.cu); calling the module directly runs one tensor-core GEMM per layer."""
from torch import nn


class MLP(nn.Module):
    def __init__(self, layers, leaky=0.0, score_scale=None, output_fn=None, output_scale=None,
                 init_zeros=False, dropout=None):
        super().__init__()
        if output_fn is not None or score_scale is not None or output_scale is not None:
            raise NotImplementedError("MLP output_fn / scaling is not on the CUDA path")
        if dropout is not None:
            raise NotImplementedError("MLP dropout is not on the CUDA path")
        layers = [int(n) for n in layers]   # (the VAE notebook passes numpy arrays)
        mods = []
        for k in range(len(layers) - 2):
            mods += [nn.Linear(layers[k], layers[k + 1]), nn.LeakyReLU(leaky)]
        mods.append(nn.Linear(layers[-2], layers[-1]))
        if init_zeros:
            nn.init.zeros_(mods[-1].weight)
            nn.init.zeros_(mods[-1].bias)
        self.net = nn.Sequential(*mods)
        self.leaky = leaky
        self.layer_sizes = list(layers)

    def linear_layers(self):
        return [m for m in self.net if isinstance(m, nn.Linear)]

    def forward(self, x):
        """Stand-alone evaluation (nets/mlp.py:57-58): one tensor-core GEMM per Linear (csrc/nfb_gemm_tc.cu).  Inside
        MaskedAffineFlow / AffineCouplingBlock the net is evaluated by the fused affine kernel instead.  Under autograd
        the backward is one nfb_mlp_backward call."""
        from .._standalone import apply_module
        return apply_module(self, x)

    def _value(self, x, context, keep):
        import torch
        from .._native import linear
        lins = self.linear_layers()
        h = x
        for i, lin in enumerate(lins):
            last = i + 1 == len(lins)
            h = linear(h, lin.weight, lin.bias, relu_out=(not last and self.leaky == 0.0))
            if not last and self.leaky != 0.0:
                h = torch.where(h > 0, h, h * self.leaky)
        return h

    def _adjoint(self, x, context, keep, grads, need_x, need_ctx):
        from .._standalone import mlp_backward
        gx, gmap = mlp_backward(self, x, grads[0], need_x)
        return gx, None, gmap
