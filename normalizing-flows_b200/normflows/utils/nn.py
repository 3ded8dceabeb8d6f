"""normflows/utils/nn.py: small nn.Module helpers.  `ActNorm` (:25-43) wraps flows.ActNorm for use INSIDE a
conditioner (ConvNet2d(actnorm=True)); on the CUDA path ConvNet2d folds it into the preceding convolution."""
import torch
from torch import nn


class ConstScaleLayer(nn.Module):
    def __init__(self, scale=1.0):
        super().__init__()
        self.register_buffer("scale", torch.tensor(scale))

    def forward(self, input):
        return input * self.scale


class ActNorm(nn.Module):
    def __init__(self, shape):
        super().__init__()
        from ..flows.affine import ActNorm as _FlowActNorm
        self.actNorm = _FlowActNorm(shape)

    def forward(self, input):
        """y = input * exp(s) + t (broadcast over the batch dims), data-dependent init on the first call
        (flows/normalization.py:19-29).  Stand-alone use only; ConvNet2d folds the layer into its convolution."""
        an = self.actNorm
        if not an._done():
            an._data_init(input, "forward")
        return input * torch.exp(an.s) + an.t


class ClampExp(nn.Module):
    def forward(self, x):
        return torch.clamp(torch.exp(x), max=1.0)


class PeriodicFeaturesElementwise(nn.Module):
    """utils/nn.py:64-130 of the reference: the features `ind` become w1 sin(scale f) + w2 cos(scale f), the others
    pass through.  Same buffers / parameter as the reference (`ind`, `ind_`, `inv_perm`, `weights`, optional `scale`
    buffer, optional `bias`); the arithmetic is csrc/nfb_kernels.cu periodic_features_kernel."""

    def __init__(self, ndim, ind, scale=1.0, bias=False, activation=None):
        super().__init__()
        if activation is not None:
            raise NotImplementedError("an activation after the periodic features is not on the CUDA path")
        self.ndim = ndim
        ind = ind.long() if torch.is_tensor(ind) else torch.tensor(ind, dtype=torch.long)
        self.register_buffer("ind", ind)
        ind_ = [i for i in range(ndim) if i not in set(ind.tolist())]
        self.register_buffer("ind_", torch.tensor(ind_, dtype=torch.long))
        perm_ = torch.cat((self.ind, self.ind_))
        inv_perm_ = torch.zeros_like(perm_)
        for i in range(ndim):
            inv_perm_[perm_[i]] = i
        self.register_buffer("inv_perm", inv_perm_)
        self.weights = nn.Parameter(torch.ones(len(self.ind), 2))
        if torch.is_tensor(scale):
            self.register_buffer("scale", scale)
        else:
            self.scale = scale
        self.apply_bias = bias
        if bias:
            self.bias = nn.Parameter(torch.zeros(len(self.ind)))
        self.activation = nn.Identity()

    def _tables(self, dev):
        """(slot [ndim] int32, weights, scale [n_periodic], bias | None) on `dev` in the kernels' layout."""
        slot = torch.full((self.ndim,), -1, dtype=torch.int32)
        slot[self.ind.cpu()] = torch.arange(len(self.ind), dtype=torch.int32)
        sc = self.scale if torch.is_tensor(self.scale) else torch.full((len(self.ind),), float(self.scale))
        sc = sc.to(device=dev, dtype=torch.float32).reshape(-1).expand(len(self.ind)).contiguous()
        return (slot.to(dev), self.weights.detach().contiguous(), sc,
                self.bias.detach() if self.apply_bias else None)

    def forward(self, inputs):
        from .._standalone import apply_module
        return apply_module(self, inputs)

    def _value(self, inputs, context, keep):
        from .._native import periodic_features, require_cuda_f32
        x = require_cuda_f32(inputs)
        slot, w, sc, bias = self._tables(x.device)
        return periodic_features(x, slot, w, sc, bias)

    def _adjoint(self, inputs, context, keep, grads, need_x, need_ctx):
        from .._standalone import periodic_backward
        gx, gmap = periodic_backward(self, inputs, grads[0])
        return gx, None, gmap
