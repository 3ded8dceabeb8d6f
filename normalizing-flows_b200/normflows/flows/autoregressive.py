"""Masked affine autoregressive flow -- MAF (reference: normflows/flows/affine/autoregressive.py:9-128).

Same class names, constructor and module tree (`autoregressive_net` = nets.MADE with output_multiplier 2).  `forward`
is ONE conditioner pass + an element-wise affine; `inverse` is D sequential passes (:29-38), exactly like the
reference.  The conditioner runs as tensor-core GEMMs (csrc/nfb_gemm_tc.cu via nets.MADE.forward), the element-wise
part and its log-det reduction in csrc/nfb_kernels.cu (`maf_affine_kernel`).  Under grad, `inverse` goes through
`MafInverseFn`, whose backward is the fixed-point adjoint of the D-pass loop (nfb_maf_inverse_backward, DESIGN §3.9)."""
import numpy as np
import torch
from torch.nn import functional as F

from .. import _lib as L
from .._image_autograd import wants_grad
from .._native import require_cuda_f32
from ..nets import made as made_module
from .base import Flow


class Autoregressive(Flow):
    def __init__(self, autoregressive_net):
        super().__init__()
        self.autoregressive_net = autoregressive_net

    def forward(self, inputs, context=None):
        params = self.autoregressive_net(inputs, context)
        return self._elementwise_forward(inputs, params)

    def inverse(self, inputs, context=None):
        num_inputs = int(np.prod(inputs.shape[1:]))
        outputs = torch.zeros_like(inputs)
        logabsdet = None
        for _ in range(num_inputs):
            params = self.autoregressive_net(outputs, context)
            outputs, logabsdet = self._elementwise_inverse(inputs, params)
        return outputs, logabsdet

    def _output_dim_multiplier(self):
        raise NotImplementedError()

    def _elementwise_forward(self, inputs, autoregressive_params):
        raise NotImplementedError()

    def _elementwise_inverse(self, inputs, autoregressive_params):
        raise NotImplementedError()


class MaskedAffineAutoregressive(Autoregressive):
    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, use_residual_blocks=True,
                 random_mask=False, activation=F.relu, dropout_probability=0.0, use_batch_norm=False):
        self.features = features
        made = made_module.MADE(features=features, hidden_features=hidden_features, context_features=context_features,
                                num_blocks=num_blocks, output_multiplier=self._output_dim_multiplier(),
                                use_residual_blocks=use_residual_blocks, random_mask=random_mask, activation=activation,
                                dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)
        super().__init__(made)

    def _output_dim_multiplier(self):
        return 2

    def inverse(self, inputs, context=None):
        """The density direction; differentiable (MafInverseFn) when a gradient is wanted."""
        if wants_grad(self, inputs, context):
            x = require_cuda_f32(inputs)
            ctx = require_cuda_f32(context, "context") if context is not None else None
            return MafInverseFn.apply(self, x, ctx, *self.parameters())
        return super().inverse(inputs, context)

    def _affine(self, inputs, params, inverse):
        x = require_cuda_f32(inputs)
        if x.dim() != 2 or x.shape[1] != self.features:
            raise ValueError("Expected a [batch, {}] input.".format(self.features))
        params = params.contiguous()
        y = torch.empty_like(x)
        ld = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
        if x.shape[0]:
            with torch.cuda.device(x.device):
                L.check(L.lib().nfb_maf_affine(L.ptr(x), L.ptr(params), L.ptr(y), L.ptr(ld), x.shape[0], self.features,
                                               int(inverse), 0, L.stream_ptr()))
        return y, ld

    def _elementwise_forward(self, inputs, autoregressive_params):
        return self._affine(inputs, autoregressive_params, False)

    def _elementwise_inverse(self, inputs, autoregressive_params):
        return self._affine(inputs, autoregressive_params, True)


class MafInverseFn(torch.autograd.Function):
    """(y, log_det) = MaskedAffineAutoregressive.inverse(x, context): the forward is the layer's D-pass loop under
    no_grad (the value path, so values are bit-identical with and without grad); the backward is the fixed-point
    adjoint nfb_maf_inverse_backward, which equals the gradient of the unrolled loop.  Refuses to run the backward if a
    parameter was modified in place after the forward."""

    @staticmethod
    def forward(ctx, layer, x, context, *params):
        y, ld = Autoregressive.inverse(layer, x, context)
        ctx.layer, ctx.params = layer, params
        ctx.versions = [p._version for p in params]
        ctx.save_for_backward(x, y, context)
        return y, ld

    @staticmethod
    def backward(ctx, g_y, g_ld):
        from .._standalone import maf_inverse_backward
        x, y, context = ctx.saved_tensors
        layer = ctx.layer
        if any(p._version != v for p, v in zip(ctx.params, ctx.versions)):
            raise RuntimeError(f"{type(layer).__name__} backward: a parameter was modified in place after the "
                               "forward pass")
        need_x, need_ctx = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        gx, gctx, gmap = maf_inverse_backward(layer.autoregressive_net, layer.features, x, y, context,
                                              g_y.contiguous() if g_y is not None else None,
                                              g_ld.contiguous() if g_ld is not None else None, need_x, need_ctx)
        return (None, gx, gctx, *[gmap.get(p) if p.requires_grad else None for p in ctx.params])
