"""MADE parameter container (reference: normflows/nets/made.py:14-304).

Same module tree and buffers (`mask`, `degrees` on every MaskedLinear), so reference checkpoints load
verbatim.  Degree assignment: inputs 1..D (made.py:14-16), hidden unit j gets
j % max(1, D-1) + min(1, D-1) (:72-76), output feature j's `multiplier` rows get degree j+1 and use a
strict > mask (:57-60); hidden masks use >=.  The mask multiply the reference redoes on every call
(:80-81) happens once per parameter update in the packer (csrc/nfb_api.cu)."""
import torch
from torch import nn
from torch.nn import functional as F, init

from .resnet import _check_plain, _preprocess


class MaskedLinear(nn.Linear):
    def __init__(self, in_degrees, out_features, autoregressive_features, random_mask, is_output,
                 bias=True, out_degrees_=None):
        super().__init__(in_features=len(in_degrees), out_features=out_features, bias=bias)
        if random_mask:
            raise NotImplementedError("random masks are not on the CUDA path")
        d = autoregressive_features
        if is_output:
            base = torch.arange(1, d + 1) if out_degrees_ is None else out_degrees_
            degrees = base.reshape(-1).repeat_interleave(out_features // d)
            mask = (degrees[:, None] > in_degrees[None, :]).float()
        else:
            degrees = torch.arange(out_features) % max(1, d - 1) + min(1, d - 1)
            mask = (degrees[:, None] >= in_degrees[None, :]).float()
        self.register_buffer("mask", mask)
        self.register_buffer("degrees", degrees)


class MaskedResidualBlock(nn.Module):
    def __init__(self, in_degrees, autoregressive_features, context_features=None, random_mask=False,
                 activation=F.relu, dropout_probability=0.0, use_batch_norm=False, zero_initialization=True):
        if random_mask:
            raise ValueError("Masked residual block can't be used with random masks.")
        super().__init__()
        _check_plain(activation, dropout_probability, use_batch_norm, context_features)
        features = len(in_degrees)
        if context_features is not None:  # made.py:159-160
            self.context_layer = nn.Linear(context_features, features)
        l0 = MaskedLinear(in_degrees, features, autoregressive_features, False, False)
        l1 = MaskedLinear(l0.degrees, features, autoregressive_features, False, False)
        self.linear_layers = nn.ModuleList([l0, l1])
        self.degrees = l1.degrees
        if not bool(torch.all(self.degrees >= in_degrees)):
            raise RuntimeError("In a masked residual block, the output degrees can't be less than the "
                               "corresponding input degrees.")
        if zero_initialization:
            init.uniform_(self.linear_layers[-1].weight, a=-1e-3, b=1e-3)
            init.uniform_(self.linear_layers[-1].bias, a=-1e-3, b=1e-3)


class MADE(nn.Module):
    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, output_multiplier=1,
                 use_residual_blocks=True, random_mask=False, permute_mask=False, activation=F.relu,
                 dropout_probability=0.0, use_batch_norm=False, preprocessing=None):
        if use_residual_blocks and random_mask:
            raise ValueError("Residual blocks can't be used with random masks.")
        super().__init__()
        _check_plain(activation, dropout_probability, use_batch_norm, context_features)
        if not use_residual_blocks:
            raise NotImplementedError("feed-forward MADE blocks are not on the CUDA path")
        # (made.py:241-244: an elementwise module in front of the first masked layer, e.g. PeriodicFeaturesElementwise)
        self.preprocessing = preprocessing
        in_deg = torch.arange(1, features + 1)
        if permute_mask:
            in_deg = in_deg[torch.randperm(features)]
        self.initial_layer = MaskedLinear(in_deg, hidden_features, features, random_mask, False)
        if context_features is not None:  # made.py:261-262
            self.context_layer = nn.Linear(context_features, hidden_features)
        blocks, prev = [], self.initial_layer.degrees
        for _ in range(num_blocks):
            blocks.append(MaskedResidualBlock(prev, features, context_features, random_mask, activation))
            prev = blocks[-1].degrees
        self.blocks = nn.ModuleList(blocks)
        self.final_layer = MaskedLinear(prev, features * output_multiplier, features, random_mask, True,
                                        out_degrees_=in_deg)

    def forward(self, inputs, context=None):
        """nets/made.py:296-304, stand-alone call: masked weights, pre-activation residual blocks."""
        from .._standalone import apply_module
        return apply_module(self, inputs, context)

    def _value(self, inputs, context, keep):
        from .._native import resnet_forward
        if self.preprocessing is not None:
            inputs = _preprocess(self.preprocessing, inputs)
        return resnet_forward(self, inputs, masked=True, context=context)

    def _adjoint(self, inputs, context, keep, grads, need_x, need_ctx):
        from .._standalone import conditioner_backward
        return conditioner_backward(self, True, inputs, context, grads[0], need_x, need_ctx)
