"""ResidualNet parameter container (reference: normflows/nets/resnet.py:7-104).

Identical module tree / state_dict keys: initial_layer, blocks.<n>.linear_layers.<0|1>, final_layer.
Pre-activation residual blocks with ReLU; the second linear of each block starts U(-1e-3, 1e-3)
(resnet.py:33-35).  The forward pass is part of the fused coupling kernel (csrc/nfb_fused_rqs.cu)
or, for shapes it does not cover, the fp32 tiles in csrc/nfb_kernels.cu."""
import torch
from torch import nn
from torch.nn import functional as F, init


def _check_plain(activation, dropout_probability, use_batch_norm, context_features):
    relu = activation is F.relu or isinstance(activation, nn.ReLU) or activation is torch.relu
    if not relu:
        raise NotImplementedError("only ReLU conditioners are on the CUDA path")
    if dropout_probability != 0.0:
        raise NotImplementedError("dropout in the conditioner is not on the CUDA path")
    if use_batch_norm:
        raise NotImplementedError("batch-norm in the conditioner is not on the CUDA path")


def _preprocess(module, inputs):
    """Value of the conditioner's preprocessing module (kernel path for PeriodicFeaturesElementwise, else its call)."""
    return module._value(inputs, None, None) if hasattr(module, "_value") else module(inputs)


class ResidualBlock(nn.Module):
    def __init__(self, features, context_features=None, activation=F.relu, dropout_probability=0.0,
                 use_batch_norm=False, zero_initialization=True):
        super().__init__()
        _check_plain(activation, dropout_probability, use_batch_norm, context_features)
        if context_features is not None:  # registered before linear_layers, like the reference (resnet.py:27-31)
            self.context_layer = nn.Linear(context_features, features)
        self.linear_layers = nn.ModuleList([nn.Linear(features, features) for _ in range(2)])
        if zero_initialization:
            init.uniform_(self.linear_layers[-1].weight, -1e-3, 1e-3)
            init.uniform_(self.linear_layers[-1].bias, -1e-3, 1e-3)


class ResidualNet(nn.Module):
    def __init__(self, in_features, out_features, hidden_features, context_features=None, num_blocks=2,
                 activation=F.relu, dropout_probability=0.0, use_batch_norm=False, preprocessing=None):
        super().__init__()
        _check_plain(activation, dropout_probability, use_batch_norm, context_features)
        self.hidden_features = hidden_features
        self.context_features = context_features
        self.preprocessing = preprocessing  # (a module, e.g. utils.nn.PeriodicFeaturesElementwise; resnet.py:71,93-96)
        self.initial_layer = nn.Linear(in_features + (context_features or 0), hidden_features)
        self.blocks = nn.ModuleList([ResidualBlock(hidden_features, context_features, activation) for _ in range(num_blocks)])
        self.final_layer = nn.Linear(hidden_features, out_features)

    def forward(self, inputs, context=None):
        """nets/resnet.py:92-104, stand-alone call (inside a flow the net is part of the fused kernel)."""
        from .._standalone import apply_module
        return apply_module(self, inputs, context)

    def _value(self, inputs, context, keep):
        from .._native import resnet_forward
        if self.preprocessing is not None:
            inputs = _preprocess(self.preprocessing, inputs)
        return resnet_forward(self, inputs, masked=False, context=context)

    def _adjoint(self, inputs, context, keep, grads, need_x, need_ctx):
        from .._standalone import conditioner_backward
        return conditioner_backward(self, False, inputs, context, grads[0], need_x, need_ctx)
