"""Radial flow (Rezende & Mohamed 2015; reference: normflows/flows/radial.py:8-46).

    f(z) = z + beta_hat / (|alpha| + r) (z - z_0),  r = |z - z_0|,  beta_hat = log(1 + exp(beta)) - |alpha|

Runs with its Planar / Radial neighbours as one launch of csrc/nfb_planar.cu; the sampling direction (`forward`) is
differentiated natively.  It has no algebraic inverse."""
import ctypes as C

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .base import NativeFlow
from .planar import check_features


class Radial(NativeFlow):
    _planar_family = True
    _no_inverse = True

    def __init__(self, shape, z_0=None):
        super().__init__()
        # registration order and RNG draws as in the reference: buffer d, beta, alpha, then z_0
        self.d_cpu = torch.prod(torch.tensor(shape))
        self.register_buffer("d", self.d_cpu)
        self.beta = nn.Parameter(torch.empty(1))
        lim = 1.0 / np.prod(shape)
        nn.init.uniform_(self.beta, -lim - 1.0, lim - 1.0)
        self.alpha = nn.Parameter(torch.empty(1))
        nn.init.uniform_(self.alpha, -lim, lim)
        if z_0 is not None:
            self.z_0 = nn.Parameter(z_0)
        else:
            self.z_0 = nn.Parameter(torch.randn(shape)[None])

    def inverse(self, z, context=None):
        raise NotImplementedError("This flow has no algebraic inverse.")

    def _native_tensors(self):
        return [self.beta, self.alpha, self.z_0]

    def _native_add(self, handle, features):
        check_features("Radial", self.z_0)
        if self.z_0.numel() != features:
            raise ValueError(f"Radial: z_0 of shape {tuple(self.z_0.shape)} for {features} features")
        d = L.RadialDesc()
        d.features, d.beta, d.alpha, d.z0 = features, self.beta.data_ptr(), self.alpha.data_ptr(), self.z_0.data_ptr()
        L.check(L.lib().nfb_flow_add_radial(handle, C.byref(d)))
