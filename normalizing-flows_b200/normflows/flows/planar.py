"""Planar flow (Rezende & Mohamed 2015; reference: normflows/flows/planar.py:8-81).

    f(z) = z + u_hat h(w.z + b),  u_hat = u + (log(1 + exp(w.u)) - 1 - w.u) w / |w|^2   (so that w.u_hat > -1)

Consecutive Planar / Radial layers run as one launch of csrc/nfb_planar.cu, one thread per row; the sampling direction
(`forward`) is differentiated natively (nfb_flow_sampling_backward).  Only the leaky-ReLU layer has a density direction."""
import ctypes as C

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .base import NativeFlow

MAX_FEATURES = 64   # csrc/nfb_kernels.h kPlanarMaxD


def check_features(name, p):
    """A [1, D] parameter with D <= 64: the shapes the CUDA path covers."""
    if p.dim() > 2:
        raise NotImplementedError(f"{name} with image-shaped parameters is not on the CUDA path")
    if p.numel() > MAX_FEATURES:
        raise NotImplementedError(f"{name} on the CUDA path supports at most {MAX_FEATURES} features, got {p.numel()}")


class Planar(NativeFlow):
    _planar_family = True

    def __init__(self, shape, act="tanh", u=None, w=None, b=None):
        super().__init__()
        lim_w = np.sqrt(2.0 / np.prod(shape))
        lim_u = np.sqrt(2)
        # parameter order and RNG draws as in the reference: u, then w, then b
        if u is not None:
            self.u = nn.Parameter(u)
        else:
            self.u = nn.Parameter(torch.empty(shape)[None])
            nn.init.uniform_(self.u, -lim_u, lim_u)
        if w is not None:
            self.w = nn.Parameter(w)
        else:
            self.w = nn.Parameter(torch.empty(shape)[None])
            nn.init.uniform_(self.w, -lim_w, lim_w)
        if b is not None:
            self.b = nn.Parameter(b)
        else:
            self.b = nn.Parameter(torch.zeros(1))
        self.act = act
        if act == "tanh":
            self.h = torch.tanh
        elif act == "leaky_relu":
            self.h = torch.nn.LeakyReLU(negative_slope=0.2)
        else:
            raise NotImplementedError("Nonlinearity is not implemented.")

    @property
    def _no_inverse(self):
        return self.act != "leaky_relu"

    def inverse(self, z, context=None):
        if self._no_inverse:
            raise NotImplementedError("This flow has no algebraic inverse.")
        return super().inverse(z, context)

    def _native_tensors(self):
        return [self.u, self.w, self.b]

    def _native_add(self, handle, features):
        check_features("Planar", self.w)
        if self.u.numel() != features or self.w.numel() != features or self.b.numel() != 1:
            raise ValueError(f"Planar: parameters of shape {tuple(self.w.shape)} for {features} features")
        d = L.PlanarDesc()
        d.features, d.u, d.w, d.b = features, self.u.data_ptr(), self.w.data_ptr(), self.b.data_ptr()
        if self.act == "tanh":
            d.act, d.slope = L.NFB_PLANAR_TANH, 0.0
        else:
            d.act, d.slope = L.NFB_PLANAR_LEAKY_RELU, float(self.h.negative_slope)
        L.check(L.lib().nfb_flow_add_planar(handle, C.byref(d)))
