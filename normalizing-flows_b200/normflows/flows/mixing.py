"""Linear / permutation layers (reference: normflows/flows/mixing.py:9-54 Permute,
:213-247 _Permutation, :368-532 _LULinear, :535-563 LULinearPermute)."""
import ctypes as C

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .base import Flow, NativeFlow


class _PermutationBuf(nn.Module):
    def __init__(self, permutation):
        super().__init__()
        self.register_buffer("_permutation", permutation)


class _LUParams(nn.Module):
    """Packed LU parameters, registered in the reference's order (bias first, mixing.py:282,376-384)."""

    def __init__(self, features, identity_init=True, eps=1e-3):
        super().__init__()
        self.features, self.eps = features, eps
        n_tri = ((features - 1) * features) // 2
        self.bias = nn.Parameter(torch.zeros(features))
        self.lower_entries = nn.Parameter(torch.zeros(n_tri))
        self.upper_entries = nn.Parameter(torch.zeros(n_tri))
        self.unconstrained_upper_diag = nn.Parameter(torch.zeros(features))
        if identity_init:
            nn.init.constant_(self.unconstrained_upper_diag, float(np.log(np.exp(1 - eps) - 1)))
        else:
            stdv = 1.0 / np.sqrt(features)
            for p in (self.lower_entries, self.upper_entries, self.unconstrained_upper_diag):
                nn.init.uniform_(p, -stdv, stdv)


class LULinearPermute(NativeFlow):
    """Fixed random permutation followed by an LU-parameterised linear map.  In the density direction
    this layer is folded into the prologue of the next spline block's kernel (one 64x64 split-bf16
    GEMM on the tensor core) when the stack is run through `NormalizingFlow`."""

    def __init__(self, num_channels, identity_init=True):
        super().__init__()
        self.permutation = _PermutationBuf(torch.randperm(num_channels))
        self.linear = _LUParams(num_channels, identity_init=identity_init)

    def _native_tensors(self):
        return list(self.linear.parameters()) + [self.permutation._permutation]

    def _native_add(self, handle, features):
        if features != self.linear.features:
            raise ValueError("Dimension 1 in inputs must be of size {}.".format(self.linear.features))
        d = L.LuDesc()
        lin = self.linear
        d.features = lin.features
        d.permutation = self.permutation._permutation.data_ptr()
        d.lower_entries, d.upper_entries = lin.lower_entries.data_ptr(), lin.upper_entries.data_ptr()
        d.unconstrained_upper_diag, d.bias = lin.unconstrained_upper_diag.data_ptr(), lin.bias.data_ptr()
        d.eps = lin.eps
        L.check(L.lib().nfb_flow_add_lu_linear_permute(handle, C.byref(d)))


class Permute(NativeFlow):
    _affine_family = True

    def __init__(self, num_channels, mode="shuffle"):
        super().__init__()
        if mode not in ("shuffle", "swap"):
            raise NotImplementedError("The mode " + mode + " is not implemented.")
        self.mode, self.num_channels = mode, num_channels
        if mode == "shuffle":
            perm = torch.randperm(num_channels)
            inv = torch.empty_like(perm).scatter_(0, perm, torch.arange(num_channels))
            self.register_buffer("perm", perm)
            self.register_buffer("inv_perm", inv)

    def _index_lists(self):
        c = self.num_channels
        if self.mode == "shuffle":
            return self.perm.tolist(), self.inv_perm.tolist()
        h_f, h_i = c // 2, (c + 1) // 2  # mixing.py:34-37 / :47-50
        return list(range(h_f, c)) + list(range(h_f)), list(range(h_i, c)) + list(range(h_i))

    def _native_tensors(self):
        return [self.perm, self.inv_perm] if self.mode == "shuffle" else []

    def _native_add(self, handle, features):
        f, i = self._index_lists()
        d = L.PermuteDesc()
        d.features = self.num_channels
        fa, ia = (C.c_int32 * len(f))(*f), (C.c_int32 * len(i))(*i)
        d.perm, d.inv_perm = fa, ia
        L.check(L.lib().nfb_flow_add_permute(handle, C.byref(d)))


class InvertibleAffine(Flow):
    """Invertible affine map without shift, the 2-D ([batch, channels]) version of the invertible 1x1 convolution
    (reference: flows/mixing.py:136-207; both parameterisations).  z' = z W runs as one tensor-core GEMM
    (csrc/nfb_gemm_tc.cu); assembling W / its double-precision inverse / slogdet is C x C parameter preparation."""

    def __init__(self, num_channels, use_lu=True):
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

    @torch.no_grad()
    def _matrix(self, inverse):
        """(W or W^-1, log|det W|) as the reference forms them (:160-177, :179-205)."""
        if self.use_lu:
            Lm = torch.tril(self.L, diagonal=-1) + self.eye
            Um = torch.triu(self.U, diagonal=1) + torch.diag(self.sign_S * torch.exp(self.log_S))
            if inverse:
                W = (torch.inverse(Um.double()) @ torch.inverse(Lm.double())).float() @ self.P.t()
            else:
                W = self.P @ Lm @ Um
            return W, torch.sum(self.log_S)
        W = torch.inverse(self.W.double()).float() if inverse else self.W.detach()
        return W, torch.linalg.slogdet(self.W.double())[1].float()

    def _run(self, z, inverse_matrix):
        from .._native import linear
        W, logdet = self._matrix(inverse_matrix)
        return linear(z, W.t().contiguous()), (-logdet if inverse_matrix else logdet)

    def forward(self, z, context=None):
        return self._run(z, True)

    def inverse(self, z, context=None):
        return self._run(z, False)
