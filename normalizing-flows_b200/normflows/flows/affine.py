"""Affine family (reference: normflows/flows/affine/coupling.py:9-54 AffineConstFlow,
:99-171 AffineCoupling, :174-229 MaskedAffineFlow, :232-267 AffineCouplingBlock;
flows/normalization.py:7-39 ActNorm; flows/reshape.py Split/Merge)."""
import ctypes as C

import torch
from torch import nn

from .. import _lib as L
from .._native import mlp_desc
from ..nets.mlp import MLP
from .base import Flow, NativeFlow


class AffineConstFlow(NativeFlow):
    _affine_family = True

    def __init__(self, shape, scale=True, shift=True):
        super().__init__()
        if isinstance(shape, int):
            shape = (shape,)
        if scale:
            self.s = nn.Parameter(torch.zeros(shape)[None])
        else:
            self.register_buffer("s", torch.zeros(shape)[None])
        if shift:
            self.t = nn.Parameter(torch.zeros(shape)[None])
        else:
            self.register_buffer("t", torch.zeros(shape)[None])
        self.n_dim = self.s.dim()
        self.batch_dims = [i for i, n in enumerate(self.s.shape) if n == 1]

    def _native_tensors(self):
        return [self.s, self.t]

    def _native_add(self, handle, features):
        if self.s.numel() != features:
            raise NotImplementedError("AffineConstFlow with broadcast (image) shapes is not on the CUDA path yet")
        d = L.AffineConstDesc()
        d.features, d.s, d.t = features, self.s.data_ptr(), self.t.data_ptr()
        L.check(L.lib().nfb_flow_add_affine_const(handle, C.byref(d)))


class ActNorm(AffineConstFlow):
    """AffineConstFlow with data-dependent initialisation on the first batch
    (flows/normalization.py:19-39).  The one-time statistics use torch reductions on the device; the
    per-step transform is the fused affine kernel.  Unlike the reference the flag is kept on the host
    (no device->host sync per call, SURVEY 3.4)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.register_buffer("data_dep_init_done", torch.tensor(0.0))
        self._init_done_host = None

    def _done(self):
        if self._init_done_host is None:
            self._init_done_host = bool(self.data_dep_init_done.item() > 0.0)
        return self._init_done_host

    def _load_from_state_dict(self, *a, **k):
        super()._load_from_state_dict(*a, **k)
        self._init_done_host = None

    def _mark_done(self):
        self.data_dep_init_done.fill_(1.0)
        self._init_done_host = True

    @torch.no_grad()
    def _batch_stats(self, z):
        """mean / unbiased std over the batch dims (normalization.py:23-24,35-36).  Under data parallelism
        (torch.distributed initialised, world > 1) the statistics are those of the GLOBAL batch: one all-reduce
        of (sum x, sum x^2, n) in float64, so that every replica initialises the same s, t -- the single-process
        reference has no precedent; per-rank statistics would silently make the replicas different models."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return z.mean(dim=self.batch_dims, keepdim=True), z.std(dim=self.batch_dims, keepdim=True)
        zd = z.double()
        n = 1
        for d in self.batch_dims:
            n *= z.shape[d]
        buf = torch.cat([zd.sum(dim=self.batch_dims, keepdim=True).reshape(-1),
                         (zd * zd).sum(dim=self.batch_dims, keepdim=True).reshape(-1),
                         torch.tensor([float(n)], dtype=torch.float64, device=z.device)])
        dist.all_reduce(buf)
        c = (buf.numel() - 1) // 2
        n = buf[-1]
        mean = buf[:c] / n
        var = (buf[c:2 * c] - n * mean * mean) / (n - 1)
        shape = [1 if i in self.batch_dims else z.shape[i] for i in range(z.dim())]
        return mean.reshape(shape).to(z.dtype), var.clamp_min(0).sqrt().reshape(shape).to(z.dtype)

    @torch.no_grad()
    def _data_init(self, z, direction):
        mean, std = self._batch_stats(z)
        if direction == "forward":
            s = -torch.log(std + 1e-6)
            self.s.copy_(s)  # in place on the Parameter itself: bumps _version, which the packed caches watch
            self.t.copy_(-mean * torch.exp(s))
        else:
            self.s.copy_(torch.log(std + 1e-6))
            self.t.copy_(mean)
        self._mark_done()

    def forward(self, z, context=None):
        if not self._done():
            self._data_init(z, "forward")
        return super().forward(z)

    def inverse(self, z, context=None):
        if not self._done():
            self._data_init(z, "inverse")
        return super().inverse(z)


class MaskedAffineFlow(NativeFlow):
    _affine_family = True

    def __init__(self, b, t=None, s=None):
        super().__init__()
        self.register_buffer("b", b.view(1, *b.size()).float())
        for name, net in (("s", s), ("t", t)):
            if net is not None and not isinstance(net, MLP):
                raise NotImplementedError("MaskedAffineFlow on the CUDA path takes nets.MLP (or None) for s/t")
        # registration order follows the reference (coupling.py:198-206): s, then t
        if s is not None:
            self.add_module("s", s)
        else:
            self.s = None
        if t is not None:
            self.add_module("t", t)
        else:
            self.t = None

    def _native_tensors(self):
        ts = [self.b]
        for net in (self.s, self.t):
            if net is not None:
                ts += list(net.parameters())
        return ts

    def _native_add(self, handle, features):
        d = L.MaskedAffineDesc()
        d.features, d.b = features, self.b.data_ptr()
        d.s, d.t = mlp_desc(self.s), mlp_desc(self.t)
        L.check(L.lib().nfb_flow_add_masked_affine(handle, C.byref(d)))


class Split(Flow):
    def __init__(self, mode="channel"):
        super().__init__()
        if mode not in ("channel", "channel_inv"):
            raise NotImplementedError("Mode " + mode + " is not implemented.")
        self.mode = mode


class Merge(Split):
    pass


class AffineCoupling(Flow):
    def __init__(self, param_map, scale=True, scale_map="exp"):
        super().__init__()
        self.add_module("param_map", param_map)
        self.scale, self.scale_map = scale, scale_map


_MAPS = {"exp": 0, "sigmoid": 1, "sigmoid_inv": 2}   # scale-map enum of the coupling kernels (include/nfb200.h)


class AffineCouplingBlock(NativeFlow):
    _affine_family = True

    def __init__(self, param_map, scale=True, scale_map="exp", split_mode="channel"):
        super().__init__()
        if scale_map not in _MAPS:
            raise NotImplementedError("This scale map is not implemented.")
        if not isinstance(param_map, MLP):
            raise NotImplementedError("AffineCouplingBlock on the CUDA path takes a nets.MLP param_map")
        # same module tree as the reference (coupling.py:248-255): flows.0 Split, .1 coupling, .2 Merge
        self.flows = nn.ModuleList([Split(split_mode), AffineCoupling(param_map, scale, scale_map),
                                    Merge(split_mode)])
        self.scale, self.scale_map, self.split_mode = scale, scale_map, split_mode

    def _native_tensors(self):
        return list(self.flows[1].param_map.parameters())

    def _native_add(self, handle, features):
        d = L.AffineCouplingDesc()
        d.features, d.scale = features, int(bool(self.scale))
        d.scale_map = _MAPS[self.scale_map]
        d.split_mode = 0 if self.split_mode == "channel" else 1
        d.param_map = mlp_desc(self.flows[1].param_map)
        L.check(L.lib().nfb_flow_add_affine_coupling(handle, C.byref(d)))
