"""Input pre-transforms (reference: normflows/transforms.py): `Logit` (:8-47) and `Shift` (:50-75), used as
`MultiscaleFlow(..., transform=...)`.  Logit runs as one CUDA kernel per call (element-wise map + per-sample log-det
reduction, csrc/nfb_glow.cu `logit_kernel`)."""
import torch

from . import _lib as L
from ._image_autograd import LogitInverseFn, wants_grad
from ._native import require_cuda_f32
from .flows.base import Flow


class Logit(Flow):
    def __init__(self, alpha=0.05):
        super().__init__()
        self.alpha = alpha

    def _run(self, z, direction):
        z = require_cuda_f32(z)
        out = torch.empty_like(z)
        ld = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        if z.shape[0]:
            inner = z.numel() // z.shape[0]
            with torch.cuda.device(z.device):
                L.check(L.lib().nfb_logit_transform(L.ptr(z), L.ptr(out), L.ptr(ld), z.shape[0], inner,
                                                    float(self.alpha), direction, 0, L.stream_ptr()))
        return out, ld

    def forward(self, z):
        return self._run(z, L.NFB_FORWARD)

    def inverse(self, z):
        if wants_grad(self, z):
            return LogitInverseFn.apply(self, z)
        return self._run(z, L.NFB_INVERSE)


class Shift(Flow):
    """Shift by a constant (default -0.5: [0, 1] -> [-0.5, 0.5]).  Like the reference (:66-75) the input tensor is
    modified in place; log-det is zero."""

    def __init__(self, shift=-0.5):
        super().__init__()
        self.shift = shift

    def forward(self, z):
        z -= self.shift
        return z, torch.zeros(z.shape[0], dtype=z.dtype, device=z.device)

    def inverse(self, z):
        z += self.shift
        return z, torch.zeros(z.shape[0], dtype=z.dtype, device=z.device)
