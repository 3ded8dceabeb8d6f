"""Flow protocol (reference: normflows/flows/base.py:5-24) and the native-layer mixin."""
import torch
from torch import nn

from .. import _lib as L
from .._image_autograd import wants_grad
from .._native import FlowHandle


class Flow(nn.Module):
    """Generic flow layer: `forward(z) -> (z', log_det[B])`, `inverse(z) -> (z', log_det[B])`."""

    _no_inverse = False   # True: `inverse` raises (Planar with tanh, Radial), and so does a density pass through it

    def forward(self, z):
        raise NotImplementedError("Forward pass has not been implemented.")

    def inverse(self, z):
        raise NotImplementedError("This flow has no algebraic inverse.")


class NativeFlow(Flow):
    """A layer whose arithmetic is a kernel in libnfb200.so.  Subclasses provide
    `_native_tensors()` (every parameter/buffer the kernels read) and `_native_add(handle, D)`
    (append this layer's descriptor to an nfb_flow)."""

    use_tensor_cores = True  # class-wide switch; False forces the plain-fp32 kernels (A/B parity)
    # the sampling direction has a native backward (nfb_flow_sampling_backward) for stacks of one family
    _affine_family = False
    _planar_family = False

    def _single(self):
        h = self.__dict__.get("_nfb_single")
        if h is None or h.use_tc != type(self).use_tensor_cores:
            h = FlowHandle([self], None, type(self).use_tensor_cores)
            self.__dict__["_nfb_single"] = h
        return h

    def forward(self, z, context=None):
        # (layers without context parameters ignore the context, like the reference's `context=None` signatures)
        if self._sampling_family() and wants_grad(self, z):
            from .._standalone import stack_sampling
            return stack_sampling(self._single(), [self], z, list(self.parameters()))
        return self._single().layer_apply(0, L.NFB_FORWARD, z)

    def _sampling_family(self):
        return "affine" if self._affine_family else "planar" if self._planar_family else None

    def _sampling_differentiable(self, context=None):
        return self._sampling_family() is not None

    def inverse(self, z, context=None):
        # under autograd (a layer called on its own, e.g. between the blocks of a stack that is not all native) the call
        # joins the graph; the sampling direction (`forward`) does too for the affine and planar families
        if wants_grad(self, z):
            from .._autograd import LayerInverseFn
            return LayerInverseFn.apply(self, z, *self.parameters())
        return self._single().layer_apply(0, L.NFB_INVERSE, z)

    def _native_tensors(self):
        raise NotImplementedError

    def _native_add(self, handle, features):
        raise NotImplementedError


class Reverse(Flow):
    """Switches forward and inverse of a flow (reference: flows/base.py:27-45)."""

    def __init__(self, flow):
        super().__init__()
        self.flow = flow

    def forward(self, z):
        return self.flow.inverse(z)

    def inverse(self, z):
        return self.flow.forward(z)


class Composite(Flow):
    """Composes several flows into one (reference: flows/base.py:48-78)."""

    def __init__(self, flows):
        super().__init__()
        self.flows = nn.ModuleList(flows)

    def forward(self, z):
        log_det = torch.zeros(len(z), device=z.device)
        for f in self.flows:
            z, ld = f(z)
            log_det = log_det + ld
        return z, log_det

    def inverse(self, z):
        log_det = torch.zeros(len(z), device=z.device)
        for f in reversed(self.flows):
            z, ld = f.inverse(z)
            log_det = log_det + ld
        return z, log_det


def zero_log_det_like_z(z):
    return torch.zeros(z.shape[0], dtype=z.dtype, device=z.device)
