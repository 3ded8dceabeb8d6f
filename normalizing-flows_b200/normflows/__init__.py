"""normflows-b200: the coupling-stack hot path of `normflows` as hand-written sm_90a (H100) CUDA kernels
behind the reference's `nf.NormalizingFlow` / `nf.flows.*` nn.Module API.

    import normflows as nf            # this package; sys.path entry: <repo>/normalizing-flows_b200
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(64, trainable=False), flows).cuda()
    loss = model.forward_kld(x)       # one fused kernel per [LULinearPermute + spline block]

Scope: SURVEY.md section 8 / DESIGN.md.  Compute happens in libnfb200.so (C ABI: include/nfb200.h);
there is no CPU/eager fallback."""
from . import distributions, flows, nets, transforms, utils
from .core import NormalizingFlow, ConditionalNormalizingFlow, ClassCondFlow, MultiscaleFlow
from . import parallel
from ._native import invalidate_packed_weights

__version__ = "0.1.0+b200"
