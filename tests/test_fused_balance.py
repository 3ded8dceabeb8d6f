"""The fused spline kernel with every hidden width it packs (H = 64 .. 256, H = 192 included) and both conditioner kinds:
MADE conditioners, whose hidden GEMMs the packer balances over the two consumer warpgroups (csrc/nfb_fused_plan.h),
and unmasked ones.  Density and sampling directions against the plain-fp32 kernels, on a batch with a ragged tail."""
import numpy as np
import pytest
import torch

import normflows as nf
from normflows.flows.base import NativeFlow

pytestmark = pytest.mark.gpu

RTOL = 1e-4


@pytest.fixture(autouse=True)
def _tc_default():
    NativeFlow.use_tensor_cores = True
    yield
    NativeFlow.use_tensor_cores = True


def _model(kind, d, hidden, layers=2, seed=0, sigma=0.05):
    torch.manual_seed(seed)
    fl = []
    for i in range(layers):
        if kind == "ar":
            fl.append(nf.flows.AutoregressiveRationalQuadraticSpline(d, 2, hidden))
        else:
            fl.append(nf.flows.CoupledRationalQuadraticSpline(d, 2, hidden, reverse_mask=bool(i % 2)))
        fl.append(nf.flows.LULinearPermute(d))
    m = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=False), fl)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(sigma * torch.randn(p.shape, generator=g))
    return m.cuda()


@pytest.mark.parametrize("hidden", [64, 128, 192, 256])
@pytest.mark.parametrize("d", [5, 64])
@pytest.mark.parametrize("kind", ["ar", "coupled"])
def test_fused_matches_fp32_path(kind, d, hidden):
    torch.set_grad_enabled(False)
    try:
        model = _model(kind, d, hidden)
        B = 4096 + 37   # a ragged last tile
        x = (torch.randn(B, d, generator=torch.Generator().manual_seed(7)) * 1.5).cuda()

        # density direction
        z, ld = model.inverse_and_log_det(x)
        assert model._stack().fused_layers() == list(range(len(model.flows))), "every layer must run fused"
        lp = model.log_prob(x)
        NativeFlow.use_tensor_cores = False
        z32, ld32 = model.inverse_and_log_det(x)
        lp32 = model.log_prob(x)
        NativeFlow.use_tensor_cores = True
        lpn, lp32n = lp.cpu().numpy().astype(np.float64), lp32.cpu().numpy().astype(np.float64)
        disc = np.abs(lpn - lp32n) / (np.abs(lp32n) + 1e-12)
        assert np.mean(disc < RTOL) > 0.999 and disc.max() < 5e-4, disc.max()   # two fp32 paths, neither is truth
        dz = (z - z32).abs().max(dim=1).values.cpu().numpy()
        assert np.mean(dz < 2e-4) > 0.995 and dz.max() < 2e-3, dz.max()
        dl = (ld - ld32).abs().cpu().numpy()
        assert np.mean(dl < 2e-3) > 0.995 and dl.max() < 2e-2, dl.max()

        # sampling direction (autoregressive blocks: D conditioner passes per block inside the kernel)
        xs, lds = model.forward_and_log_det(z32)
        NativeFlow.use_tensor_cores = False
        xs32, lds32 = model.forward_and_log_det(z32)
        NativeFlow.use_tensor_cores = True
        dx = (xs - xs32).abs().max(dim=1).values.cpu().numpy()
        # chained spline inversions amplify fp32 round-off on a few rows (the reference's own fp32 run does the same)
        assert np.mean(dx < 2e-3) > 0.995 and dx.max() < 0.1, dx.max()
        dls = (lds - lds32).abs().cpu().numpy()
        assert np.median(dls) < 2e-3 and dls.max() < 0.1, dls.max()
        ex = (xs32 - x).abs().max(dim=1).values.cpu().numpy()
        assert np.median(ex) < 2e-3   # the fp32 round trip itself is sound
    finally:
        torch.set_grad_enabled(True)
