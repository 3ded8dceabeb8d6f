"""Build OUR MultiscaleFlow for the Glow goldens (examples/glow.ipynb cell 2, at reduced size and at its real size)."""
import json

import numpy as np
import torch

import normflows as nf


def build_glow_small(sd=None, L_=2, K=2, hidden=32, shape=(3, 8, 8), ncls=10):
    q0, merges, flows = [], [], []
    for i in range(L_):
        fl = [nf.flows.GlowBlock(shape[0] * 2 ** (L_ + 1 - i), hidden, split_mode="channel", scale=True)
              for _ in range(K)] + [nf.flows.Squeeze()]
        flows += [fl]
        if i > 0:
            merges += [nf.flows.ImageMerge()]
            ls = (shape[0] * 2 ** (L_ - i), shape[1] // 2 ** (L_ - i), shape[2] // 2 ** (L_ - i))
        else:
            ls = (shape[0] * 2 ** (L_ + 1), shape[1] // 2 ** L_, shape[2] // 2 ** L_)
        q0 += [nf.distributions.ClassCondDiagGaussian(ls, ncls)]
    m = nf.MultiscaleFlow(q0, flows, merges)
    if sd is not None:
        m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    return m


def build_glow_c3():
    """BASELINE config 3 = examples/glow.ipynb cell 2 verbatim: L=3, K=16, hidden 256, 3x32x32, 10 classes, constructed
    under torch.manual_seed(0) like tests/golden/make_golden.py case_glow_c3."""
    torch.manual_seed(0)
    return build_glow_small(L_=3, K=16, hidden=256, shape=(3, 32, 32), ncls=10)


def glow_c3_inputs(batch=64):
    g = torch.Generator().manual_seed(1)
    x = torch.rand(batch, 3, 32, 32, generator=g)
    return x, torch.randint(10, (batch,), generator=g)


def glow_c3_state_dict(f):
    """The fp64 state_dict of tests/golden/glow_c3.npz: this package's constructors (they draw from torch's generator
    exactly like the reference's), every parameter moved by 0.02 randn (seed 2), and the entries the reference's
    data-dependent ActNorm init set taken from the golden; checked bit for bit against the golden's digests."""
    from helpers import check_digests
    model = build_glow_c3().double()
    g = torch.Generator().manual_seed(2)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=g, dtype=p.dtype))
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    sd.update({k[6:]: f[k] for k in f.files if k.startswith("init__")})
    check_digests(sd, json.loads(str(f["sd_sha256"])), "glow C3")
    return sd
