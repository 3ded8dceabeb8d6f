"""Mint gradient goldens of MaskedAffineAutoregressive's training pass from the REAL reference (a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `forward_kld` through the reference's D-pass density loop, the
gradient of every parameter, of x and of the context.
    python tests/golden/make_maf_grads.py [case ...]
Writes tests/golden/grads_cond_<case>.npz (continued in .2.npz, ... below 1 MB), with the storage rules of
make_conditional_grads.py, which mints cases a-e (this script continues its lettering and seeds):
    f   ConditionalNormalizingFlow(DiagGaussian(2, trainable=False),
          4 x [MaskedAffineAutoregressive(2, 128, context_features=4, num_blocks=2), LULinearPermute(2)])
          (examples/conditional_flow.ipynb's third model)
    g   NormalizingFlow(DiagGaussian(8), 3 x [MaskedAffineAutoregressive(8, 64, num_blocks=2), LULinearPermute(8)]):
          7 fixed-point adjoint passes per layer
Weights are perturbed off the identity init (sigma 0.05, seeded); 512 rows.  Every file carries the float32 state_dict
(sd__*, exact in fp64), x, context, sd_sha256 and the gradients: whole (g__<name>) when at most 4096 entries, else
gv__ = G v, gu__ = u G, gn__ = |G| (tests/helpers_glow_grads.py grad_projections)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)

SEEDS = {"f": 6, "g": 7}


def build(name):
    torch.manual_seed(SEEDS[name])
    flows = []
    if name == "f":
        for _ in range(4):
            flows += [nf.flows.MaskedAffineAutoregressive(2, 128, context_features=4, num_blocks=2),
                      nf.flows.LULinearPermute(2)]
        return nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows)
    for _ in range(3):
        flows += [nf.flows.MaskedAffineAutoregressive(8, 64, num_blocks=2), nf.flows.LULinearPermute(8)]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(8), flows)


def inputs(name):
    g = torch.Generator().manual_seed(100 + SEEDS[name])
    x = torch.randn(512, 2 if name == "f" else 8, generator=g) * 1.3
    ctx = torch.randn(x.shape[0], 4, generator=g) if name == "f" else None
    return x, ctx


def mint(name):
    model = build(name)
    perturb(model, 0.05, 200 + SEEDS[name])
    x, ctx = inputs(name)
    out = {"torch_version": torch.__version__, "x": x.numpy()}
    if ctx is not None:
        out["context"] = ctx.numpy()
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    xd = x.double().requires_grad_(True)
    cd = ctx.double().requires_grad_(True) if ctx is not None else None
    loss = md.forward_kld(xd, cd) if cd is not None else md.forward_kld(xd)
    loss.backward()
    out["loss"] = np.array(loss.item())
    grads = {"x": xd.grad}
    if cd is not None:
        grads["context"] = cd.grad
    grads.update({n: p.grad for n, p in md.named_parameters() if p.requires_grad})
    for n, g in grads.items():
        assert g is not None, n
        if g.numel() <= MAX_WHOLE:
            out["g__" + n] = g.numpy()
        else:
            v, u = projections(n, tuple(g.shape))
            G = g.reshape(g.shape[0], -1)
            out["gv__" + n], out["gu__" + n] = (G @ v).numpy(), (u @ G).numpy()
            out["gn__" + n] = np.array(G.norm().item())
    save_parts(f"grads_cond_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or list(SEEDS):
        mint(c)
