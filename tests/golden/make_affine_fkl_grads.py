"""Mint gradient goldens of forward-KL training through the affine family (the density direction of MaskedAffineFlow,
ActNorm / AffineConstFlow, AffineCouplingBlock and Permute) from the REAL reference (a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `forward_kld` on stored inputs, the gradient of every parameter.
    python tests/golden/make_affine_fkl_grads.py [case ...]
Writes tests/golden/grads_fkl_<case>.npz with the storage rules of make_affine_rkl_grads.py (models in
tests/helpers_affine_fkl.py):
    colab    examples/real_nvp_colab.ipynb: 32 x [AffineCouplingBlock(MLP([1, 64, 64, 2])), Permute(2, 'swap')]
    realnvp  case m of make_affine_rkl_grads.py: 8 x [MaskedAffineFlow(MLP([2, 4, 2]) t and s), ActNorm(2)]
    every    case p: every op variant at D = 5 with a trainable DiagGaussian base
    mixed    MaskedAffineFlow + ActNorm + AutoregressiveRationalQuadraticSpline(2, 1, 32) + LULinearPermute +
             AffineCouplingBlock(sigmoid) + Permute: affine groups on both sides of a spline / LU pair
    cond     case q: ConditionalNormalizingFlow, forward_kld(x, context) (the reference's affine layers take no context
             argument: their inverse is wrapped to drop it)
Weights are perturbed off the zero init (sigma 0.05, 0.01 for the 32 colab blocks, seeded) and every ActNorm is marked
initialised."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_affine_fkl as F  # noqa: E402


def mint(name):
    model = F.build(nf, name)
    perturb(model, F.SIGMA.get(name, 0.05), 400 + F.SEEDS[name])
    F.mark_actnorm_done(model)
    if name == "cond":
        for f in model.flows:
            if isinstance(f, (nf.flows.MaskedAffineFlow, nf.flows.ActNorm)):
                f.inverse = (lambda inv: lambda z, context=None: inv(z))(f.inverse)
    x = F.data(name)
    ctx = F.context_of() if name == "cond" else None
    out = {"torch_version": torch.__version__, "x": x.numpy()}
    if ctx is not None:
        out["context"] = ctx.numpy()
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    loss = md.forward_kld(x.double(), context=ctx.double()) if ctx is not None else md.forward_kld(x.double())
    loss.backward()
    out["loss"] = np.array(loss.item())
    for n, p in md.named_parameters():
        if not p.requires_grad:
            continue
        g = p.grad
        assert g is not None, n
        if g.numel() <= MAX_WHOLE:
            out["g__" + n] = g.numpy()
        else:
            v, u = projections(n, tuple(g.shape))
            G = g.reshape(g.shape[0], -1)
            out["gv__" + n], out["gu__" + n] = (G @ v).numpy(), (u @ G).numpy()
            out["gn__" + n] = np.array(G.norm().item())
    save_parts(f"grads_fkl_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or F.CASES:
        mint(c)
