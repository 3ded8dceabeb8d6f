"""Mint gradient goldens of reverse-KL training through planar and radial flows from the REAL reference (a checkout
found by oracle/reference.py, no GPU needed): fp64 autograd of the loss, the gradient of every parameter.
    python tests/golden/make_planar_rkl_grads.py [case ...]
Writes tests/golden/grads_rkl_<case>.npz with the storage rules of make_reverse_kld_grads.py, continuing the lettering
of make_affine_rkl_grads.py (models in tests/helpers_planar_rkl.py):
    r   8 x Planar((2,)) on DiagGaussian(2), TwoModes(2, 0.1): examples/planar.ipynb scaled down, reverse_kld(beta=0.5)
    s   8 x Radial((2,)), Smiley(0.15), reverse_kld; also the five comparison-notebook targets' log_prob at the base
        draws (p_log_prob__<name>)
    t   6 x Planar((5,), act="leaky_relu"), a 5-D Gaussian target, reverse_kld(score_fn=False) (the density direction)
    u   the same model, forward_kld on stored data
    v   D = 40, 10 x [Planar((40,)), Radial((40,))], a 40-D Gaussian target, reverse_kld: the VAE notebook's latent size
Every case stores the state_dict as constructed under its seed (init__<key>), which pins the initialisation order, and
the one after perturbing every parameter off its init (sigma 0.05, seeded; sd__<key>).  The base's draws are stored and
replayed."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_planar_rkl as P  # noqa: E402


def mint(name):
    model = P.build(nf, name)
    out = {"torch_version": torch.__version__}
    for k, v in model.state_dict().items():
        out["init__" + k] = v.detach().clone().numpy()
    perturb(model, 0.05, 400 + P.SEEDS[name])
    eps = P.draws(name)
    out["eps"] = eps.numpy()
    for k, v in model.state_dict().items():
        out["sd__" + k] = v.detach().numpy()
    md = model.double()
    if name == "s":
        for tn, t in P.notebook_targets(nf).items():
            out["p_log_prob__" + tn] = t.log_prob(eps.double()).detach().numpy()
    x = None
    if name == "u":
        x = P.data()
        out["x"] = x.numpy()
        x = x.double()
    md.q0.forward = P.replay_forward(md.q0, eps.double())
    loss = P.loss_of(name, md, eps.shape[0], x)
    loss.backward()
    out["loss"] = np.array(loss.item())
    for n, p in md.named_parameters():
        g = p.grad
        assert g is not None, n
        if g.numel() <= MAX_WHOLE:
            out["g__" + n] = g.numpy()
        else:
            v, u = projections(n, tuple(g.shape))
            G = g.reshape(g.shape[0], -1)
            out["gv__" + n], out["gu__" + n] = (G @ v).numpy(), (u @ G).numpy()
            out["gn__" + n] = np.array(G.norm().item())
    save_parts(f"grads_rkl_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or list(P.SEEDS):
        mint(c)
