"""Mint gradient goldens of reverse-KL training of coupled spline + LULinearPermute stacks from the REAL reference (a
checkout found by oracle/reference.py, no GPU needed): fp64 autograd of `reverse_kld` / `reverse_alpha_div`, the
gradient of every parameter.
    python tests/golden/make_coupled_rkl_grads.py [case ...]
Writes tests/golden/grads_rkl_<case>.npz (continued in .2.npz, ... below 1 MB), with the storage rules of
make_reverse_kld_grads.py (cases h-v; these continue the lettering); models in tests/helpers_coupled_rkl.py:
    w   NormalizingFlow(DiagGaussian(6), 4 x [CoupledRationalQuadraticSpline(6, 2, 64, reverse_mask=i % 2),
          LULinearPermute(6)], p=Target6), reverse_kld(512); eight draws lie beyond the tail bound 3 in every feature
    x   the same model and draws, reverse_alpha_div(dreg=True, alpha=1): the density pass re-evaluated with parameter
          gradients switched off
    y   2 x [CoupledRationalQuadraticSpline(64, 2, 256, reverse_mask=i % 2), LULinearPermute(64)] on DiagGaussian(64),
          reverse_kld(256) against Target64 (the benchmark's shapes; gradients stored as projections); the 256 draws are
          the first candidates at least 1e-4 (relative) from every conditioner ReLU kink of the fp64 pass
    z   3 x CoupledRationalQuadraticSpline(5, 1, 32, reverse_mask=i % 2) on a trainable DiagGaussian(5),
          reverse_kld(512, score_fn=False)
Weights are perturbed off the identity init (sigma 0.05, seeded).  Every file carries the float32 state_dict (sd__*,
exact in fp64), sd_sha256, eps, loss and the gradients: whole (g__<name>) when at most 4096 entries, else gv__ = G v,
gu__ = u G, gn__ = |G| (tests/helpers_glow_grads.py grad_projections)."""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_coupled_rkl as H  # noqa: E402
import helpers_rkl as R  # noqa: E402


def relu_margin(model, z):
    """Per row, the smallest |ReLU input| of any conditioner along the sampling pass, relative to that input's median."""
    m = torch.full((z.shape[0],), float("inf"), dtype=z.dtype)

    def hook(mod, inp):
        nonlocal m
        a = inp[0].abs()
        m = torch.minimum(m, (a / a.median()).min(1).values)
    hooks = [mod.register_forward_pre_hook(hook) for mod in model.modules() if isinstance(mod, torch.nn.ReLU)]
    with torch.no_grad():
        model.forward(z)
    for h in hooks:
        h.remove()
    return m


def mint(name):
    model = H.build(nf, name)
    perturb(model, 0.05, 200 + H.SEEDS[name])
    eps = H.draws(name)
    if name == "y":   # 256 rows at least 1e-4 (relative) from every ReLU kink of the fp64 pass: a float32 pass takes the
        # same side of each kink, so the stored gradients hold at float32 accuracy
        md = copy.deepcopy(model).double()
        z, _ = R.replay_forward(md.q0, eps.double())(eps.shape[0])
        eps = eps[relu_margin(md, z) > 1e-4][:256]
        assert eps.shape[0] == 256
    out = {"torch_version": torch.__version__, "eps": eps.numpy()}
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    md.q0.forward = R.replay_forward(md.q0, eps.double())
    loss = H.loss_of(name, md, eps.shape[0])
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
    for c in sys.argv[1:] or list(H.SEEDS):
        mint(c)
