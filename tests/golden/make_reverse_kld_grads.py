"""Mint gradient goldens of reverse-KL training (the sampling direction of the stand-alone spline layers) from the REAL
reference (a checkout found by oracle/reference.py, no GPU needed): fp64 autograd of `reverse_kld` /
`reverse_alpha_div`, the gradient of every parameter.
    python tests/golden/make_reverse_kld_grads.py [case ...]
Writes tests/golden/grads_rkl_<case>.npz (continued in .2.npz, ... below 1 MB), with the storage rules of
make_maf_grads.py (cases a-g are gradients of forward_kld; these continue the lettering):
    h   NormalizingFlow(UniformGaussian(2, [1], [1, 2 pi]),
          3 x CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1], num_bins=10, tail_bound=[5, pi],
          permute_mask=True), p=GaussianVonMises): examples/paper_example_nsf.ipynb scaled down, reverse_kld();
          six draws of feature 0 lie beyond its bound of 5
    i   the same model and draws, reverse_kld(score_fn=False)
    j   NormalizingFlow(DiagGaussian(5), 2 x CircularAutoregressiveRationalQuadraticSpline(5, 2, 64, [1, 3])),
          reverse_alpha_div(dreg=True, alpha=1): 4 fixed-point passes per layer and a trainable base
    k   NormalizingFlow(DiagGaussian(3), 2 x CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6,
          tail_bound=[pi, 4, 3])), reverse_kld()
    l   ConditionalNormalizingFlow(DiagGaussian(2, trainable=False), [AutoregressiveRationalQuadraticSpline,
          CoupledRationalQuadraticSpline, AutoregressiveRationalQuadraticSpline] (2, 1, 64, num_context_channels=4)),
          reverse_kld(512, context) against a context-dependent target
The base's random draws (eps, 512 rows) are stored and replayed by patching the base's `forward`
(tests/helpers_rkl.py replay_forward), so the loss is a deterministic function of the parameters.  Weights are perturbed
off the identity init (sigma 0.05, seeded).  Every file carries the float32 state_dict (sd__*, exact in fp64),
sd_sha256, eps, [context], loss and the gradients: whole (g__<name>) when at most 4096 entries, else gv__ = G v,
gu__ = u G, gn__ = |G| (tests/helpers_glow_grads.py grad_projections)."""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_rkl as R  # noqa: E402

SEEDS = {"h": 8, "i": 8, "j": 10, "k": 11, "l": 12}


def build(name):
    torch.manual_seed(SEEDS[name])
    if name in ("h", "i"):
        tb = torch.tensor([5.0, math.pi])
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1], num_bins=10, tail_bound=tb,
                                                                        permute_mask=True) for _ in range(3)]
        q0 = nf.distributions.UniformGaussian(2, [1], torch.tensor([1.0, 2 * math.pi]))
        return nf.NormalizingFlow(q0, flows, R.gaussian_von_mises(nf.distributions.Target))
    if name == "j":
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(5, 2, 64, [1, 3]) for _ in range(2)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows, R.TorusTarget5())
    if name == "k":
        tb = torch.tensor([math.pi, 4.0, 3.0])
        flows = [nf.flows.CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6, tail_bound=tb,
                                                                  reverse_mask=bool(i % 2)) for i in range(2)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(3), flows, R.TorusTarget3())
    flows = [nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 64, num_context_channels=4),
             nf.flows.CoupledRationalQuadraticSpline(2, 1, 64, num_context_channels=4),
             nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 64, num_context_channels=4)]
    return nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows, R.ContextTarget())


def loss_of(name, model, n, context):
    if name in ("h", "k"):
        return model.reverse_kld(n)
    if name == "i":
        return model.reverse_kld(n, score_fn=False)
    if name == "j":
        return model.reverse_alpha_div(n, alpha=1, dreg=True)
    return model.reverse_kld(n, context=context)


def mint(name):
    model = build(name)
    perturb(model, 0.05, 200 + SEEDS[name])
    eps = R.draws(name)
    ctx = R.context_of() if name == "l" else None
    out = {"torch_version": torch.__version__, "eps": eps.numpy()}
    if ctx is not None:
        out["context"] = ctx.numpy()
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    md.q0.forward = R.replay_forward(md.q0, eps.double())
    loss = loss_of(name, md, eps.shape[0], ctx.double() if ctx is not None else None)
    loss.backward()
    out["loss"] = np.array(loss.item())
    grads = {n: p.grad for n, p in md.named_parameters() if p.requires_grad}
    for n, g in grads.items():
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
    for c in sys.argv[1:] or list(SEEDS):
        mint(c)
