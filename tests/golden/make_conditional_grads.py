"""Mint gradient goldens of the stand-alone layers' training pass from the REAL reference (a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `forward_kld`, the gradient of every parameter, of x and of the
context.
    python tests/golden/make_conditional_grads.py [case ...]
Writes tests/golden/grads_cond_<case>.npz (continued in .2.npz, ... below 1 MB).  Cases (examples/conditional_flow.ipynb,
examples/circular_nsf.ipynb):
    a   ConditionalNormalizingFlow(DiagGaussian(2, trainable=False),
          4 x [AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4), LULinearPermute(2)])
    b   the same with CoupledRationalQuadraticSpline
    c   ConditionalDiagGaussian(2, MLP([4, 64, 64, 4], leaky=0.01)) under 2 x [AR spline with context, LULinearPermute]
    d   NormalizingFlow(DiagGaussian(2), 3 x CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1],
          tail_bound=tensor([5, pi]), permute_mask=True))
    e   NormalizingFlow(DiagGaussian(3), 2 x CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6,
          tail_bound=tensor([pi, 4, 3]))): the circular identity feature is not feature 0 in the first layer
Weights are perturbed off the identity init (sigma 0.05, seeded); rows: 96 (512 for c and e, whose conditioners' ReLU kinks make the fp32 gradients of 96 rows miss 2e-3 of the scale), some inputs beyond the interval
of the circular layers.  Every file carries the float32 state_dict (sd__*, exact in fp64), x, context, sd_sha256 and
the gradients: whole (g__<name>) when at most 4096 entries, else gv__ = G v, gu__ = u G, gn__ = |G|
(tests/helpers_glow_grads.py grad_projections)."""
import math
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
from helpers_glow_grads import grad_projections as projections  # noqa: E402

MAX_WHOLE = 4096
SEEDS = {"a": 1, "b": 2, "c": 3, "d": 4, "e": 5}


def build(name):
    torch.manual_seed(SEEDS[name])
    ctx = None
    if name in ("a", "b", "c"):
        flows = []
        for _ in range(4 if name != "c" else 2):
            if name == "b":
                flows.append(nf.flows.CoupledRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
            else:
                flows.append(nf.flows.AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
            flows.append(nf.flows.LULinearPermute(2))
        q0 = nf.distributions.DiagGaussian(2, trainable=False) if name != "c" else \
            nf.distributions.base.ConditionalDiagGaussian(2, nf.nets.MLP([4, 64, 64, 4], leaky=0.01))
        model = nf.ConditionalNormalizingFlow(q0, flows)
    elif name == "d":
        tb = torch.tensor([5.0, math.pi])
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1], tail_bound=tb, permute_mask=True)
                 for _ in range(3)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows)
    else:
        tb = torch.tensor([math.pi, 4.0, 3.0])
        flows = [nf.flows.CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6, tail_bound=tb,
                                                                  reverse_mask=bool(i % 2)) for i in range(2)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(3), flows)
    return model


def inputs(name):
    g = torch.Generator().manual_seed(100 + SEEDS[name])
    d = 3 if name == "e" else 2
    x = torch.randn(512 if name in ("c", "e") else 96, d, generator=g) * 1.3
    if name in ("d", "e"):
        x[:6] *= 4.0
    ctx = torch.randn(x.shape[0], 4, generator=g) if name in ("a", "b", "c") else None
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
    print("wrote", name, float(loss))


if __name__ == "__main__":
    for c in sys.argv[1:] or list(SEEDS):
        mint(c)
