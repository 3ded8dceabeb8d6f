"""Mint gradient goldens of reverse-KL training through the affine family (the sampling direction of MaskedAffineFlow,
ActNorm / AffineConstFlow, AffineCouplingBlock and Permute) from the REAL reference (a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `reverse_kld` / `reverse_alpha_div`, the gradient of every
parameter.
    python tests/golden/make_affine_rkl_grads.py [case ...]
Writes tests/golden/grads_rkl_<case>.npz with the storage rules of make_reverse_kld_grads.py (cases h-l), whose
lettering these continue (models in tests/helpers_affine_rkl.py):
    m   NormalizingFlow(DiagGaussian(2), 8 x [MaskedAffineFlow(MLP([2, 4, 2]) t and s), ActNorm(2)], TwoModes(2, 0.1)):
          examples/real_nvp.ipynb scaled down, reverse_kld(beta=0.5)
    n   the same model, reverse_alpha_div(dreg=True, alpha=1)
    o   examples/augmented_flow.ipynb scaled down (4 x [MaskedAffineFlow(MLP([4, 16, 4])), ActNorm(4)], target
          TwoIndependent(TwoMoons(), DiagGaussian(2))), reverse_kld(score_fn=False): the target's DiagGaussian is trained
    p   D = 5: AffineCouplingBlocks with exp / sigmoid / sigmoid_inv / no scale and channel / channel_inv splits, Permute
          swap and shuffle, MaskedAffineFlow with s=None and with t=None, AffineConstFlow(scale=False), ActNorm; reverse_kld
    q   ConditionalNormalizingFlow(DiagGaussian(2, trainable=False), [MaskedAffineFlow, ActNorm, AutoregressiveRational-
          QuadraticSpline(2, 1, 32, num_context_channels=4), MaskedAffineFlow, ActNorm]), reverse_kld(512, context)
          (the reference's affine layers take no context argument: their forward is wrapped to drop it)
The base's draws are stored and replayed (helpers_rkl.replay_forward); weights are perturbed off the zero init (sigma
0.05, seeded) and every ActNorm is marked initialised.  m and o also store the reference target's log_prob at the base
draws (p_log_prob), which pins TwoModes and TwoIndependent."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_affine_rkl as A  # noqa: E402
import helpers_rkl as R  # noqa: E402


def loss_of(name, model, n, context):
    if name == "m":
        return model.reverse_kld(n, beta=0.5)
    if name == "n":
        return model.reverse_alpha_div(n, alpha=1, dreg=True)
    if name == "o":
        return model.reverse_kld(n, score_fn=False)
    if name == "p":
        return model.reverse_kld(n)
    return model.reverse_kld(n, context=context)


def mint(name):
    model = A.build(nf, name)
    perturb(model, 0.05, 300 + A.SEEDS[name])
    A.mark_actnorm_done(model)
    if name == "q":
        for f in model.flows:
            if isinstance(f, (nf.flows.MaskedAffineFlow, nf.flows.ActNorm)):
                f.forward = (lambda fwd: lambda z, context=None: fwd(z))(f.forward)
    eps = A.draws(name)
    ctx = A.context_of() if name == "q" else None
    out = {"torch_version": torch.__version__, "eps": eps.numpy()}
    if ctx is not None:
        out["context"] = ctx.numpy()
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    if name in ("m", "o"):
        out["p_log_prob"] = md.p.log_prob(eps.double()).detach().numpy()
    md.q0.forward = R.replay_forward(md.q0, eps.double())
    loss = loss_of(name, md, eps.shape[0], ctx.double() if ctx is not None else None)
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
    save_parts(f"grads_rkl_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or list(A.SEEDS):
        mint(c)
