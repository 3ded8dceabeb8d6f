"""Mint goldens of the Gaussian-mixture base from the REAL reference (a checkout found by oracle/reference.py, no GPU
needed): fp64 autograd of `forward_kld` on stored inputs, the gradient of every parameter, and log_prob values.
    python tests/golden/make_mixture_grads.py [case ...]
Writes tests/golden/grads_mix_<case>.npz with the storage rules of make_affine_fkl_grads.py (models in
tests/helpers_mixture.py):
    cbd     the second model of examples/change_base_distribution.ipynb: 32 x [AffineCouplingBlock(MLP([1, 64, 64, 2])),
            Permute(2, 'swap')] on GaussianMixture(2, 2, loc, scale) as written
    nsf     2 x [AutoregressiveRationalQuadraticSpline(5, 1, 16), LULinearPermute(5)] on GaussianMixture(4, 5) with
            non-uniform weights
    loop    2 x [Residual(LipschitzMLP([2, 16, 16, 2])), ActNorm(2)] on a 3-mode mixture
    values  log_prob of the value cases of helpers_mixture.value_cases (seeded and explicit construction, far z, a weight
            whose softmax underflows, K = 1) and each case's state_dict
Weights are perturbed off their init (seeded) and every ActNorm is marked initialised.  Case loop runs in eval mode,
where the reference takes iResBlock's exact 2-D log-det instead of its stochastic estimator."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_mixture as M  # noqa: E402


def mint(name):
    model = M.build(nf, name)
    perturb(model, M.SIGMA[name], 500 + M.SEEDS[name])
    M.mark_actnorm_done(model)
    model.train(name != "loop")   # loop: the exact 2-D log-det of iResBlock (eval), not the stochastic estimator
    x = M.data(name)
    out = {"torch_version": torch.__version__, "x": x.numpy()}
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    for k, v in sd.items():
        out["sd__" + k] = v
    out["sd_sha256"] = np.array(sha256(np.concatenate([np.asarray(v, np.float64).ravel() for v in sd.values()])))
    md = model.double()
    loss = md.forward_kld(x.double())
    loss.backward()
    out["loss"] = np.array(loss.item())
    for n, p in md.named_parameters():
        if not p.requires_grad:
            continue
        g = p.grad
        if g is None:   # iResBlock.geom_p / lamb: unused by the reference's exact 2-D log-det
            assert n.endswith(("geom_p", "lamb")), n
            continue
        if g.numel() <= MAX_WHOLE:
            out["g__" + n] = g.numpy()
        else:
            v, u = projections(n, tuple(g.shape))
            G = g.reshape(g.shape[0], -1)
            out["gv__" + n], out["gu__" + n] = (G @ v).numpy(), (u @ G).numpy()
            out["gn__" + n] = np.array(G.norm().item())
    save_parts(f"grads_mix_{name}", out)
    print("wrote", name, loss.item())


def mint_values():
    out = {"torch_version": torch.__version__}
    for name, spec in M.value_cases().items():
        q = M.value_case_model(nf, spec)
        for k, v in q.state_dict().items():
            out[f"{name}__sd__{k}"] = v.detach().numpy()
        out[f"{name}__z"] = spec["z"]
        with torch.no_grad():
            out[f"{name}__log_prob"] = q.log_prob(torch.tensor(spec["z"], dtype=torch.float64)).numpy()
    save_parts("grads_mix_values", out)
    print("wrote values")


if __name__ == "__main__":
    for c in sys.argv[1:] or M.CASES + ["values"]:
        mint_values() if c == "values" else mint(c)
