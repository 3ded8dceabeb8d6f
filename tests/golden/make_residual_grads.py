"""Mint gradient goldens of the residual flow's training pass from the REAL reference (normflows 1.7.3; a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `NormalizingFlow.forward_kld(x)` (or of a weighted log_prob sum),
x.grad and every parameter gradient.
    python tests/golden/make_residual_grads.py [case ...]
Writes tests/golden/grads_res_<case>.npz (split into <name>.2.npz, ... below 1 MB).  Cases:
    d2_geo, d4_geo    3 x [Residual(LipschitzMLP([d, 32, 32, d])), ActNorm(d)], trainable DiagGaussian, training mode,
                      geometric truncation (the Neumann-series gradient)
    d2_poisson, d4_poisson   the same with n_dist="poisson"
    d2_brute          brute_force=True, d = 2, training mode (exact 2 x 2 log-det)
    d2_eval, d4_eval  eval mode: exact log-det (d = 2), basic estimator with no log-det gradient (d = 4)
    d4_weighted       loss (log_prob(x) * wts).sum() with non-uniform wts: pins that row 0's cotangent scales the
                      Neumann gradient of every row (residual.py:335)
    c5                BASELINE config 5's shape, 16 x Residual(LipschitzMLP([2, 128, 128, 128, 2])), 1024 rows
The ActNorm layers are initialised (one no-grad pass with the real RNG) before the state_dict is taken, so the minted
pass consumes only the injected draws: np.random.geometric / np.random.poisson return n_inj[call] and
torch.randn_like returns eps[call], per estimator call in call order (flows last to first; the exact path draws
nothing).  Every file carries spec, the float32 state_dict (exact in fp64), x, n_inj, eps, cot (the per-row cotangent
of log_prob: -1/B for forward_kld), sd_sha256 / x_sha256 and the gradients: whole when at most 4096 entries, else
gradv__ = G v, gradu__ = u G, gnorm__ = |G| (tests/helpers_glow_grads.py grad_projections)."""
import json
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


def build(d, widths, n_blocks, actnorm, trainable_base, init_zeros=False, **res_kw):
    flows = []
    for _ in range(n_blocks):
        net = nf.nets.LipschitzMLP([d] + widths + [d], init_zeros=init_zeros, lipschitz_const=0.9)
        flows.append(nf.flows.Residual(net, reduce_memory=True, **res_kw))
        if actnorm:
            flows.append(nf.flows.ActNorm(d))
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=trainable_base), flows)
    spec = {"flows": [{"type": "actnorm"} if isinstance(f, nf.flows.ActNorm) else
                      {"type": "residual", "coeff": 0.9, "n_layers": len(widths) + 1,
                       "n_dist": res_kw.get("n_dist", "geometric"), "brute_force": res_kw.get("brute_force", False),
                       "n_exact_terms": 2, "n_power_series": None} for f in flows],
            "base_trainable": trainable_base}
    return model, spec


def mint(name, seed, d, B, training, widths=(32, 32), n_blocks=3, actnorm=True, trainable_base=True, weighted=False,
         init_zeros=False, sigma=0.4, **res_kw):
    torch.manual_seed(seed)
    np.random.seed(seed)
    model, spec = build(d, list(widths), n_blocks, actnorm, trainable_base, init_zeros, **res_kw)
    g = torch.Generator().manual_seed(seed + 1)
    x = (torch.randn(B, d, generator=g) * 1.2).float()
    with torch.no_grad():
        model.train()
        model.log_prob(x)      # ActNorm data-dependent init with the real RNG (not stored draws)
        perturb(model, sigma, seed + 2)
        nf.utils.update_lipschitz(model, 50)
    sd = {k: v.detach().numpy().copy() for k, v in model.state_dict().items()}
    n_calls = sum(1 for f in spec["flows"] if f["type"] == "residual"
                  and not ((f["brute_force"] or not training) and d == 2))
    dist = res_kw.get("n_dist", "geometric")
    n_inj = np.array([[1 + (3 * i + seed) % 4] for i in range(n_calls)])
    eps = torch.randn(max(n_calls, 1), B, d, generator=g, dtype=torch.float64)
    wts = (torch.rand(B, generator=g, dtype=torch.float64) * 2 + 0.1) if weighted else None
    cot = wts.numpy() if weighted else np.full(B, -1.0 / B)
    calls = {"n": 0, "e": 0}
    orig = np.random.geometric, np.random.poisson, torch.randn_like

    def draw_n(*a, **k):
        i = calls["n"]
        calls["n"] += 1
        return n_inj[i]

    def draw_eps(t, **k):
        j = calls["e"]
        calls["e"] += 1
        return eps[j].to(t)
    md = model.double()
    xx = x.double().requires_grad_(True)
    np.random.geometric, np.random.poisson, torch.randn_like = draw_n, draw_n, draw_eps
    try:
        md.train(training)
        lp = md.log_prob(xx)
        loss = (lp * wts).sum() if weighted else -torch.mean(lp)
        loss.backward()
    finally:
        np.random.geometric, np.random.poisson, torch.randn_like = orig
    assert calls["n"] == calls["e"] == n_calls, (calls, n_calls)
    out = {"spec": json.dumps(spec), "torch_version": torch.__version__, "training": np.asarray(training),
           "x": x.numpy(), "n_inj": n_inj, "eps": eps.numpy(), "cot": cot, "loss": loss.detach().numpy(),
           "log_prob": lp.detach().numpy(), "n_dist": np.asarray(dist),
           "x_sha256": sha256(x.numpy()), "sd_sha256": json.dumps({k: sha256(v) for k, v in sd.items()})}
    out.update({"sd__" + k: v for k, v in sd.items()})
    for k, p in [("x", xx)] + list(md.named_parameters()):
        if p.grad is None:
            continue
        if p.numel() <= MAX_WHOLE:
            out["grad__" + k] = p.grad.numpy()
        else:
            G = p.grad.reshape(p.shape[0], -1)
            v, u = projections(k, tuple(p.shape))
            out["gradv__" + k], out["gradu__" + k] = (G @ v).numpy(), (u @ G).numpy()
            out["gnorm__" + k] = np.asarray(G.norm().item())
    save_parts("grads_res_" + name, out)


CASES = {
    "d2_geo": lambda: mint("d2_geo", 61, 2, 96, True),
    "d4_geo": lambda: mint("d4_geo", 62, 4, 96, True),
    "d2_poisson": lambda: mint("d2_poisson", 63, 2, 96, True, n_dist="poisson"),
    "d4_poisson": lambda: mint("d4_poisson", 64, 4, 96, True, n_dist="poisson"),
    "d2_brute": lambda: mint("d2_brute", 65, 2, 96, True, brute_force=True),
    "d2_eval": lambda: mint("d2_eval", 66, 2, 96, False),
    "d4_eval": lambda: mint("d4_eval", 67, 4, 96, False),
    "d4_weighted": lambda: mint("d4_weighted", 68, 4, 96, True, weighted=True),
    "c5": lambda: mint("c5", 69, 2, 1024, True, widths=(128, 128, 128), n_blocks=16, actnorm=False,
                       trainable_base=False, init_zeros=True, sigma=0.05),
}

if __name__ == "__main__":
    for name in (sys.argv[1:] or list(CASES)):
        CASES[name]()
        print("wrote", name)
