"""Mint goldens of the affine family's wide path from the REAL reference (a checkout found by oracle/reference.py, no GPU
needed): fp64 autograd of forward_kld / reverse_kld / the flow-VAE loss, the gradient of every parameter, and fp64 values
of the density and sampling directions.
    python tests/golden/make_affine_wide_grads.py [case ...]
Writes tests/golden/grads_wide_<case>.npz (models in tests/helpers_affine_wide.py) with the storage rules of
make_affine_fkl_grads.py: weights perturbed off their init, ActNorms marked initialised, base and encoder draws stored and
replayed, inputs and draws kept away from the nets' ReLU kinks (away_from_kinks).  The state_dict is pinned by its digests (sd_sha256; w17 stores it whole as sd__<key>).  Forward-KL cases also
hold log_q = log_prob(x), inverse_and_log_det(x) (inv_z, inv_ld), forward_and_log_det(x) (fwd_x, fwd_ld; not mixed64)
and flows[0]'s inverse / forward of x on its own (l0_inv_z, l0_inv_ld, l0_fwd_x, l0_fwd_ld)."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, save_parts  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_affine_wide as W  # noqa: E402
import helpers_rkl as R  # noqa: E402


def grads(out, md):
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


KINK = 1e-5


def away_from_kinks(md, run, pool, n):
    """The first n rows of `pool` whose every hidden pre-activation (the input of each LeakyReLU of the flows' nets, in
    the fp64 pass `run`) is at least KINK away from 0.  A float32 pass may take the other side of a kink than fp64 on a
    row closer than that, which moves the row's share of a weight gradient by O(1)."""
    acts = [m for m in md.flows.modules() if isinstance(m, (torch.nn.LeakyReLU, torch.nn.ReLU))]
    margins = []
    hooks = [m.register_forward_hook(lambda mod, inp, out: margins.append(inp[0].detach().abs().min(1).values))
             for m in acts]
    with torch.no_grad():
        run(pool.double())
    for h in hooks:
        h.remove()
    if not margins:
        return pool[:n]
    keep = torch.stack(margins).min(0).values >= KINK
    assert int(keep.sum()) >= n, int(keep.sum())
    return pool[keep][:n]


def mint(name):
    model = W.build(nf, name)
    W.perturb(model, name)
    out = {"torch_version": torch.__version__, "sd_sha256": np.array(W.digests(model))}
    if name == "w17":
        for k, v in model.state_dict().items():
            out["sd__" + k] = v.detach().numpy()
    md = model.double()
    if name in W.FKL:
        x = away_from_kinks(md, md.log_prob, W.data(name, 4096), 512)
        out["x"] = x.numpy()
        xd = x.double()
        with torch.no_grad():
            out["log_q"] = md.log_prob(xd).numpy()
            z, ld = md.inverse_and_log_det(xd)
            out["inv_z"], out["inv_ld"] = z.numpy(), ld.numpy()
            z, ld = md.flows[0].inverse(xd)
            out["l0_inv_z"], out["l0_inv_ld"] = z.numpy(), ld.numpy()
            z, ld = md.flows[0].forward(xd)
            out["l0_fwd_x"], out["l0_fwd_ld"] = z.numpy(), ld.numpy()
            if name != "mixed64":
                z, ld = md.forward_and_log_det(xd)
                out["fwd_x"], out["fwd_ld"] = z.numpy(), ld.numpy()
        loss = md.forward_kld(xd)
    elif name == "rnvp64_rkl":
        pool = W.draws(name, 4096)
        eps = away_from_kinks(md, lambda e: md.forward_and_log_det(md.q0.loc + torch.exp(md.q0.log_scale) * e), pool,
                              512)
        out["eps"] = eps.numpy()
        md.q0.forward = R.replay_forward(md.q0, eps.double())
        loss = md.reverse_kld(eps.shape[0])
    else:
        x, eps = W.data(name), W.draws(name)
        out["x"], out["eps"] = x.numpy(), eps.numpy()
        md.prior = torch.distributions.MultivariateNormal(torch.zeros(W.DIMS[name], dtype=torch.float64),
                                                          torch.eye(W.DIMS[name], dtype=torch.float64))
        randn = torch.randn
        torch.randn = lambda *a, **k: eps.double().clone()
        torch.set_default_dtype(torch.float64)
        try:
            z, log_q, log_p = md(x.double(), W.VAE_S)
        finally:
            torch.randn = randn
            torch.set_default_dtype(torch.float32)
        assert torch.isfinite(z).all() and torch.isfinite(log_q).all() and torch.isfinite(log_p).all()
        out["z"], out["log_q"], out["log_p"] = z.detach().numpy(), log_q.detach().numpy(), log_p.detach().numpy()
        loss = torch.mean(log_q) - torch.mean(log_p)
    loss.backward()
    out["loss"] = np.array(loss.item())
    grads(out, md)
    save_parts(f"grads_wide_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or W.CASES:
        mint(c)
