"""Mint goldens of the flow-VAE from the REAL reference (a checkout found by oracle/reference.py, no GPU needed): fp64
autograd of the VAE notebook's loss mean(log_q) - mean(log_p) through NormalizingFlowVAE.forward, with the encoder's
standard-normal draws stored and replayed.
    python tests/golden/make_vae_grads.py [case ...]
Writes tests/golden/grads_vae_<case>.npz (models in tests/helpers_vae.py), each holding
    init__<key>   the state_dict as constructed under the case's seed (pins the construction order)
    sd__<key>     the one after perturb_case -- for case e, too large to store, sd_sha256 instead: the digests of the
                  float32 arrays that helpers_vae.build + perturb_case rebuild with this package's constructors
    x, eps, z, log_q, log_p, loss
    g__<name> (or, above MAX_WHOLE entries, gv__ / gu__ / gn__ projections) for every parameter
    enc_log_prob  q0.log_prob(z0, x) at the encoder's draws z0
    dec_forward   decoder(z) at the flows' output (dec_forward_std: the Gaussian decoder's std)
The forward runs with float64 as torch's default dtype, so that the reference's Dirac log_q (torch.zeros) is fp64."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_conditional_grads import MAX_WHOLE, projections  # noqa: E402
from make_golden import nf, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
import helpers_vae as V  # noqa: E402


def mint(name):
    model = V.build(nf, name)
    out = {"torch_version": torch.__version__}
    if name != "e":
        for k, v in model.state_dict().items():
            out["init__" + k] = v.detach().clone().numpy()
    V.perturb_case(model, name)
    sd = model.state_dict()
    if name == "e":
        out["sd_sha256"] = np.array(json.dumps({k: sha256(v.detach().numpy()) for k, v in sd.items()}))
    else:
        for k, v in sd.items():
            out["sd__" + k] = v.detach().numpy()
    x, eps = V.data(name), V.draws(name)
    out["x"], out["eps"] = x.numpy(), eps.numpy()
    md = model.double()
    if name == "b":
        md.prior = md.prior.double()
    else:
        md.prior = V.mvn(V.LATENT[name])
        md.prior = torch.distributions.MultivariateNormal(md.prior.loc.double(), md.prior.covariance_matrix.double())
    randn = torch.randn
    torch.randn = lambda *a, **k: eps.double().clone()
    torch.set_default_dtype(torch.float64)
    try:
        xd = x.double()
        z, log_q, log_p = md(xd, V.SHAPES[name][1])
        loss = torch.mean(log_q) - torch.mean(log_p)
        loss.backward()
        with torch.no_grad():
            z0, _ = md.q0(xd, V.SHAPES[name][1])
            out["enc_log_prob"] = md.q0.log_prob(z0, xd).numpy()
            if md.decoder is not None:
                dec = md.decoder(z.reshape(-1, z.shape[2]))
                if isinstance(dec, tuple):
                    out["dec_forward"], out["dec_forward_std"] = dec[0].numpy(), dec[1].numpy()
                else:
                    out["dec_forward"] = dec.numpy()
    finally:
        torch.randn = randn
        torch.set_default_dtype(torch.float32)
    out["z"], out["log_q"], out["log_p"] = z.detach().numpy(), log_q.detach().numpy(), log_p.detach().numpy()
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
    save_parts(f"grads_vae_{name}", out)
    print("wrote", name, loss.item())


if __name__ == "__main__":
    for c in sys.argv[1:] or V.CASES:
        mint(c)
