"""Shared by tests/golden/make_vae_grads.py (run against the reference) and tests/test_vae_training.py (run against this
package): the flow-VAE cases a-e, their data and stored encoder draws, and an fp64 torch restatement of
NormalizingFlowVAE.forward on a state_dict.  `nf` is whichever package is passed in; only constructor arguments the
reference and this package share are used.

    a       NNDiagGaussian(MLP([12, 16, 8])) -> 6 x Planar((4,)) -> NNBernoulliDecoder(MLP([4, 16, 12])),
            MultivariateNormal prior, B = 5, S = 3
    b       as a with Radial flows, a zero-initialised decoder (every score exactly 0), a DiagGaussian(4) prior, S = 1
    c       examples/vae.ipynb's RealNVP option scaled down: 6 x MaskedAffineFlow(b, MLP([4, 4]), MLP([4, 4])) with an
            NNDiagGaussianDecoder on real-valued x
    d       ConstDiagGaussian + 4 x Planar((4,)), no decoder
    d_dirac Dirac + 2 x Planar((4,)), no decoder
    e       examples/vae.ipynb's model as written (784-512-256-80, 40 x Planar((40,)), 40-256-512-784 Bernoulli), B = 4,
            S = 32"""
import math

import torch

CASES = ["a", "b", "c", "d", "d_dirac", "e"]
SEEDS = {"a": 41, "b": 42, "c": 43, "d": 44, "d_dirac": 45, "e": 46}
SHAPES = {"a": (5, 3), "b": (5, 1), "c": (5, 3), "d": (5, 3), "d_dirac": (5, 3), "e": (4, 32)}   # (B, S)
DATA = {"a": 12, "b": 12, "c": 6, "d": 4, "d_dirac": 4, "e": 784}
LATENT = {"a": 4, "b": 4, "c": 4, "d": 4, "d_dirac": 4, "e": 40}
# parameters left at their init by perturb_case: the zero-initialised decoder's last layer of case b
KEEP = {"b": ("decoder.net.net.2.weight", "decoder.net.net.2.bias")}
SIGMA = 0.05


def mvn(d, device=None):
    return torch.distributions.MultivariateNormal(torch.zeros(d, device=device), torch.eye(d, device=device))


def build(nf, name, device=None):
    torch.manual_seed(SEEDS[name])
    d = LATENT[name]
    D = nf.distributions
    if name in ("a", "b"):
        enc = D.NNDiagGaussian(nf.nets.MLP([12, 16, 2 * d]))
        flows = [nf.flows.Planar((d,)) if name == "a" else nf.flows.Radial((d,)) for _ in range(6)]
        dec = D.NNBernoulliDecoder(nf.nets.MLP([d, 16, 12], init_zeros=(name == "b")))
        prior = mvn(d, device) if name == "a" else D.DiagGaussian(d)
        return nf.NormalizingFlowVAE(prior, enc, flows, dec)
    if name == "c":
        enc = D.NNDiagGaussian(nf.nets.MLP([6, 16, 2 * d]))
        b = torch.tensor(d // 2 * [0, 1] + d % 2 * [0])
        flows = []
        for i in range(6):
            s = nf.nets.MLP([d, d])
            t = nf.nets.MLP([d, d])
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
        dec = D.NNDiagGaussianDecoder(nf.nets.MLP([d, 16, 12]))
        return nf.NormalizingFlowVAE(mvn(d, device), enc, flows, dec)
    if name == "d":
        enc = D.encoder.ConstDiagGaussian(torch.linspace(-0.5, 0.5, d), torch.linspace(0.6, 1.4, d))
        return nf.NormalizingFlowVAE(mvn(d, device), enc, [nf.flows.Planar((d,)) for _ in range(4)])
    if name == "d_dirac":
        return nf.NormalizingFlowVAE(mvn(d, device), D.Dirac(), [nf.flows.Planar((d,)) for _ in range(2)])
    enc = D.NNDiagGaussian(nf.nets.MLP([784, 512, 256, 2 * d]))     # e: the notebook
    dec = D.NNBernoulliDecoder(nf.nets.MLP([d, 256, 512, 784]))
    return nf.NormalizingFlowVAE(mvn(d, device), enc, [nf.flows.Planar((d,)) for _ in range(40)], dec)


def perturb_case(model, name):
    """Every parameter off its init (sigma 0.05, seeded), except those of KEEP."""
    g = torch.Generator().manual_seed(600 + SEEDS[name])
    with torch.no_grad():
        for n, p in model.named_parameters():
            step = SIGMA * torch.randn(p.shape, generator=g, dtype=p.dtype)
            if n not in KEEP.get(name, ()):
                p.add_(step)


def data(name):
    """x [B, n]: binarised for the Bernoulli decoders, real-valued otherwise."""
    B = SHAPES[name][0]
    g = torch.Generator().manual_seed(700 + SEEDS[name])
    x = torch.rand(B, DATA[name], generator=g)
    return (x > 0.5).float() if name in ("a", "b", "e") else 2 * x - 1


def draws(name):
    """The stored standard-normal encoder draws eps [B, S, d] (float32)."""
    B, S = SHAPES[name]
    g = torch.Generator().manual_seed(800 + SEEDS[name])
    return torch.randn(B, S, LATENT[name], generator=g)


# ---- fp64 restatement -------------------------------------------------------------------------------------------------
def _mlp(P, prefix, h):
    idx = sorted({int(k[len(prefix):].split(".")[0]) for k in P if k.startswith(prefix) and k.endswith(".weight")})
    for n, i in enumerate(idx):
        h = h @ P[f"{prefix}{i}.weight"].T + P[f"{prefix}{i}.bias"]
        if n + 1 < len(idx):
            h = torch.relu(h)
    return h


def _log_sig(a):
    return -torch.relu(-a) - torch.log(1 + torch.exp(-torch.abs(a)))


def planar(z, u, w, b):
    lin = torch.sum(w * z, 1, keepdim=True) + b
    inner = torch.sum(w * u)
    u = u + (torch.log(1 + torch.exp(inner)) - 1 - inner) * w / torch.sum(w ** 2)
    return z + u * torch.tanh(lin), torch.log(torch.abs(1 + torch.sum(w * u) / torch.cosh(lin.reshape(-1)) ** 2))


def radial(z, z_0, alpha, beta):
    beta = torch.log(1 + torch.exp(beta)) - torch.abs(alpha)
    dz = z - z_0
    r = torch.linalg.vector_norm(dz, dim=1, keepdim=True)
    h = beta / (torch.abs(alpha) + r)
    h_ = -beta * r / (torch.abs(alpha) + r) ** 2
    return z + h * dz, ((z.shape[1] - 1) * torch.log(1 + h) + torch.log(1 + h + h_)).reshape(-1)


def masked_affine(z, P, p):
    b = P[p + "b"]
    zm = b * z
    scale, trans = _mlp(P, p + "s.net.", zm), _mlp(P, p + "t.net.", zm)
    return zm + (1 - b) * (z * torch.exp(scale) + trans), torch.sum((1 - b) * scale, 1)


def encoder_draw(name, P, x, eps):
    """(z0 [B, S, d], log_q [B, S]) of the encoder."""
    d = eps.shape[2]
    c = -0.5 * d * math.log(2 * math.pi)
    if name == "d_dirac":
        return x.unsqueeze(1).repeat(1, eps.shape[1], 1), x.new_zeros(eps.shape[:2])
    if name == "d":
        loc, scale = P["q0.loc"], P["q0.scale"]
        return loc + scale * eps, c - torch.sum(torch.log(scale) + 0.5 * eps ** 2, 2)
    ms = _mlp(P, "q0.net.net.", x)
    n = ms.shape[1] // 2
    mean, std = ms[:, :n].unsqueeze(1), torch.exp(0.5 * ms[:, n:2 * n].unsqueeze(1))
    return mean + std * eps, c - torch.sum(torch.log(std) + 0.5 * eps ** 2, 2)


def encoder_log_prob(name, P, z, x):
    """q0.log_prob(z, x) for z [B, S, d]."""
    d = z.shape[2]
    c = -0.5 * d * math.log(2 * math.pi)
    if name == "d_dirac":
        return z.new_zeros(z.shape[:2])
    if name == "d":
        loc, scale = P["q0.loc"], P["q0.scale"]
        return c - torch.sum(torch.log(scale) + 0.5 * ((z - loc) / scale) ** 2, 2)
    ms = _mlp(P, "q0.net.net.", x)
    n = ms.shape[1] // 2
    mean, var = ms[:, :n].unsqueeze(1), torch.exp(ms[:, n:2 * n].unsqueeze(1))
    return c - 0.5 * torch.sum(torch.log(var) + (z - mean) ** 2 / var, 2)


def decoder_forward(name, P, z):
    out = _mlp(P, "decoder.net.net.", z)
    if name == "c":
        n = out.shape[1] // 2
        return out[:, :n], torch.exp(0.5 * out[:, n:])
    return torch.sigmoid(out)


def decoder_log_prob(name, P, x, z):
    out = _mlp(P, "decoder.net.net.", z)
    x = x.repeat_interleave(len(z) // len(x), 0)
    if name == "c":
        n = out.shape[1] // 2
        mean, lv = out[:, :n], out[:, n:]
        return -0.5 * z.shape[1] * math.log(2 * math.pi) - 0.5 * torch.sum(lv + (x - mean) ** 2 / torch.exp(lv), 1)
    return torch.sum(x * _log_sig(out) + (1 - x) * _log_sig(-out), 1)


def flows_forward(name, P, z):
    ld = z.new_zeros(z.shape[0])
    for i in range(len({k.split(".")[1] for k in P if k.startswith("flows.")})):
        p = f"flows.{i}."
        if name == "b":
            z, l = radial(z, P[p + "z_0"], P[p + "alpha"], P[p + "beta"])
        elif name == "c":
            z, l = masked_affine(z, P, p)
        else:
            z, l = planar(z, P[p + "u"], P[p + "w"], P[p + "b"])
        ld = ld + l
    return z, ld


def prior_log_prob(name, P, z):
    d = z.shape[1]
    if name == "b":
        loc, ls = P["prior.loc"], P["prior.log_scale"]
        return -0.5 * d * math.log(2 * math.pi) - torch.sum(ls + 0.5 * ((z - loc) / torch.exp(ls)) ** 2, 1)
    return -0.5 * d * math.log(2 * math.pi) - 0.5 * torch.sum(z ** 2, 1)


def restate(name, P, x, eps):
    """(z [B, S, d], log_q [B, S], log_p [B, S], loss) of NormalizingFlowVAE.forward with parameters P (name -> tensor)
    and encoder draws eps; loss = mean(log_q) - mean(log_p), the notebook's."""
    B, S, d = eps.shape
    z, log_q = encoder_draw(name, P, x, eps)
    z, log_q = z.reshape(B * S, d), log_q.reshape(-1)
    z, ld = flows_forward(name, P, z)
    log_q = log_q - ld
    log_p = prior_log_prob(name, P, z)
    if name not in ("d", "d_dirac"):
        log_p = log_p + decoder_log_prob(name, P, x, z)
    log_q, log_p = log_q.view(B, S), log_p.view(B, S)
    return z.view(B, S, d), log_q, log_p, torch.mean(log_q) - torch.mean(log_p)
