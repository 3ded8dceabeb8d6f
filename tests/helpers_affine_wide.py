"""Shared by tests/golden/make_affine_wide_grads.py (run against the reference) and tests/test_affine_wide.py (run against
this package): the wide-path cases of the affine family, their stored inputs, and the parameter perturbation.  `nf` is
whichever package is passed in; only constructor arguments the reference and this package share are used, and the
constructors draw from torch's generator in the same order in both, so that a case's state_dict is pinned by digests
instead of being stored (w17 stores it: Permute's shuffle is drawn by the constructor).

    w17        every op variant at D = 17: MaskedAffineFlow with both nets (t with LeakyReLU 0.2), s only and t only,
               ActNorm, AffineCouplingBlock exp / sigmoid / sigmoid_inv / no scale over both split modes, Permute swap
               and shuffle; a trainable DiagGaussian base; forward KL
    w2wide     examples/real_nvp_colab.ipynb's architecture with MLP([1, 256, 256, 2]) param maps (32 blocks); forward KL
    rnvp64     8 x [MaskedAffineFlow(alternating b, MLP([64, 256, 256, 64]) for t and s), ActNorm(64)], the flows'
               parameters scaled by 0.1; forward KL
    rnvp64_rkl the same model unscaled, reverse_kld against an 8-mode 64-D GaussianMixture target, base draws replayed
    mixed64    wide affine groups on both sides of AutoregressiveRationalQuadraticSpline(64, 1, 64) + LULinearPermute(64);
               forward KL
    vae40      examples/vae.ipynb's RealNVP option (40 features, 40 MaskedAffineFlows with MLP([40, 40]) nets, 784-512-
               256-80 encoder, 40-256-512-784 Bernoulli decoder), its flows' parameters scaled by 0.01 (then moved by
               0.005 sigma) so that every value is finite (the notebook's default
               initialisation overflows exp(s) in the reference too); B = 4, S = 32, encoder draws replayed"""
import hashlib
import json

import numpy as np
import torch

CASES = ["w17", "w2wide", "rnvp64", "rnvp64_rkl", "mixed64", "vae40"]
FKL = ["w17", "w2wide", "rnvp64", "mixed64"]
SEEDS = {"w17": 51, "w2wide": 52, "rnvp64": 53, "rnvp64_rkl": 53, "mixed64": 55, "vae40": 56}
DIMS = {"w17": 17, "w2wide": 2, "rnvp64": 64, "rnvp64_rkl": 64, "mixed64": 64, "vae40": 40}
SIGMA = {"w2wide": 0.01}   # 32 blocks at 0.05 overflow the log-det in float32 (as for real_nvp_colab)
VAE_B, VAE_S = 4, 32
FLOW_SIGMA = 0.005   # vae40: 40 layers of exp(s) stay finite on the encoder's draws
# the flows' parameters scaled before the perturbation: vae40's 40 layers, and rnvp64's default-initialised nets, whose
# density direction overflows exp(-s) on the stored data in the reference as well
FLOW_SCALE = {"vae40": 0.01, "rnvp64": 0.1}


def _alt(D):
    return torch.tensor([float(j % 2 == 0) for j in range(D)])


def build(nf, name):
    torch.manual_seed(SEEDS[name])
    D = DIMS[name]
    if name == "w17":
        mlp = lambda i, o, leaky=0.0: nf.nets.MLP([i, 32, o], leaky=leaky)
        b = _alt(D)
        h = (D + 1) // 2
        flows = [nf.flows.MaskedAffineFlow(b, mlp(D, D, 0.2), mlp(D, D)), nf.flows.ActNorm(D),
                 nf.flows.MaskedAffineFlow(1 - b, None, mlp(D, D)), nf.flows.Permute(D, "shuffle"),
                 nf.flows.MaskedAffineFlow(b, mlp(D, D), None)]
        for k, (scale, smap, split) in enumerate([(True, "exp", "channel"), (True, "sigmoid", "channel_inv"),
                                                  (True, "sigmoid_inv", "channel"), (False, "exp", "channel_inv")]):
            n1 = h if split == "channel" else D - h
            flows.append(nf.flows.AffineCouplingBlock(mlp(n1, (2 if scale else 1) * (D - n1)), scale, smap, split))
            if k == 1:
                flows.append(nf.flows.Permute(D, "swap"))
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows)
    if name == "w2wide":
        flows = []
        for _ in range(32):
            flows += [nf.flows.AffineCouplingBlock(nf.nets.MLP([1, 256, 256, 2], init_zeros=True)),
                      nf.flows.Permute(2, mode="swap")]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows)
    if name in ("rnvp64", "rnvp64_rkl"):
        flows = []
        for i in range(8):
            s, t = nf.nets.MLP([D, 256, 256, D]), nf.nets.MLP([D, 256, 256, D])
            flows += [nf.flows.MaskedAffineFlow(_alt(D) if i % 2 == 0 else 1 - _alt(D), t, s), nf.flows.ActNorm(D)]
        target = None
        if name == "rnvp64_rkl":
            g = torch.Generator().manual_seed(57)
            target = nf.distributions.GaussianMixture(8, D, loc=(1.5 * torch.randn(8, D, generator=g)).numpy(),
                                                      scale=np.ones((8, D)), trainable=False)
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows, p=target)
    if name == "mixed64":
        b = _alt(D)
        flows = [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([D, 32, D]), nf.nets.MLP([D, 32, D], leaky=0.2)),
                 nf.flows.ActNorm(D), nf.flows.AutoregressiveRationalQuadraticSpline(D, 1, 64),
                 nf.flows.LULinearPermute(D), nf.flows.AffineCouplingBlock(nf.nets.MLP([32, 32, 64]), True, "sigmoid"),
                 nf.flows.Permute(D, "swap")]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows)
    assert name == "vae40"
    prior = torch.distributions.MultivariateNormal(torch.zeros(D), torch.eye(D))
    enc = nf.distributions.NNDiagGaussian(nf.nets.MLP(np.array([784, 512, 256, 2 * D])))
    dec = nf.distributions.NNBernoulliDecoder(nf.nets.MLP(np.array([D, 256, 512, 784])))
    b = torch.tensor(D // 2 * [0, 1] + D % 2 * [0])
    flows = []
    for i in range(40):
        s, t = nf.nets.MLP([D, D]), nf.nets.MLP([D, D])
        flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
    return nf.NormalizingFlowVAE(prior, enc, flows, dec)


def perturb(model, name):
    """The flows' parameters scaled by FLOW_SCALE first (vae40's then moved by FLOW_SIGMA).  Every parameter moved by
    sigma * randn (seeded) off its init, and every ActNorm marked initialised."""
    g = torch.Generator().manual_seed(800 + SEEDS[name])
    with torch.no_grad():
        if name in FLOW_SCALE:
            for p in model.flows.parameters():
                p.mul_(FLOW_SCALE[name])
        for n, p in model.named_parameters():
            sigma = FLOW_SIGMA if name == "vae40" and n.startswith("flows.") else SIGMA.get(name, 0.05)
            p.add_(sigma * torch.randn(p.shape, generator=g, dtype=p.dtype))
    for f in model.flows:
        if hasattr(f, "data_dep_init_done"):
            f.data_dep_init_done.fill_(1.0)


def data(name, n=512):
    """Forward-KL cases: the stored inputs x [n, D] (float32), a correlated Gaussian.  vae40: binarised x [B, 784]."""
    g = torch.Generator().manual_seed(900 + SEEDS[name])
    if name == "vae40":
        return (torch.rand(VAE_B, 784, generator=g) > 0.5).float()
    D = DIMS[name]
    A = 0.3 * torch.randn(D, D, generator=g) / D ** 0.5 + torch.eye(D)
    return torch.randn(n, D, generator=g) @ A * 0.8


def draws(name, n=512):
    """rnvp64_rkl: standardised base draws [n, D]; vae40: encoder draws [B, S, D] (float32)."""
    g = torch.Generator().manual_seed(1000 + SEEDS[name])
    if name == "vae40":
        return torch.randn(VAE_B, VAE_S, DIMS[name], generator=g)
    return torch.randn(n, DIMS[name], generator=g)


def digest(v):
    """sha256 of an entry as float32 (the reference keeps GaussianMixture's buffers in float64 and an integer mask b of
    MaskedAffineFlow as given, this package both in float32)."""
    a = np.asarray(v.detach().cpu().numpy() if torch.is_tensor(v) else v)
    if a.dtype.kind in "fiub":
        a = a.astype(np.float32)
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def digests(model):
    return json.dumps({k: digest(v) for k, v in model.state_dict().items()})
