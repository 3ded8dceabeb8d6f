"""Mint gradient goldens of the Glow training pass from the REAL reference (normflows 1.7.3; a checkout found by
oracle/reference.py, no GPU needed): fp64 autograd of `MultiscaleFlow.forward_kld(x, y)`, every parameter gradient and
x.grad.
    python tests/golden/make_glow_grads.py [glow_small|glow_width|options|glow_c3]
Writes tests/golden/grads_<case>.npz (split into <name>.2.npz, ... below 1 MB):
    glow_small  the model and inputs of glow_small.npz (L=2, K=2, hidden 32, 3x8x8: generic conditioner path)
    glow_width  L=2, K=2, hidden 64, 3x16x16 on 64 images (Glow-shaped conditioner: fused kernel, tap-form coupling);
                its state_dict is stored here
    options     the model and inputs of options.npz (use_lu=False, net_actnorm=True, Logit transform)
    glow_c3     BASELINE config 3 at its real shape, the model of glow_c3.npz (rebuilt by its recipe, digests checked)
                on its 64 images
Every file carries sd_sha256 (digests of the state_dict the gradients belong to) and x_sha256 / y_sha256.  Tensors
with more than 4096 entries are stored as gradv__ = G v, gradu__ = u G (G = the gradient reshaped to [shape[0], -1];
v, u drawn by tests/helpers_glow_grads.py grad_projections from a seed derived from the parameter name) and gnorm__ = |G|."""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import nf, perturb, save_parts, sha256  # noqa: E402  (nf = the reference)
sys.path.insert(0, os.path.dirname(HERE))
from helpers_glow_grads import grad_projections as projections  # noqa: E402  (the draw the tests repeat)

MAX_WHOLE = 4096


def grads_of(model, x, y, project_x=False):
    """fp64 autograd of forward_kld: {'kld', 'grad__x' | 'gradv__/gradu__/gnorm__x', 'grad__<p>' |
    'gradv__/gradu__/gnorm__<p>'}."""
    model = model.double()
    xx = x.double().requires_grad_(True)
    loss = model.forward_kld(xx, y)
    loss.backward()
    out = {"kld": loss.detach().numpy()}   # x.grad of many images: grad__x__0, grad__x__1, ... along the batch
    named = [("x", xx)] + list(model.named_parameters())
    for k, p in named:
        if p.grad is None:
            continue
        if k == "x" and not project_x and p.numel() > 65536:   # whole, in 16-image pieces (files stay below 1 MB)
            for i in range(0, p.shape[0], 16):
                out[f"grad__x__{i // 16}"] = p.grad[i:i + 16].numpy()
        elif p.numel() <= MAX_WHOLE or (k == "x" and not project_x):
            out["grad__" + k] = p.grad.numpy()
        else:
            G = p.grad.reshape(p.shape[0], -1)
            v, u = projections(k, tuple(p.shape))
            out["gradv__" + k], out["gradu__" + k] = (G @ v).numpy(), (u @ G).numpy()
            out["gnorm__" + k] = np.asarray(G.norm().item())
    return out


def build(L, K, hidden, shape, ncls, **kw):
    q0, merges, flows = [], [], []
    for i in range(L):
        flows.append([nf.flows.GlowBlock(shape[0] * 2 ** (L + 1 - i), hidden, split_mode="channel", scale=True, **kw)
                      for _ in range(K)] + [nf.flows.Squeeze()])
        if i > 0:
            merges.append(nf.flows.Merge())
            ls = (shape[0] * 2 ** (L - i), shape[1] // 2 ** (L - i), shape[2] // 2 ** (L - i))
        else:
            ls = (shape[0] * 2 ** (L + 1), shape[1] // 2 ** L, shape[2] // 2 ** L)
        q0.append(nf.distributions.ClassCondDiagGaussian(ls, ncls))
    return q0, flows, merges


def header(model, x, y):
    return {"torch_version": torch.__version__, "x_sha256": sha256(x.numpy()), "y_sha256": sha256(y.numpy()),
            "sd_sha256": json.dumps({k: sha256(v.detach().numpy()) for k, v in model.state_dict().items()})}


def from_golden(name, transform=None, **kw):
    """A model whose float32 state_dict and inputs are stored in tests/golden/<name>.npz."""
    f = np.load(os.path.join(HERE, name + ".npz"))
    model = nf.MultiscaleFlow(*build(**kw), transform=transform)
    model.load_state_dict({k[4:]: torch.from_numpy(f[k]) for k in f.files if k.startswith("sd__")}, strict=True)
    x, y = torch.from_numpy(f["x"]).float(), torch.from_numpy(f["y"])
    return model, x, y


def case_glow_small():
    model, x, y = from_golden("glow_small", L=2, K=2, hidden=32, shape=(3, 8, 8), ncls=10)
    out = header(model, x, y)
    out.update(grads_of(model, x, y))
    save_parts("grads_glow_small", out)


def case_options():
    model, x, y = from_golden("options", transform=nf.transforms.Logit(0.05), L=2, K=2, hidden=16, shape=(3, 8, 8),
                              ncls=10, use_lu=False, net_actnorm=True)
    out = header(model, x, y)
    out.update(grads_of(model, x, y))
    save_parts("grads_glow_options", out)


def case_glow_width():
    torch.manual_seed(31)
    model = nf.MultiscaleFlow(*build(L=2, K=2, hidden=64, shape=(3, 16, 16), ncls=10))
    g = torch.Generator().manual_seed(32)
    x = torch.rand(64, 3, 16, 16, generator=g)
    y = torch.randint(10, (64,), generator=g)
    with torch.no_grad():
        model.log_prob(x, y)   # ActNorm data-dependent init
    perturb(model, 0.03, 33)
    out = header(model, x, y)
    out["x"], out["y"] = x.numpy(), y.numpy()
    out.update({"sd__" + k: v.detach().numpy() for k, v in model.state_dict().items()})
    out.update(grads_of(model, x, y))
    save_parts("grads_glow_width", out)


def case_glow_c3():
    """The model of glow_c3.npz (make_golden.py case_glow_c3: constructors under seed 0, ActNorm init on 64 images,
    0.02 randn perturbation under seed 2), checked against its digests, on the same 64 images (tests/helpers_glow.py
    glow_c3_inputs()).  64 rather than 16 images: the coarsest level is 4x4, and with 16 images its 256 pixels per
    channel let one ReLU kink that fp32 and fp64 resolve differently shift whole rows of a conditioner's gradient."""
    torch.manual_seed(0)
    model = nf.MultiscaleFlow(*build(L=3, K=16, hidden=256, shape=(3, 32, 32), ncls=10)).double()
    g = torch.Generator().manual_seed(1)
    x64 = torch.rand(64, 3, 32, 32, generator=g)
    y64 = torch.randint(10, (64,), generator=g)
    with torch.no_grad():
        model.log_prob(x64.double(), y64)
        perturb(model, 0.02, 2)
    f = np.load(os.path.join(HERE, "glow_c3.npz"))
    want = json.loads(str(f["sd_sha256"]))
    got = {k: sha256(v.detach().numpy()) for k, v in model.state_dict().items()}
    assert got == want, "glow_c3: rebuilt state_dict differs from glow_c3.npz"
    x, y = x64, y64
    out = header(model, x, y)
    out.update(grads_of(model, x, y))
    save_parts("grads_glow_c3", out)


CASES = {"glow_small": case_glow_small, "glow_width": case_glow_width, "options": case_options, "glow_c3": case_glow_c3}

if __name__ == "__main__":
    for name in (sys.argv[1:] or list(CASES)):
        CASES[name]()
        print("wrote", name)
