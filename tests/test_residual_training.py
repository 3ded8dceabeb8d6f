"""Training pass of the residual flow: `NormalizingFlow.forward_kld(x).backward()` for stacks of Residual(LipschitzMLP) and
ActNorm layers (examples/residual.ipynb).

CPU tests check that the library exports the new entry points and that the numpy fp64 oracle
(oracle/nf_oracle_residual.py) reproduces the gradient goldens minted from the reference's fp64 autograd
(tests/golden/make_residual_grads.py).  GPU tests check the new kernels against torch fp64 autograd, whole models against
the goldens, the identity of the values with and without gradients, the error paths, and a short run of the notebook's
training loop."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

import normflows as nf
from normflows import _lib as L
from helpers import load_npz_parts
from helpers_glow_grads import grad_projections
from oracle import nf_oracle_residual as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = ["d2_geo", "d4_geo", "d2_poisson", "d4_poisson", "d2_brute", "d2_eval", "d4_eval", "d4_weighted", "c5"]
NEW_SYMBOLS = ("nfb_lipschitz_mlp_dual_backward", "nfb_lipschitz_mlp_dual_backward_workspace_bytes", "nfb_swish_dual",
               "nfb_swish_dual_adjoint", "nfb_logabsdet_i_plus_j_2x2_backward")


def load_case(name):
    f = load_npz_parts(os.path.join(GOLDEN, f"grads_res_{name}.npz"))
    spec = json.loads(str(f["spec"]))
    sd = {k[4:]: f[k] for k in f if k.startswith("sd__")}
    return f, spec, sd


def golden_grads(f):
    """{name: ('whole', G) | ('proj', Gv, uG, |G|)}"""
    out = {k[6:]: ("whole", f[k]) for k in f if k.startswith("grad__")}
    out.update({k[7:]: ("proj", f[k], f["gradu__" + k[7:]], float(f["gnorm__" + k[7:]])) for k in f if k.startswith("gradv__")})
    return out


def check_grad(name, got, ref, tol):
    """every entry (or projection) within tol x the largest |ref| entry of that tensor"""
    if ref[0] == "whole":
        err, scale = np.abs(got - ref[1]).max(), np.abs(ref[1]).max()
        assert err <= tol * scale, (name, err, scale)
        return
    G = got.reshape(got.shape[0], -1)
    v, u = grad_projections(name, got.shape)
    for a, b in ((G @ v.numpy(), ref[1]), (u.numpy() @ G, ref[2])):
        assert np.abs(a - b).max() <= tol * np.abs(b).max(), (name, np.abs(a - b).max(), np.abs(b).max())
    assert abs(np.linalg.norm(G) - ref[3]) <= tol * ref[3], (name, np.linalg.norm(G), ref[3])


def test_new_symbols_exported():
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    handle = ctypes.CDLL(L.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in L.SYMBOLS, name


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_gradients(name):
    f, spec, sd = load_case(name)
    lp, grads = R.log_prob_and_grads(spec, sd, f["x"].astype(np.float64), f["cot"], bool(f["training"]),
                                     list(zip(f["n_inj"], f["eps"])))
    np.testing.assert_allclose(lp, f["log_prob"], rtol=1e-10, atol=0)
    ref = golden_grads(f)
    assert set(ref) == set(grads), set(ref) ^ set(grads)
    for k, r in ref.items():
        check_grad(k, grads[k], r, 1e-10)


# ---- GPU: the kernels against torch fp64 autograd -----------------------------------------------------------------
def _swish64(h, b):
    return h * torch.sigmoid(b * h) / 1.1


def _dual64(H, bias, b, B, nt):
    """A = [sigma(h); sigma'(h) t_1; ...] in fp64 torch with sigma' by autograd (create_graph: differentiable)."""
    h = H[:B] + bias
    hh = h if h.requires_grad else h.requires_grad_(True)
    a = _swish64(hh, b)
    d1 = torch.autograd.grad(a.sum(), hh, create_graph=True)[0]
    return torch.cat([a] + [d1 * H[(k + 1) * B:(k + 2) * B] for k in range(nt)], 0)


@pytest.mark.gpu
@pytest.mark.parametrize("w", [2, 32, 128])
@pytest.mark.parametrize("nt", [0, 1, 2])
@pytest.mark.parametrize("B", [0, 1, 129, 1000])
def test_swish_dual_and_adjoint_match_torch(w, nt, B):
    g = torch.Generator().manual_seed(w * 100 + nt * 10 + B)
    H = torch.randn((1 + nt) * B, w, generator=g, dtype=torch.float64) * 2
    bias = torch.randn(w, generator=g, dtype=torch.float64) * 0.5
    b = 0.7
    Abar = torch.randn((1 + nt) * B, w, generator=g, dtype=torch.float64)
    Hd, bd, Ad = H.float().cuda(), bias.float().cuda(), Abar.float().cuda()
    A = torch.empty_like(Hd)
    L.check(L.lib().nfb_swish_dual(L.ptr(Hd), L.ptr(bd), b, B, w, nt, L.ptr(A), None))
    with torch.enable_grad():
        Hr = H.clone().requires_grad_(True)
        br = torch.tensor(b, dtype=torch.float64, requires_grad=True)
        Aref = _dual64(Hr, bias, br, B, nt)
        if B:
            gH, gb = torch.autograd.grad(Aref, (Hr, br), Abar)
        else:
            gH, gb = torch.zeros_like(H), torch.zeros((), dtype=torch.float64)
    tol = lambda r: 2e-6 * max(1.0, float(r.abs().max()) if r.numel() else 1.0)
    assert (A.double().cpu() - Aref.detach()).abs().max() <= tol(Aref) if B else True
    outp = torch.full((B, w), float("nan"), device="cuda")
    outt = torch.full((nt * B, w), float("nan"), device="cuda")
    partials = torch.empty(L.SWISH_DUAL_PARTIALS, dtype=torch.float64, device="cuda")
    gbd = torch.full((1,), float("nan"), device="cuda")
    L.check(L.lib().nfb_swish_dual_adjoint(L.ptr(Hd), L.ptr(bd), b, B, w, nt, L.ptr(Ad), L.ptr(outp), L.ptr(outt),
                                           L.ptr(partials), L.ptr(gbd), None))
    got = torch.cat([outp, outt], 0).double().cpu()
    assert (got - gH).abs().max() <= tol(gH) if B else True
    assert abs(float(gbd) - float(gb)) <= 1e-5 * max(1.0, abs(float(gb))) + 1e-6 * H.numel(), (float(gbd), float(gb))
    # in place (out_primal / out_tangent aliasing Abar), as the block backward runs it; bit-identical to the above
    L.check(L.lib().nfb_swish_dual_adjoint(L.ptr(Hd), L.ptr(bd), b, B, w, nt, L.ptr(Ad), L.ptr(Ad),
                                           L.ptr(Ad[B:]) if nt else None, L.ptr(partials), None, None))
    if B:
        assert torch.equal(Ad, torch.cat([outp, outt], 0))


@pytest.mark.gpu
@pytest.mark.parametrize("B", [0, 1, 300])
def test_logdet2_backward_matches_torch(B):
    g = torch.Generator().manual_seed(B)
    jt = torch.randn(2, B, 2, generator=g, dtype=torch.float64) * 0.3
    gld = torch.randn(B, generator=g, dtype=torch.float64)
    seeds = torch.empty(2, B, 2, device="cuda")
    jd, gd = jt.float().cuda(), gld.float().cuda()   # held by name until the kernel has run
    L.check(L.lib().nfb_logabsdet_i_plus_j_2x2_backward(L.ptr(jd), L.ptr(gd), B, L.ptr(seeds), None))
    with torch.enable_grad():
        j = jt.clone().requires_grad_(True)
        ld = torch.log(torch.abs((j[0, :, 0] + 1) * (j[1, :, 1] + 1) - j[1, :, 0] * j[0, :, 1]))
        ref = torch.autograd.grad(ld, j, gld)[0] if B else torch.zeros_like(jt)
    np.testing.assert_allclose(seeds.double().cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-6)


# ---- GPU: whole models ---------------------------------------------------------------------------------------------
def build(spec, sd, d):
    flows = []
    for blk in spec["flows"]:
        if blk["type"] == "actnorm":
            flows.append(nf.flows.ActNorm(d))
            continue
        pre = f"flows.{len(flows)}.iresblock.nnet.net."
        widths = [sd[f"{pre}{2 * l + 1}.weight"].shape[0] for l in range(blk["n_layers"])]
        net = nf.nets.LipschitzMLP([d] + widths, lipschitz_const=blk["coeff"], init_zeros=False)
        flows.append(nf.flows.Residual(net, reduce_memory=True, brute_force=blk["brute_force"], n_dist=blk["n_dist"]))
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=spec["base_trainable"]), flows)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, strict=True)
    return model.cuda()


def inject(model, f, training):
    """the golden's draws, per estimator call in call order (flows last to first; the exact path draws nothing)"""
    call = 0
    for flow in reversed(list(model.flows)):
        if isinstance(flow, nf.flows.Residual):
            blk = flow.iresblock
            if not ((blk.brute_force or not training) and f["x"].shape[1] == 2):
                blk._inject_n = f["n_inj"][call]
                blk._inject_eps = torch.from_numpy(f["eps"][call]).float().cuda()
                call += 1
    assert call == len(f["n_inj"])


def loss_of(model, x, f):
    """the golden's loss: forward_kld = -mean(log_prob), or the weighted sum sum_r cot[r] log_prob(x_r)"""
    lp = model.log_prob(x)
    return (lp * torch.from_numpy(f["cot"]).float().cuda()).sum(), lp


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_model_gradients_match_reference(name):
    f, spec, sd = load_case(name)
    d = f["x"].shape[1]
    training = bool(f["training"])
    model = build(spec, sd, d)
    model.train(training)
    with torch.enable_grad():
        x = torch.from_numpy(f["x"]).float().cuda().requires_grad_(True)
        inject(model, f, training)
        loss, lp = loss_of(model, x, f)
        loss.backward()
    np.testing.assert_allclose(lp.detach().cpu().numpy(), f["log_prob"], rtol=1e-4, atol=1e-4)
    got = {"x": x.grad.double().cpu().numpy()}
    got.update({k: p.grad.double().cpu().numpy() for k, p in model.named_parameters() if p.grad is not None})
    ref = golden_grads(f)
    assert set(got) == set(ref), set(got) ^ set(ref)
    for k, r in ref.items():
        check_grad(k, got[k], r, 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["d4_geo", "d2_eval", "d2_brute"])
def test_values_identical_with_and_without_grad(name):
    f, spec, sd = load_case(name)
    model = build(spec, sd, f["x"].shape[1])
    training = bool(f["training"])
    model.train(training)
    x = torch.from_numpy(f["x"]).float().cuda()
    inject(model, f, training)
    lp0 = model.log_prob(x)
    inject(model, f, training)
    kld0 = model.forward_kld(x)
    with torch.enable_grad():
        inject(model, f, training)
        lp1 = model.log_prob(x)
        inject(model, f, training)
        kld1 = model.forward_kld(x)
    assert lp1.requires_grad and kld1.requires_grad
    assert torch.equal(lp0, lp1.detach()) and torch.equal(kld0, kld1.detach())


@pytest.mark.gpu
def test_update_lipschitz_between_forward_and_backward_raises():
    f, spec, sd = load_case("d4_geo")
    model = build(spec, sd, 4)
    model.train()
    with torch.enable_grad():
        inject(model, f, True)
        loss = model.forward_kld(torch.from_numpy(f["x"]).float().cuda())
        nf.utils.update_lipschitz(model, 5)
        with pytest.raises(RuntimeError, match="modified in place"):
            loss.backward()


@pytest.mark.gpu
def test_reduce_memory_false_training_gradient_raises():
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(4),
                               [nf.flows.Residual(nf.nets.LipschitzMLP([4, 16, 4]), reduce_memory=False)]).cuda()
    x = torch.randn(8, 4, device="cuda")
    model.train()
    with torch.enable_grad(), pytest.raises(NotImplementedError, match="reduce_memory=True"):
        model.forward_kld(x)
    with torch.no_grad():   # the value is still available
        assert torch.isfinite(model.forward_kld(x))


def notebook_model(hidden=(128, 128)):
    """examples/residual.ipynb: 16 x [Residual(LipschitzMLP([2, 128, 128, 2])), ActNorm(2)], fixed DiagGaussian"""
    torch.manual_seed(0)
    flows = []
    for _ in range(16):
        net = nf.nets.LipschitzMLP([2] + list(hidden) + [2], init_zeros=True, lipschitz_const=0.9)
        flows += [nf.flows.Residual(net, reduce_memory=True), nf.flows.ActNorm(2)]
    return nf.NormalizingFlow(q0=nf.distributions.DiagGaussian(2, trainable=False), flows=flows).cuda()


def moons(n, seed):
    """sklearn.datasets.make_moons(n, noise=0.1) restated with a seeded torch generator (the notebook's data)"""
    g = torch.Generator().manual_seed(seed)
    n_out = n // 2
    t_out, t_in = torch.linspace(0, np.pi, n_out), torch.linspace(0, np.pi, n - n_out)
    x = torch.cat([torch.stack([torch.cos(t_out), torch.sin(t_out)], 1),
                   torch.stack([1 - torch.cos(t_in), 1 - torch.sin(t_in) - 0.5], 1)])
    x = x[torch.randperm(n, generator=g)] + 0.1 * torch.randn(n, 2, generator=g)
    return x.cuda()


@pytest.mark.gpu
def test_notebook_model_every_parameter_gets_a_gradient():
    model = notebook_model()
    np.random.seed(0)
    with torch.enable_grad():
        model.log_prob(moons(512, 1))    # ActNorm init (notebook cell 2)
        model.forward_kld(moons(512, 2)).backward()
    for name, p in model.named_parameters():
        if name.endswith("geom_p") or name.endswith("lamb"):
            assert p.grad is None, name
            continue
        assert p.grad is not None, name
        assert torch.isfinite(p.grad).all(), name


@pytest.mark.gpu
def test_notebook_training_loop_learns():
    model = notebook_model()
    np.random.seed(0)
    with torch.enable_grad():
        model.log_prob(moons(512, 1))
        opt = torch.optim.Adam(model.parameters(), lr=3e-4, weight_decay=1e-5)
        losses = []
        for it in range(300):
            opt.zero_grad()
            loss = model.forward_kld(moons(512, 100 + it))
            if not (torch.isnan(loss) | torch.isinf(loss)):
                loss.backward()
                opt.step()
            nf.utils.update_lipschitz(model, 50)
            losses.append(loss.item())
    # the loss of a 512-sample batch scatters by ~0.1 around its mean, so 20-step means are good to ~0.02
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    assert last < first - 0.05, (first, last)
    # the trained weights: eval-mode log_prob (exact 2 x 2 path) against the fp64 oracle built from the state_dict
    model.eval()
    x = moons(1000, 7)
    lp = model.log_prob(x).double().cpu().numpy()
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    spec = {"flows": [{"type": "actnorm"} if isinstance(fl, nf.flows.ActNorm) else
                      {"type": "residual", "coeff": 0.9, "n_layers": 3, "n_dist": "geometric", "brute_force": False}
                      for fl in model.flows], "base_trainable": False}
    ref, _ = R.log_prob_and_grads(spec, sd, x.double().cpu().numpy(), np.zeros(1000), False, [])
    np.testing.assert_allclose(lp, ref, rtol=1e-4, atol=1e-4)
