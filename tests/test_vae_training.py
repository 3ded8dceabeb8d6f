"""The flow-VAE (reference core.py NormalizingFlowVAE, distributions/encoder.py, distributions/decoder.py;
examples/vae.ipynb): the encoder draw, the Gaussian densities and the Bernoulli likelihood kernels (csrc/nfb_vae.cu) and
their native backward, and the VAE driver with the flows passed through one stack.

CPU: the host-compiled element math (csrc/nfb_vae.cuh) against fp64 autograd and central differences, the zero-score
rule and saturated scores included; the fp64 restatement (tests/helpers_vae.py) against the reference's goldens;
construction order and state_dict keys.
GPU: each kernel against fp64 torch over rows, S and d; the goldens with replayed draws; bit-identical values with and
without grad and between runs; the in-place refusal and CPU inputs; flows without a differentiable sampling direction;
strict loading of reference state_dicts; the notebook's training cell."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import helpers_vae as V
from conftest import ROOT

NEW_SYMBOLS = ("nfb_vae_reparam_sample", "nfb_vae_reparam_sample_backward", "nfb_vae_gaussian_log_prob",
               "nfb_vae_gaussian_log_prob_backward", "nfb_bernoulli_log_prob", "nfb_bernoulli_log_prob_backward",
               "nfb_sigmoid", "nfb_sigmoid_backward")


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


def test_new_symbols_exported():
    from normflows import _lib
    hdr = open(os.path.join(ROOT, "include", "nfb200.h")).read()
    for name in NEW_SYMBOLS:
        assert name + "(" in hdr and name in _lib.SYMBOLS, name
        assert hasattr(_lib.lib(), name), name
    assert _lib.lib().nfb_abi_version() == 1


def test_exports_match_the_reference():
    import normflows as nf
    for name in ("BaseEncoder", "Dirac", "Uniform", "NNDiagGaussian", "BaseDecoder", "NNDiagGaussianDecoder",
                 "NNBernoulliDecoder"):
        assert hasattr(nf.distributions, name), name
    assert nf.distributions.Uniform is nf.distributions.encoder.Uniform
    assert hasattr(nf.distributions.encoder, "ConstDiagGaussian")
    assert nf.NormalizingFlowVAE is nf.core.NormalizingFlowVAE
    mlp = nf.nets.MLP(np.array([784, 512, 80]))
    assert [l.in_features for l in mlp.linear_layers()] == [784, 512]
    assert all(type(n) is int for n in mlp.layer_sizes)


# ---- shapes are checked before any kernel reads them --------------------------------------------------------------------
def test_data_width_must_match_the_net_output():
    """The kernels take the net's width as the row stride of the data they pair with it, so a mismatch is refused in
    Python (on CPU tensors too, before any device work); the reference fails to broadcast in the same cases."""
    import normflows as nf
    from torch import nn
    z = torch.randn(15, 4)
    with pytest.raises(ValueError, match="widths differ"):
        nf.distributions.NNBernoulliDecoder(nn.Linear(4, 800)).log_prob(torch.zeros(5, 784), z)
    with pytest.raises(ValueError, match="expected \\[rows, 10\\]"):
        nf.distributions.NNDiagGaussianDecoder(nn.Linear(4, 20)).log_prob(torch.zeros(5, 12), z)
    enc = nf.distributions.NNDiagGaussian(nn.Linear(12, 8))
    for width in (3, 5):
        with pytest.raises(ValueError, match="expected \\[rows, 4\\]"):
            enc.log_prob(torch.randn(5, 3, width), torch.zeros(5, 12))
    from normflows import _vae
    with pytest.raises(ValueError, match="rows"):
        _vae.bernoulli_log_prob(torch.zeros(15, 7), torch.zeros(4, 7), 3)
    with pytest.raises(ValueError, match="rows"):
        _vae.gaussian_log_prob(torch.zeros(4, 3), 15, 3, 1, 3, net=torch.zeros(15, 6))
    with pytest.raises(ValueError, match="rows"):
        _vae.reparam_sample(torch.zeros(5, 2, 3), net=torch.zeros(4, 6))


def test_const_encoder_scale_must_fit_loc():
    import normflows as nf
    C_ = nf.distributions.encoder.ConstDiagGaussian
    for n in (3, 5):
        with pytest.raises(ValueError, match="scale has"):
            C_(torch.zeros(4), torch.ones(n))
    q = C_(torch.zeros(4), torch.tensor([0.5]))       # one entry broadcasts over the features, as in the reference
    assert q.state_dict()["scale"].shape == (1,) and q._scale().shape == (4,)
    with pytest.raises(ValueError, match="expected \\[rows, 4\\]"):
        C_(torch.zeros(4), torch.ones(4)).log_prob(torch.zeros(2, 3, 5), None)


# ---- element math on the host -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def vaelib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "vae_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "vae_host_check.cu")])
    return C.CDLL(so)


def _a(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def _P(v):
    return v.ctypes.data_as(C.c_void_p)


def host_gauss(lib, kind, m, p, e, gz, g, use_float=0):
    m, p, e, gz, g = (_a(v) for v in (m, p, e, gz, g))
    outs = [np.empty_like(m) for _ in range(8)]
    lib.vae_gauss_check(C.c_int(kind), C.c_int(m.size), C.c_int(use_float), *[_P(v) for v in (m, p, e, gz, g)],
                        *[_P(o) for o in outs])
    return outs


def host_bern(lib, s, x, use_float=0):
    s, x = _a(s), _a(x)
    outs = [np.empty_like(s) for _ in range(3)]
    lib.vae_bernoulli_check(C.c_int(s.size), C.c_int(use_float), _P(s), _P(x), *[_P(o) for o in outs])
    return outs


def _std(p, kind):
    return torch.exp(0.5 * p) if kind == 0 else p


@pytest.mark.parametrize("kind", [0, 1])
def test_host_gaussian_element_math_matches_autograd_and_central_differences(vaelib, kind):
    rng = np.random.default_rng(3 + kind)
    n = 40
    m, e, gz, g = rng.normal(size=n), rng.normal(size=n) * 1.5, rng.normal(size=n), rng.normal(size=n)
    p = rng.normal(size=n) * 0.6 if kind == 0 else rng.uniform(0.3, 2.0, size=n)
    z, nlq, g_m, g_p, dens, gd_v, gd_m, gd_p = host_gauss(vaelib, kind, m, p, e, gz, g)
    M, Pp, E = (torch.tensor(v, requires_grad=True) for v in (m, p, e))
    sd = _std(Pp, kind)
    zt = M + sd * E
    nt = torch.log(sd) + 0.5 * E.detach() ** 2
    ((zt * torch.tensor(gz)).sum() - (nt * torch.tensor(g)).sum()).backward()
    np.testing.assert_allclose(z, zt.detach().numpy(), rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(nlq, nt.detach().numpy(), rtol=1e-14, atol=1e-14)
    np.testing.assert_allclose(g_m, M.grad.numpy(), rtol=1e-13, atol=1e-13)
    np.testing.assert_allclose(g_p, Pp.grad.numpy(), rtol=1e-12, atol=1e-12)
    M.grad = Pp.grad = E.grad = None
    sd = _std(Pp, kind)
    dt = torch.log(sd) + 0.5 * ((E - M) / sd) ** 2          # the reference's -log p share (as 0.5 (log var + ...))
    (-(dt * torch.tensor(g)).sum()).backward()
    np.testing.assert_allclose(dens, dt.detach().numpy(), rtol=1e-13, atol=1e-13)
    for got, ref in ((gd_v, E.grad), (gd_m, M.grad), (gd_p, Pp.grad)):
        np.testing.assert_allclose(got, ref.numpy(), rtol=1e-11, atol=1e-12)
    h = 1e-6                                                 # central differences of the density in each argument
    for got, which in ((gd_v, 2), (gd_m, 0), (gd_p, 1)):
        args_hi, args_lo = [m.copy(), p.copy(), e.copy()], [m.copy(), p.copy(), e.copy()]
        args_hi[which] += h
        args_lo[which] -= h
        fd = -(host_gauss(vaelib, kind, *args_hi[:2], args_hi[2], gz, g)[4]
               - host_gauss(vaelib, kind, *args_lo[:2], args_lo[2], gz, g)[4]) * g / (2 * h)
        np.testing.assert_allclose(got, fd, rtol=1e-5, atol=1e-6)
    f32 = host_gauss(vaelib, kind, m, p, e, gz, g, use_float=1)
    for a, r in zip(f32, (z, nlq, g_m, g_p, dens, gd_v, gd_m, gd_p)):
        np.testing.assert_allclose(a, r, rtol=1e-5, atol=1e-5 * max(1.0, np.abs(r).max()))


def _ref_bernoulli(s, x):
    S = torch.tensor(s, requires_grad=True)
    X = torch.tensor(x, requires_grad=True)
    t = X * V._log_sig(S) + (1 - X) * V._log_sig(-S)
    t.sum().backward()
    return t.detach().numpy(), S.grad.numpy(), X.grad.numpy()


def test_host_bernoulli_element_math_zero_score_rule_and_saturation(vaelib):
    rng = np.random.default_rng(11)
    s = np.r_[rng.normal(size=30) * 3, 0.0, 0.0, -0.0, 20, -20, 80, -80, 1e4, -1e4, 1e4, -1e4]
    x = np.r_[(rng.uniform(size=30) > 0.5).astype(float), 1.0, 0.0, 0.3, 1, 0, 0, 1, 1, 0, 0, 1]
    x[:5] = rng.uniform(size=5)                       # real-valued x as well
    term, ds, sig = host_bern(vaelib, s, x)
    rt, rs, _ = _ref_bernoulli(s, x)
    fin = np.isfinite(rt)
    np.testing.assert_allclose(term[fin], rt[fin], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ds, rs, rtol=1e-12, atol=1e-14)
    assert (ds[30:33] == 0).all(), ds[30:33]          # s == 0 exactly: the reference's gradient is 0, not x - 1/2
    np.testing.assert_allclose(sig, torch.sigmoid(torch.tensor(s)).numpy(), rtol=1e-14, atol=1e-300)
    for use_float in (0, 1):
        t, d, sg = host_bern(vaelib, s, x, use_float)
        assert np.isfinite(t).all() and np.isfinite(d).all() and np.isfinite(sg).all(), use_float
    sat = slice(33, None)
    # saturated scores: the reference formula's value (-|s| on the losing side, ~0 on the winning one)
    np.testing.assert_allclose(term[sat], x[sat] * np.minimum(s[sat], 0) + (1 - x[sat]) * np.minimum(-s[sat], 0),
                               rtol=1e-12, atol=1e-8)
    t32 = host_bern(vaelib, s, x, 1)[0]
    np.testing.assert_allclose(t32[sat], term[sat], rtol=1e-6, atol=1e-6)
    h = 1e-6
    ok = np.abs(s) > 1e-3
    fd = (host_bern(vaelib, s + h, x)[0] - host_bern(vaelib, s - h, x)[0]) / (2 * h)
    np.testing.assert_allclose(ds[ok], fd[ok], rtol=1e-5, atol=1e-7)


# ---- goldens: the reference (tests/golden/make_vae_grads.py) ------------------------------------------------------------
def _golden(name):
    from helpers import load_npz_parts
    return load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_vae_{name}.npz"))


def _state_dict(name, gd):
    """The perturbed state_dict of case `name` (float32): stored, or for case e rebuilt and checked bit for bit."""
    import normflows as nf
    from helpers import check_digests
    if "sd_sha256" not in gd:
        return {k[4:]: v for k, v in gd.items() if k.startswith("sd__")}
    model = V.build(nf, name)
    V.perturb_case(model, name)
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    check_digests(sd, json.loads(str(gd["sd_sha256"])), f"vae case {name}")
    return sd


def _check_golden(got, gd, name, tol):
    from test_maf_training import check_golden
    check_golden(got, gd, name, tol)


@pytest.mark.parametrize("name", V.CASES)
def test_fp64_restatement_matches_reference_goldens(name):
    gd = _golden(name)
    sd = _state_dict(name, gd)
    P = {k: torch.tensor(np.asarray(v, np.float64), requires_grad=True) for k, v in sd.items()}
    x, eps = torch.tensor(gd["x"]).double(), torch.tensor(gd["eps"]).double()
    z, log_q, log_p, loss = V.restate(name, P, x, eps)
    loss.backward()
    for key, got in (("z", z), ("log_q", log_q), ("log_p", log_p)):
        np.testing.assert_allclose(got.detach().numpy(), gd[key], rtol=1e-10, atol=1e-10, err_msg=key)
    assert abs(loss.item() - float(gd["loss"])) <= 1e-10 * max(1.0, abs(float(gd["loss"])))
    for n, p in P.items():
        if "g__" + n in gd or "gv__" + n in gd:
            _check_golden(p.grad, gd, n, 1e-10)
    with torch.no_grad():
        z0, _ = V.encoder_draw(name, P, x, eps)
        np.testing.assert_allclose(V.encoder_log_prob(name, P, z0, x).numpy(), gd["enc_log_prob"], rtol=1e-10,
                                   atol=1e-10)
        if "dec_forward" in gd:
            dec = V.decoder_forward(name, P, z.reshape(-1, z.shape[2]))
            dec = dec if isinstance(dec, tuple) else (dec,)
            for got, key in zip(dec, ("dec_forward", "dec_forward_std")):
                np.testing.assert_allclose(got.numpy(), gd[key], rtol=1e-10, atol=1e-12, err_msg=key)
    if name == "b":   # the zero-initialised decoder: every score is 0, and so is its last layer's gradient
        assert float(P["decoder.net.net.2.weight"].grad.abs().max()) == 0.0


@pytest.mark.parametrize("name", [c for c in V.CASES if c != "e"])
def test_construction_matches_reference(name):
    """Keys, shapes and values of the as-constructed state_dict (the order in which constructors draw from torch's
    generator); the perturbed one for case e is pinned by its digests in _state_dict."""
    import normflows as nf
    gd = _golden(name)
    own = V.build(nf, name).state_dict()
    ref = {k[6:]: v for k, v in gd.items() if k.startswith("init__")}
    assert list(own) == list(ref), (list(own), list(ref))
    for k, v in own.items():
        assert tuple(v.shape) == ref[k].shape, k
        np.testing.assert_array_equal(v.numpy(), ref[k].astype(v.numpy().dtype), err_msg=k)


def test_notebook_model_rebuilds_from_its_digests():
    _state_dict("e", _golden("e"))


# ================================================ GPU ================================================================
def _close(got, ref, name, tol=2e-3):
    from test_affine_rkl_training import _close as close
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    if ref.numel():
        close(got, ref, name, tol)


def _gpu_model(name, gd):
    """Case `name` built by this package on the GPU with the golden's parameters and replayed encoder draws."""
    import normflows as nf
    model = V.build(nf, name, device="cuda")
    sd = _state_dict(name, gd)
    model.load_state_dict({k: torch.tensor(np.asarray(v)) for k, v in sd.items()}, strict=True)
    model = model.cuda()
    eps = torch.tensor(gd["eps"]).cuda()
    model.q0._draw_eps = lambda shape, device: eps.reshape(shape).clone()
    return model, torch.tensor(gd["x"]).float().cuda(), eps


@pytest.mark.gpu
@pytest.mark.parametrize("name", V.CASES)
def test_model_gradients_match_reference_goldens(name):
    gd = _golden(name)
    model, x, _ = _gpu_model(name, gd)
    z, log_q, log_p = model(x, V.SHAPES[name][1])
    loss = torch.mean(log_q) - torch.mean(log_p)
    loss.backward()
    for key, got in (("z", z), ("log_q", log_q), ("log_p", log_p)):
        _close(got.detach().cpu(), torch.tensor(gd[key]), key)
    assert abs(loss.item() - float(gd["loss"])) <= 2e-3 * max(1.0, abs(float(gd["loss"]))), (loss.item(), gd["loss"])
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        if "g__" + n in gd or "gv__" + n in gd:
            _check_golden(p.grad.cpu(), gd, n, 2e-3)
    with torch.no_grad():
        z0, _ = model.q0(x, V.SHAPES[name][1])
        _close(model.q0.log_prob(z0, x).cpu(), torch.tensor(gd["enc_log_prob"]), "enc_log_prob")
        if model.decoder is not None:
            dec = model.decoder(z.reshape(-1, z.shape[2]))
            dec = dec if isinstance(dec, tuple) else (dec,)
            for got, key in zip(dec, ("dec_forward", "dec_forward_std")):
                _close(got.cpu(), torch.tensor(gd[key]), key)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c for c in V.CASES if c != "e"])
def test_reference_state_dict_loads_strictly(name):
    import normflows as nf
    gd = _golden(name)
    model = V.build(nf, name)
    ref = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    model.load_state_dict(ref, strict=True)
    for k, v in model.state_dict().items():
        assert torch.equal(v, ref[k].to(v.dtype)), k


# ---- kernels against fp64 torch --------------------------------------------------------------------------------------
def _encoder_net_out(B, d, seed, odd=False):
    g = torch.Generator().manual_seed(seed)
    out = torch.randn(B, 2 * d + int(odd), generator=g)
    out[:, d:] *= 0.5
    return out.cuda()


def _ref_draw(net, eps):
    d = eps.shape[2]
    n = net.double()
    mean, std = n[:, :d].unsqueeze(1), torch.exp(0.5 * n[:, d:2 * d].unsqueeze(1))
    e = eps.double()
    return mean + std * e, -0.5 * d * math.log(2 * math.pi) - torch.sum(torch.log(std) + 0.5 * e ** 2, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,d", [(0, 3, 4), (1, 1, 1), (1061, 1, 5), (7, 3, 64), (33, 32, 40), (1061, 3, 17)])
def test_encoder_draw_and_log_prob_match_fp64(B, S, d):
    from normflows import _vae
    net0 = _encoder_net_out(B, d, B + S + d, odd=(d == 17))
    g = torch.Generator().manual_seed(d)
    eps = torch.randn(B, S, d, generator=g).cuda()
    gz, glq, gl = (torch.randn(*s, generator=g).cuda() for s in ((B, S, d), (B, S), (B, S)))
    net = net0.clone().requires_grad_(True)
    z, lq = _vae.reparam_sample(eps, net=net)
    with torch.no_grad():
        z_ng, lq_ng = _vae.reparam_sample(eps, net=net0)
    assert torch.equal(z, z_ng) and torch.equal(lq, lq_ng)
    ((z * gz).sum() + (lq * glq).sum()).backward()
    nd = net0.double().requires_grad_(True)
    zr, lqr = _ref_draw(nd, eps)
    ((zr * gz.double()).sum() + (lqr * glq.double()).sum()).backward()
    _close(z.detach(), zr.detach(), "z", 1e-5)
    _close(lq.detach(), lqr.detach(), "log_q", 1e-5)
    _close(net.grad, nd.grad, "g_net")
    # the encoder's density of z [B, S, d] given x, through the grouped kernel (S rows per parameter row)
    zz = zr.detach().float().requires_grad_(True)
    net.grad = None
    out = _vae.gaussian_log_prob(zz.reshape(B * S, d), B * S, 1, S, d, net=net).reshape(B, S)
    (out * gl).sum().backward()
    zd = zr.detach().requires_grad_(True)
    nd.grad = None
    mean, var = nd[:, :d].unsqueeze(1), torch.exp(nd[:, d:2 * d].unsqueeze(1))
    ref = -0.5 * d * math.log(2 * math.pi) - 0.5 * torch.sum(torch.log(var) + (zd - mean) ** 2 / var, 2)
    (ref * gl.double()).sum().backward()
    _close(out.detach(), ref.detach(), "enc log_prob", 1e-5)
    _close(zz.grad, zd.grad, "g_z")
    _close(net.grad, nd.grad, "g_net (log_prob)")
    if B == 0:
        assert net.grad.shape == (0, net0.shape[1])


@pytest.mark.gpu
@pytest.mark.parametrize("rows,d", [(0, 3), (1, 1), (1061, 8), (96, 64)])
def test_const_encoder_matches_fp64(rows, d):
    import normflows as nf
    g = torch.Generator().manual_seed(rows + d)
    q = nf.distributions.encoder.ConstDiagGaussian(torch.randn(d, generator=g),
                                                   torch.rand(d, generator=g) + 0.5).cuda()
    eps = torch.randn(rows, 3, d, generator=g).cuda()
    q._draw_eps = lambda shape, device: eps
    x = torch.zeros(rows, 2, device="cuda")
    gz, glq = torch.randn(rows, 3, d, generator=g).cuda(), torch.randn(rows, 3, generator=g).cuda()
    z, lq = q(x, 3)
    ((z * gz).sum() + (lq * glq).sum()).backward()
    loc, scale = (t.detach().double().requires_grad_(True) for t in (q.loc, q.scale))
    zr = loc + scale * eps.double()
    lqr = -0.5 * d * math.log(2 * math.pi) - torch.sum(torch.log(scale) + 0.5 * eps.double() ** 2, 2)
    ((zr * gz.double()).sum() + (lqr * glq.double()).sum()).backward()
    _close(z.detach(), zr.detach(), "z", 1e-5)
    _close(lq.detach(), lqr.detach(), "log_q", 1e-5)
    _close(q.loc.grad, loc.grad, "g_loc")
    _close(q.scale.grad, scale.grad, "g_scale")
    if rows == 0:
        assert (q.loc.grad == 0).all() and (q.scale.grad == 0).all()
    q.zero_grad()
    loc.grad = scale.grad = None
    zz = zr.detach().float()
    lp = q.log_prob(zz, x)
    (lp * glq).sum().backward()
    ref = -0.5 * d * math.log(2 * math.pi) - torch.sum(torch.log(scale) + 0.5 * ((zr.detach() - loc) / scale) ** 2, 2)
    (ref * glq.double()).sum().backward()
    _close(lp.detach(), ref.detach(), "const log_prob", 1e-5)
    _close(q.loc.grad, loc.grad, "g_loc (log_prob)")
    _close(q.scale.grad, scale.grad, "g_scale (log_prob)")


@pytest.mark.gpu
def test_const_encoder_one_element_scale_matches_fp64():
    import normflows as nf
    d = 5
    q = nf.distributions.encoder.ConstDiagGaussian(torch.linspace(-1, 1, d), torch.tensor([0.7])).cuda()
    g = torch.Generator().manual_seed(9)
    eps = torch.randn(6, 3, d, generator=g).cuda()
    q._draw_eps = lambda shape, device: eps
    gz, glq = torch.randn(6, 3, d, generator=g).cuda(), torch.randn(6, 3, generator=g).cuda()
    z, lq = q(torch.zeros(6, 2, device="cuda"), 3)
    lp = q.log_prob(z.detach(), None)
    ((z * gz).sum() + (lq * glq).sum() + (lp * glq).sum()).backward()
    loc, scale = (t.detach().double().requires_grad_(True) for t in (q.loc, q.scale))
    zr = loc + scale * eps.double()
    c = -0.5 * d * math.log(2 * math.pi)
    lqr = c - torch.sum(torch.log(scale) + 0.5 * eps.double() ** 2, 2)
    lpr = c - torch.sum(torch.log(scale) + 0.5 * ((zr.detach() - loc) / scale) ** 2, 2)
    ((zr * gz.double()).sum() + (lqr * glq.double()).sum() + (lpr * glq.double()).sum()).backward()
    _close(z.detach(), zr.detach(), "z", 1e-5)
    _close(lq.detach(), lqr.detach(), "log_q", 1e-5)
    _close(lp.detach(), lpr.detach(), "log_prob", 1e-5)
    _close(q.loc.grad, loc.grad, "g_loc")
    _close(q.scale.grad, scale.grad, "g_scale")


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,n,latent", [(0, 3, 784, 40), (1, 1, 1, 1), (1061, 1, 12, 4), (5, 3, 784, 40),
                                          (33, 32, 784, 40), (7, 32, 64, 64)])
def test_decoders_match_fp64(B, S, n, latent):
    """NNBernoulliDecoder.log_prob (and its g_x), NNDiagGaussianDecoder.log_prob (x repeated S times, in place) and
    NNBernoulliDecoder.forward against fp64 torch on the same net outputs."""
    from normflows import _vae
    g = torch.Generator().manual_seed(B * 7 + S + n)
    N = B * S
    score0 = (torch.randn(N, n, generator=g) * 3).cuda()
    score0[:, :1] = 0.0                                         # exact zeros: the zero-score rule
    x0 = (torch.rand(B, n, generator=g) > 0.5).float().cuda()
    glp = torch.randn(N, generator=g).cuda()
    score, x = score0.clone().requires_grad_(True), x0.clone().requires_grad_(True)
    lp = _vae.bernoulli_log_prob(score, x, S)
    with torch.no_grad():
        assert torch.equal(lp, _vae.bernoulli_log_prob(score0, x0, S))
    (lp * glp).sum().backward()
    sd, xd = score0.double().requires_grad_(True), x0.double().requires_grad_(True)
    xr = xd.repeat_interleave(S, 0)
    ref = torch.sum(xr * V._log_sig(sd) + (1 - xr) * V._log_sig(-sd), 1)
    (ref * glp.double()).sum().backward()
    _close(lp.detach(), ref.detach(), "bernoulli log_p", 1e-5)
    _close(score.grad, sd.grad, "g_score")
    _close(x.grad, xd.grad, "g_x")
    assert (score.grad[:, 0] == 0).all()
    y = _vae.sigmoid(score)
    (y * score0).sum().backward()
    _close(y.detach(), torch.sigmoid(sd.detach()), "sigmoid", 1e-6)
    # the Gaussian decoder: net output [N, 2 n], x [B, n] read S times
    net0 = torch.randn(N, 2 * n, generator=g).cuda() * 0.5
    xv0 = torch.randn(B, n, generator=g).cuda()
    net, xv = net0.clone().requires_grad_(True), xv0.clone().requires_grad_(True)
    out = _vae.gaussian_log_prob(xv, N, S, 1, latent, net=net)
    (out * glp).sum().backward()
    nd, xvd = net0.double().requires_grad_(True), xv0.double().requires_grad_(True)
    mean, lv = nd[:, :n], nd[:, n:]
    xr = xvd.repeat_interleave(S, 0)
    ref = -0.5 * latent * math.log(2 * math.pi) - 0.5 * torch.sum(lv + (xr - mean) ** 2 / torch.exp(lv), 1)
    (ref * glp.double()).sum().backward()
    _close(out.detach(), ref.detach(), "gaussian decoder log_p", 1e-5)
    _close(net.grad, nd.grad, "g_net")
    _close(xv.grad, xvd.grad, "g_x (gaussian)")


@pytest.mark.gpu
def test_two_runs_are_bitwise_equal():
    gd = _golden("e")
    model, x, _ = _gpu_model("e", gd)
    grads, vals = [], []
    for _ in range(2):
        model.zero_grad()
        z, log_q, log_p = model(x, 32)
        (log_q.mean() - log_p.mean()).backward()
        vals.append((z.detach().clone(), log_q.detach().clone(), log_p.detach().clone()))
        grads.append([p.grad.clone() for p in model.parameters()])
    with torch.no_grad():
        z, log_q, log_p = model(x, 32)
    for a, b in zip(vals[0], vals[1]):
        assert torch.equal(a, b)
    for a, b in zip(vals[0], (z, log_q, log_p)):   # with and without grad
        assert torch.equal(a, b)
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_in_place_change_refuses_the_backward_and_cpu_inputs_raise():
    import normflows as nf
    gd = _golden("d")
    model, x, _ = _gpu_model("d", gd)
    z, log_q, log_p = model(x, 3)
    with torch.no_grad():
        model.q0.scale.add_(0.01)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        (log_q.mean() - log_p.mean()).backward()
    gd = _golden("a")
    model, x, _ = _gpu_model("a", gd)
    with pytest.raises(RuntimeError, match="CUDA"):
        model(x.cpu(), 3)
    dec = nf.distributions.NNBernoulliDecoder(nf.nets.MLP([4, 8, 12])).cuda()
    with pytest.raises(RuntimeError, match="CUDA"):
        dec.log_prob(x.cpu(), torch.zeros(5, 4, device="cuda"))


@pytest.mark.gpu
def test_flows_without_a_differentiable_sampling_direction_raise_under_grad():
    import normflows as nf
    torch.manual_seed(0)
    d = 4
    flows = [nf.flows.AutoregressiveRationalQuadraticSpline(d, 1, 16), nf.flows.LULinearPermute(d)]
    enc = nf.distributions.NNDiagGaussian(nf.nets.MLP([12, 16, 2 * d]))
    dec = nf.distributions.NNBernoulliDecoder(nf.nets.MLP([d, 16, 12]))
    model = nf.NormalizingFlowVAE(V.mvn(d, "cuda"), enc, flows, dec).cuda()
    x = (torch.rand(6, 12, device="cuda") > 0.5).float()
    with pytest.raises(NotImplementedError, match="gradients through the sampling direction are not on the CUDA path"):
        model(x, 2)
    with torch.no_grad():
        z, log_q, log_p = model(x, 2)
    assert z.shape == (6, 2, d) and log_q.shape == (6, 2) and log_p.shape == (6, 2)
    assert torch.isfinite(z).all() and torch.isfinite(log_q).all() and torch.isfinite(log_p).all()


@pytest.mark.gpu
def test_image_shaped_data_raise():
    import normflows as nf
    enc = nf.distributions.NNDiagGaussian(nf.nets.MLP([12, 8])).cuda()
    with pytest.raises(NotImplementedError, match="flat"):
        enc(torch.zeros(2, 3, 4, device="cuda"), 1)


def _notebook(flow_type, device="cuda", n_bottleneck=40, n_flows=40, init_zeros=False):
    """examples/vae.ipynb's model cell as written (n_bottleneck = n_flows = 40, init_zeros False)."""
    import normflows as nf
    hidden_units_encoder = np.array([28 ** 2, 512, 256, n_bottleneck * 2])
    hidden_units_decoder = np.array([n_bottleneck, 256, 512, 28 ** 2])
    prior = torch.distributions.MultivariateNormal(torch.zeros(n_bottleneck, device=device),
                                                   torch.eye(n_bottleneck, device=device))
    encoder = nf.distributions.NNDiagGaussian(nf.nets.MLP(hidden_units_encoder))
    decoder = nf.distributions.NNBernoulliDecoder(nf.nets.MLP(hidden_units_decoder))
    if flow_type == 'Planar':
        flows = [nf.flows.Planar((n_bottleneck,)) for k in range(n_flows)]
    elif flow_type == 'Radial':
        flows = [nf.flows.Radial((n_bottleneck,)) for k in range(n_flows)]
    else:
        b = torch.tensor(n_bottleneck // 2 * [0, 1] + n_bottleneck % 2 * [0])
        flows = []
        for i in range(n_flows):
            s = nf.nets.MLP([n_bottleneck, n_bottleneck], init_zeros=init_zeros)
            t = nf.nets.MLP([n_bottleneck, n_bottleneck], init_zeros=init_zeros)
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
    nfm = nf.NormalizingFlowVAE(prior, encoder, flows, decoder)
    return nfm.to(device)


def synthetic_mnist(n, seed=0):
    """Binarised 28 x 28 'digits': a few seeded blob templates plus pixel noise, flattened to [n, 784]."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(28.0), torch.arange(28.0), indexing="ij")
    templates = []
    for k in range(10):
        cy, cx = 8 + torch.rand(2, generator=g) * 12
        r = 4 + 3 * torch.rand(1, generator=g)
        templates.append((((yy - cy) ** 2 + (xx - cx) ** 2).sqrt() - r).abs() < 1.5)
    T = torch.stack(templates).float().reshape(10, 784)
    idx = torch.randint(0, 10, (n,), generator=g)
    flip = torch.rand(n, 784, generator=g) < 0.03
    return (T[idx] != flip.float()).float()


@pytest.mark.gpu
def test_notebook_training_cell_trains():
    """The notebook's optimizer and loop, 200 steps of batch 64 on synthetic binarised 28 x 28 data."""
    from torch import optim
    torch.manual_seed(0)
    nfm = _notebook("Planar")
    data = synthetic_mnist(200 * 64).cuda()
    num_samples = 32
    before = {n: p.detach().clone() for n, p in nfm.named_parameters()}
    optimizer = optim.Adam(nfm.parameters(), lr=1e-4, weight_decay=1e-4)
    hist, seen = [], set()
    for it in range(200):
        x = data[it * 64:(it + 1) * 64]
        optimizer.zero_grad()
        z, log_q, log_p = nfm(x.view(x.size(0), 28 ** 2), num_samples)
        loss = torch.mean(log_q) - torch.mean(log_p)
        loss.backward()
        seen |= {n for n, p in nfm.named_parameters() if p.grad is not None and p.grad.abs().max() > 0}
        optimizer.step()
        hist.append(loss.item())
    h = np.array(hist)
    assert np.isfinite(h).all()
    assert h[-20:].mean() < h[:20].mean(), (h[:20].mean(), h[-20:].mean())
    names = {n for n, _ in nfm.named_parameters()}
    assert seen == names, names - seen
    for n, p in nfm.named_parameters():
        assert not torch.equal(p.detach(), before[n]), n
    x_out = nfm.decoder(torch.randn((1, 40), device="cuda"))   # the notebook's last cell
    assert x_out.view((28, 28)).shape == (28, 28)


@pytest.mark.gpu
@pytest.mark.parametrize("flow_type", ["Radial", "RealNVP"])
def test_other_flow_types_run_one_step(flow_type):
    """RealNVP at the 16-feature setting of DESIGN §7's known limitation."""
    from torch import optim
    torch.manual_seed(0)
    nfm = _notebook(flow_type, **({"n_bottleneck": 16, "init_zeros": True} if flow_type == "RealNVP" else {}))
    optimizer = optim.Adam(nfm.parameters(), lr=1e-4, weight_decay=1e-4)
    x = synthetic_mnist(64).cuda()
    optimizer.zero_grad()
    z, log_q, log_p = nfm(x, 32)
    loss = torch.mean(log_q) - torch.mean(log_p)
    loss.backward()
    optimizer.step()
    assert np.isfinite(loss.item()) and z.shape == (64, 32, nfm.prior.loc.shape[0])
    for n, p in nfm.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
