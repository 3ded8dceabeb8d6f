"""The Gaussian-mixture base (reference distributions/base.py:573-659 GaussianMixture; the second model of
examples/change_base_distribution.ipynb): its log-density kernel and deterministic backward (csrc/nfb_mixture.cu), the
stand-alone MixtureLogProbFn, and the flow object's mixture base (nfb_flow_set_base_gaussian_mixture) under log_prob,
forward_kld and nfb_flow_log_prob_backward for every all-native stack.

CPU: the host-compiled element math (csrc/nfb_mixture.cuh) against fp64 autograd and central differences, far z, an
underflowing weight and a NaN row included; the fp64 restatement against the reference's goldens; construction, seeded
defaults and strict loading of reference state_dicts.
GPU: log_prob against the fp64 restatement over K, D and rows; gradients of the stand-alone Function and of fused
spline, affine, mixed and layer-loop stacks against fp64 autograd; reverse_kld on affine and planar stacks; the goldens;
K = 1 against DiagGaussian; bit-identical values and gradients; launch counts; zero rows; no use of the torch restatement;
the notebook's training cell."""
import copy
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import helpers_mixture as M
from conftest import ROOT

NEW_SYMBOLS = ("nfb_gaussian_mixture_log_prob", "nfb_gaussian_mixture_log_prob_backward",
               "nfb_gaussian_mixture_log_prob_backward_workspace_bytes", "nfb_flow_set_base_gaussian_mixture")


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


# ---- element math on the host -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "mixture_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "mixture_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_mixture(lib, z, loc, ls, ws, g, use_float=0):
    f = lambda v: np.ascontiguousarray(v, dtype=np.float64)
    z, loc, ls, ws, g = (f(v) for v in (z, loc, ls, ws, g))
    (n, D), K = z.shape, ws.size
    lp, gz, gl, gs, gw = np.empty(n), np.empty((n, D)), np.empty((K, D)), np.empty((K, D)), np.empty(K)
    P = lambda v: v.ctypes.data_as(C.c_void_p)
    lib.mixture_adjoint_check(C.c_int(K), C.c_int(D), C.c_int(n), C.c_int(use_float), P(z), P(loc), P(ls), P(ws), P(g),
                              P(lp), P(gz), P(gl), P(gs), P(gw))
    return lp, gz, gl, gs, gw


def torch_mixture(z, loc, ls, ws):
    """log p [N] in torch (any dtype), log_softmax for the weights; loc / ls [K, D], ws [K]."""
    e = (torch.log_softmax(ws, 0)[None] - 0.5 * z.shape[1] * math.log(2 * math.pi)
         - torch.sum(ls[None] + 0.5 * ((z[:, None, :] - loc[None]) / torch.exp(ls[None])) ** 2, 2))
    return torch.logsumexp(e, 1)


def autograd_mixture(z, loc, ls, ws, g):
    xs = [torch.tensor(np.asarray(v, np.float64), requires_grad=True) for v in (z, loc, ls, ws)]
    lp = torch_mixture(*xs)
    (lp * torch.as_tensor(g)).sum().backward()
    return lp.detach().numpy(), [v.grad.numpy() for v in xs]


def _params(rng, K, D, spread=1.0):
    return rng.normal(size=(K, D)) * spread, rng.normal(size=(K, D)) * 0.4, rng.normal(size=K)


@pytest.mark.parametrize("K,D", [(1, 1), (2, 2), (3, 5), (7, 3)])
def test_host_element_math_matches_autograd_and_central_differences(mixlib, K, D):
    rng = np.random.default_rng(K * 10 + D)
    loc, ls, ws = _params(rng, K, D)
    z, g = rng.normal(size=(13, D)) * 1.5, rng.normal(size=13)
    lp, gz, gl, gs, gw = host_mixture(mixlib, z, loc, ls, ws, g)
    lp_a, (gz_a, gl_a, gs_a, gw_a) = autograd_mixture(z, loc, ls, ws, g)
    np.testing.assert_allclose(lp, lp_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(lp, M.log_prob(z, loc, ls, ws), rtol=1e-12, atol=1e-12)
    for a, r in ((gz, gz_a), (gl, gl_a), (gs, gs_a), (gw, gw_a)):
        np.testing.assert_allclose(a, r, rtol=1e-10, atol=1e-12)
    for a, r in zip((gz, gl, gs, gw), M.log_prob_grads(z, loc, ls, ws, g)):
        np.testing.assert_allclose(a, r, rtol=1e-10, atol=1e-12)
    h = 1e-6
    args = [z, loc, ls, ws]
    for i, got in enumerate((gz, gl, gs, gw)):
        fd = np.zeros_like(got).reshape(-1)
        for j in range(fd.size):
            hi = [a.copy() for a in args]
            lo = [a.copy() for a in args]
            hi[i].reshape(-1)[j] += h
            lo[i].reshape(-1)[j] -= h
            fd[j] = ((M.log_prob(*hi) - M.log_prob(*lo)) * g).sum() / (2 * h)
        np.testing.assert_allclose(got.reshape(-1), fd, rtol=1e-5, atol=1e-6)
    f32 = host_mixture(mixlib, z, loc, ls, ws, g, use_float=1)
    for a, r in zip(f32, (lp, gz, gl, gs, gw)):
        np.testing.assert_allclose(a, r, rtol=1e-4, atol=1e-4 * max(1.0, np.abs(r).max()))


def test_host_far_z_underflowing_weight_and_nan_row(mixlib):
    rng = np.random.default_rng(3)
    K, D = 3, 2
    loc, ls, _ = _params(rng, K, D)
    ls[:] = np.log(0.001)
    ws = np.array([0.0, -800.0, 0.5])   # softmax of mode 1 underflows (the reference's log(softmax) gives -inf there)
    z = rng.normal(size=(6, D))
    z[0] = [1.0, -1.0]                  # exponents near -5e5 for every mode
    z[3] = [np.nan, 0.0]
    g = np.ones(6)
    for use_float in (0, 1):
        lp, gz, gl, gs, gw = host_mixture(mixlib, z, loc, ls, ws, g, use_float)
        ok = np.arange(6) != 3
        assert np.isfinite(lp[ok]).all() and np.isfinite(gz[ok]).all(), (use_float, lp, gz)
        assert np.isnan(lp[3]) and np.isnan(gz[3]).all()
        assert lp[0] < -1e5
        np.testing.assert_allclose(lp[ok], M.log_prob(z[ok], loc, ls, ws), rtol=1e-6 if use_float else 1e-12)
        _, gl, gs, gw = host_mixture(mixlib, z[ok], loc, ls, ws, g[ok], use_float)[1:]
        assert np.isfinite(gl).all() and np.isfinite(gs).all() and np.isfinite(gw).all()
    for a, r in zip(host_mixture(mixlib, z[ok], loc, ls, ws, g[ok])[1:], M.log_prob_grads(z[ok], loc, ls, ws, g[ok])):
        np.testing.assert_allclose(a, r, rtol=1e-9, atol=1e-9 * max(1.0, np.abs(r).max()))


# ---- goldens: the reference (tests/golden/make_mixture_grads.py) --------------------------------------------------------
def _golden(name):
    from helpers import load_npz_parts
    return load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_mix_{name}.npz"))


def test_oracle_matches_reference_log_prob_values():
    gd = _golden("values")
    for name in M.value_cases():
        sd = {k.split("__sd__")[1]: gd[k] for k in gd if k.startswith(name + "__sd__")}
        got = M.log_prob(gd[name + "__z"], sd["loc"][0], sd["log_scale"][0], sd["weight_scores"][0])
        np.testing.assert_allclose(got, gd[name + "__log_prob"], rtol=1e-10, atol=0, err_msg=name)


def test_construction_matches_reference_state_dicts():
    """Keys, shapes and (float32-rounded) values of seeded and explicit construction; strict loading of the reference's
    float64 state_dicts; trainable=False registers buffers."""
    import normflows as nf
    gd = _golden("values")
    for name, spec in M.value_cases().items():
        q = M.value_case_model(nf, spec)
        ref = {k.split("__sd__")[1]: gd[k] for k in gd if k.startswith(name + "__sd__")}
        own = q.state_dict()
        assert list(own) == ["loc", "log_scale", "weight_scores"] and set(own) == set(ref), name
        for k, v in own.items():
            assert tuple(v.shape) == ref[k].shape and v.dtype == torch.float32, (name, k)
            np.testing.assert_allclose(v.numpy(), ref[k].astype(np.float32), rtol=0, atol=0, err_msg=f"{name} {k}")
        q2 = nf.distributions.GaussianMixture(spec["kw"]["n_modes"], spec["kw"]["dim"])
        q2.load_state_dict({k: torch.tensor(v) for k, v in ref.items()}, strict=True)
        for k, v in q2.state_dict().items():
            assert v.dtype == torch.float32 and torch.equal(v, own[k]), (name, k)
    q = nf.distributions.base.GaussianMixture(3, 2, trainable=False)
    assert not list(q.parameters()) and sorted(dict(q.named_buffers())) == ["loc", "log_scale", "weight_scores"]


def _restated_fkl(model, x):
    """fp64 forward_kld: the layers' density direction by _autograd.layer_inverse, the base by torch_mixture."""
    from normflows._autograd import layer_inverse
    z, lq = x, x.new_zeros(x.shape[0])
    for f in reversed(list(model.flows)):
        z, ld = layer_inverse(f, z)
        lq = lq + ld
    q = model.q0
    return -torch.mean(lq + torch_mixture(z, q.loc[0], q.log_scale[0], q.weight_scores[0]))


def _golden_model(name, dtype=torch.float32):
    """The case built by this package (on the CPU) with the golden's parameters, in `dtype` (the reference's mixture
    holds float64 parameters: float64 keeps them exact)."""
    import normflows as nf
    gd = _golden(name)
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    model = M.build(nf, name).to(dtype)
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    model.load_state_dict({k: sd[k].to(v.dtype) for k, v in own.items()}, strict=True)
    return model, torch.tensor(gd["x"]), gd


def _check_golden(got, gd, name, tol):
    from test_maf_training import check_golden
    check_golden(got, gd, name, tol)


@pytest.mark.parametrize("name", ["cbd", "nsf"])
def test_fp64_restatement_matches_reference_goldens(name):
    model, x, gd = _golden_model(name, torch.float64)
    loss = _restated_fkl(model, x.double())
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    for n, p in model.named_parameters():
        if "g__" + n in gd or "gv__" + n in gd:
            _check_golden(p.grad, gd, n, 1e-10)


# ================================================ GPU ================================================================
def _close(got, ref, name, tol=2e-3):
    from test_affine_rkl_training import _close as close
    close(got, ref, name, tol)


def _mixture(K, D, seed, spread=2.0):
    import normflows as nf
    np.random.seed(seed)
    q = nf.distributions.GaussianMixture(K, D, scale=np.exp(np.random.normal(size=(K, D)) * 0.4),
                                         weights=np.random.uniform(0.2, 1.0, size=K))
    with torch.no_grad():
        q.loc.mul_(spread)
    return q


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 2, 3, 8, 40, 200])
@pytest.mark.parametrize("D", [1, 2, 5, 64, 130])
def test_log_prob_matches_oracle(K, D):
    """rows 0, 1, 37 and 65 536 (a sample of 600 rows, the last ones included, checked against the oracle)."""
    q = _mixture(K, D, K * 1000 + D).cuda()
    sd = [t.detach().cpu().double().numpy()[0] for t in (q.loc, q.log_scale, q.weight_scores)]
    g = torch.Generator().manual_seed(K + D)
    for rows in (0, 1, 37, 65536):
        z = (torch.randn(rows, D, generator=g) * 2.5).cuda()
        with torch.no_grad():
            lp = q.log_prob(z).cpu().numpy()
        assert lp.shape == (rows,)
        idx = np.unique(np.r_[np.arange(min(rows, 300)), np.arange(max(0, rows - 300), rows)])
        ref = M.log_prob(z.cpu().double().numpy()[idx], *sd)
        np.testing.assert_allclose(lp[idx], ref, rtol=1e-4, atol=0, err_msg=f"K={K} D={D} rows={rows}")


def _standalone_grads(q, z, g):
    zz = z.clone().requires_grad_(True)
    lp = q.log_prob(zz)
    (lp * g).sum().backward()
    return lp.detach(), [zz.grad] + [p.grad for p in (q.loc, q.log_scale, q.weight_scores)]


@pytest.mark.gpu
@pytest.mark.parametrize("K,D,rows", [(1, 1, 1), (2, 2, 37), (3, 5, 1000), (8, 64, 3000), (40, 3, 65541),
                                      (200, 130, 300), (3, 2, 70000)])
def test_standalone_gradients_match_fp64(K, D, rows):
    """65 541 and 70 000 rows: more row blocks than the backward's CTAs, each CTA walks several."""
    q = _mixture(K, D, 7 * K + D).cuda()
    gen = torch.Generator().manual_seed(rows)
    z = (torch.randn(rows, D, generator=gen) * 2.5).cuda()
    g = torch.randn(rows, generator=gen).cuda()
    _, got = _standalone_grads(q, z, g)
    sd = [t.detach().cpu().double().numpy()[0] for t in (q.loc, q.log_scale, q.weight_scores)]
    ref = M.log_prob_grads(z.cpu().double().numpy(), *sd, g.cpu().double().numpy())
    for name, a, r in zip(("g_z", "g_loc", "g_log_scale", "g_weight_scores"), got, ref):
        _close(a.reshape(r.shape).cpu(), torch.tensor(r), name)


def _stack(kind, D, seed):
    """An all-native stack on a mixture base: spline + LU (fused), affine (every op variant) or mixed."""
    import normflows as nf
    from test_affine_rkl_training import _randomise, make_stack
    torch.manual_seed(seed)
    if kind == "spline":
        flows = []
        for _ in range(2):
            flows += [nf.flows.AutoregressiveRationalQuadraticSpline(D, 1, 32), nf.flows.LULinearPermute(D)]
        for f in flows:
            _randomise(f, seed + len(flows), 0.3)
    elif kind == "affine":
        flows = make_stack(D, 16, 2, 0.2, seed)
    else:
        flows = make_stack(D, 16, 2, 0.0, seed)[:3] + [nf.flows.AutoregressiveRationalQuadraticSpline(D, 1, 16),
                                                       nf.flows.LULinearPermute(D)]
        for f in flows[3:]:
            _randomise(f, seed + 9, 0.3)
    return nf.NormalizingFlow(_mixture(3, D, seed, 1.0), flows).cuda()


def _restated_log_prob(model, x):
    from normflows import _autograd
    return _autograd.log_prob(model, x)


def _clone(model):
    """A deep copy without the cached flow object (whose native handle must have one owner)."""
    h = model.__dict__.pop("_nfb_stack", None)
    c = copy.deepcopy(model)
    if h is not None:
        model.__dict__["_nfb_stack"] = h
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,rows", [("spline", 2, 300), ("spline", 5, 1000), ("spline", 64, 700),
                                         ("affine", 2, 500), ("affine", 5, 300), ("affine", 16, 200),
                                         ("mixed", 5, 400)])
def test_flow_object_log_prob_and_gradients_match_fp64(kind, D, rows):
    model = _stack(kind, D, seed=D + rows)
    assert model._stack() is not None and model._stack().base is model.q0
    gen = torch.Generator().manual_seed(rows)
    x0 = torch.randn(rows, D, generator=gen).cuda()
    g = torch.randn(rows, generator=gen).cuda()
    x = x0.clone().requires_grad_(True)
    lq = model.log_prob(x)
    (lq * g).sum().backward()
    with torch.no_grad():   # (the fused spline kernel is not bit-reproducible run to run; the affine stack is)
        lq0 = model.log_prob(x0)
        assert torch.equal(lq0, lq.detach()) if kind == "affine" else torch.allclose(lq0, lq.detach(), rtol=1e-6)
        assert abs(float(model.forward_kld(x0)) + lq.mean().item()) <= 1e-5 * (1 + abs(lq.mean().item()))
    ref = _clone(model).double()
    xd = x0.double().requires_grad_(True)
    lr = _restated_log_prob(ref, xd)
    (lr * g.double()).sum().backward()
    _close(lq.detach(), lr.detach(), "log_q", 1e-4)
    _close(x.grad, xd.grad, "g_x")
    for (n, p), (_, pr) in zip(model.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, n
        _close(p.grad, pr.grad, n)
    assert len([n for n, _ in model.named_parameters() if n.startswith("q0.")]) == 3


@pytest.mark.gpu
def test_host_entry_points_use_the_mixture():
    model = _stack("affine", 5, seed=3)
    x = torch.randn(1000, 5)
    with torch.no_grad():
        lq = model.log_prob(x.cuda()).cpu()
        kld = float(model.forward_kld(x.cuda()))
    torch.testing.assert_close(model.log_prob_host(x), lq, rtol=0, atol=0)
    assert abs(model.forward_kld_host(x) - kld) <= 1e-6 * (1 + abs(kld))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["cbd", "nsf", "loop"])
def test_model_gradients_match_reference_goldens(name):
    """cbd: affine stack, nsf: fused spline + LU stack, loop: Residual + ActNorm layer by layer (the base through
    MixtureLogProbFn)."""
    model, x, gd = _golden_model(name)
    model = model.cuda()
    model.train(name != "loop")
    assert (model._stack() is None) == (name == "loop")
    loss = model.forward_kld(x.cuda())
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    for n, p in model.named_parameters():
        if "g__" + n in gd or "gv__" + n in gd:
            assert p.grad is not None, n
            _check_golden(p.grad, gd, n, 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["affine", "planar"])
def test_reverse_kld_is_differentiable_and_matches_fp64(kind):
    """reverse_kld through a mixture base: the same draws (torch.multinomial, torch.randn after the same seed) pushed
    through an fp64 restatement of the base and the stack's sampling direction."""
    import normflows as nf
    D = 2
    if kind == "affine":
        from test_affine_rkl_training import make_stack, sample_restated
        flows = make_stack(D, 16, 2, 0.2, 4)
    else:
        from test_planar_radial_training import make_stack, sample_restated
        flows = make_stack(D, 6, 4)
    model = nf.NormalizingFlow(_mixture(3, D, 11, 1.0), flows, nf.distributions.TwoMoons()).cuda()
    torch.manual_seed(5)
    loss = model.reverse_kld(2000)
    loss.backward()
    P = {id(p): p.detach().double().requires_grad_(True) for p in model.parameters()}
    q = model.q0
    loc, ls, ws = (P[id(t)] for t in (q.loc, q.log_scale, q.weight_scores))
    torch.manual_seed(5)
    mode = torch.multinomial(torch.softmax(q.weight_scores.detach(), 1)[0], 2000, replacement=True)
    eps = torch.randn(2000, D, device="cuda")
    z = loc[0, mode] + torch.exp(ls[0, mode]) * eps.double()
    lq0 = torch_mixture(z, loc[0], ls[0], ws[0])
    x, ld = sample_restated(model.flows, z, P)
    ref = torch.mean(lq0 - ld) - torch.mean(model.p.log_prob(x))
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-4 * (1 + abs(ref.item())), (loss.item(), ref.item())
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
        _close(p.grad, P[id(p)].grad, n)


@pytest.mark.gpu
def test_k1_agrees_with_diag_gaussian():
    import normflows as nf
    D = 5
    mix = _stack("affine", D, seed=8)
    diag = _clone(mix)
    diag.q0 = nf.distributions.DiagGaussian(D).cuda()
    mix.q0 = nf.distributions.GaussianMixture(1, D).cuda()
    with torch.no_grad():
        diag.q0.loc.normal_(0, 0.5)
        diag.q0.log_scale.normal_(0, 0.3)
        mix.q0.loc.copy_(diag.q0.loc[None])
        mix.q0.log_scale.copy_(diag.q0.log_scale[None])
    x = torch.randn(500, D, device="cuda")
    for m in (mix, diag):
        m.forward_kld(x).backward()
    with torch.no_grad():
        torch.testing.assert_close(mix.log_prob(x), diag.log_prob(x), rtol=1e-5, atol=1e-5)
    for (n, a), (_, b) in zip(mix.flows.named_parameters(), diag.flows.named_parameters()):
        torch.testing.assert_close(a.grad, b.grad, rtol=1e-4, atol=1e-5 * (1 + b.grad.abs().max().item()))
    torch.testing.assert_close(mix.q0.loc.grad[0], diag.q0.loc.grad, rtol=1e-4, atol=1e-6)
    torch.testing.assert_close(mix.q0.log_scale.grad[0], diag.q0.log_scale.grad, rtol=1e-4, atol=1e-6)
    assert mix.q0.weight_scores.grad.abs().max() < 1e-6


@pytest.mark.gpu
def test_bit_identical_values_and_gradients():
    model = _stack("affine", 5, seed=2)
    q = model.q0
    x = torch.randn(5000, 5, device="cuda")
    with torch.no_grad():
        lq0 = model.log_prob(x)
        lp0 = q.log_prob(x)
    grads = []
    for _ in range(2):
        model.zero_grad()
        lq = model.log_prob(x)
        lp = q.log_prob(x.clone().requires_grad_(True))
        assert torch.equal(lq, lq0) and torch.equal(lp, lp0)
        (lq.sum() + lp.square().sum()).backward()
        grads.append([p.grad.clone() for p in model.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_launch_counts():
    """log_prob of an all-native stack launches as many kernels on a mixture as on a DiagGaussian; the stand-alone
    backward is two kernels whatever rows and K."""
    import normflows as nf
    from torch.profiler import ProfilerActivity, profile
    for kind in ("spline", "affine"):
        mix = _stack(kind, 5, seed=1)
        diag = _clone(mix)
        diag.q0 = nf.distributions.DiagGaussian(5).cuda()
        x = torch.randn(3000, 5, device="cuda")
        counts = []
        for m in (mix, diag):
            with torch.no_grad():
                m.log_prob(x)
            counts.append(m._stack().launch_count())
        assert counts[0] == counts[1], (kind, counts)
    seen = set()
    for K, rows in ((2, 100), (50, 70000)):
        q = _mixture(K, 3, K).cuda()
        z = torch.randn(rows, 3, device="cuda", requires_grad=True)
        lp = q.log_prob(z)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lp.sum().backward()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type.name == "CUDA" and "mixture" in e.name]
        seen.add(len(names))
        assert len(names) == 2, names
    assert seen == {2}


@pytest.mark.gpu
def test_zero_rows_give_zero_gradients():
    q = _mixture(3, 4, 1).cuda()
    z = torch.zeros(0, 4, device="cuda", requires_grad=True)
    q.log_prob(z).sum().backward()
    for p in (q.loc, q.log_scale, q.weight_scores):
        assert p.grad is not None and (p.grad == 0).all()
    model = _stack("affine", 4, seed=2)
    model.log_prob(torch.zeros(0, 4, device="cuda", requires_grad=True)).sum().backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and (p.grad == 0).all(), n


@pytest.mark.gpu
def test_the_torch_restatement_is_not_reached(monkeypatch):
    import normflows._autograd as AG

    def refuse(*a, **k):
        raise AssertionError("the torch restatement was reached")
    monkeypatch.setattr(AG, "log_prob", refuse)
    monkeypatch.setattr(AG, "layer_inverse", refuse)
    for kind, D in (("spline", 5), ("affine", 2), ("mixed", 5)):
        model = _stack(kind, D, seed=4)
        model.forward_kld(torch.randn(300, D, device="cuda")).backward()
        for n, p in model.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), n


@pytest.mark.gpu
def test_change_base_distribution_training_cell_trains():
    """The second training cell of examples/change_base_distribution.ipynb, 300 iterations."""
    import normflows as nf
    torch.manual_seed(0)
    model = M.cbd(nf).cuda()
    target = nf.distributions.TwoMoons()
    optimizer = torch.optim.Adam(model.parameters(), lr=5e-4, weight_decay=1e-5)
    hist = []
    for it in range(300):
        optimizer.zero_grad()
        x = target.sample(2 ** 9).cuda()
        loss = model.forward_kld(x)
        if ~(torch.isnan(loss) | torch.isinf(loss)):
            loss.backward()
            optimizer.step()
        hist.append(loss.item())
    h = np.array(hist)
    assert np.isfinite(h).all() and h[:10].mean() > h[-10:].mean() + 0.1, (h[:10].mean(), h[-10:].mean())
    for n, p in model.named_parameters():
        assert torch.isfinite(p).all(), n
