"""Planar and radial flows (examples/planar.ipynb, examples/comparison_plan_rad_aff.ipynb): `nf.flows.Planar` /
`nf.flows.Radial`, whose stack runs as one planar_stack_kernel launch and whose sampling direction is differentiated by
one nfb_flow_sampling_backward call, and the comparison notebook's targets.

CPU: the per-layer constants, element adjoints and parameter chains (csrc/nfb_planar_bwd.cuh), compiled for the host,
against fp64 autograd of the reference's formulas and central differences, including the edge cases (softplus overflow,
saturated tanh, leaky ReLU at 0, z = z_0, alpha = 0); constructors, state_dicts and seeded initial values against the
reference's, strict loading; the targets against the reference's values; an fp64 restatement against goldens r-v; the
NotImplementedErrors.
GPU: stacks against fp64 autograd of a torch restatement, bit-identical values with and without grad, reproducible
gradients, the in-place refusal, zero rows, shared parameters, launch counts, goldens r-v, the notebooks' training."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- fp64 torch restatement of the reference's formulas (flows/planar.py:51-81, flows/radial.py:37-46) --------------
def planar_fwd(z, u, w, b, act, slope=0.2):
    lin = torch.sum(w * z, 1, keepdim=True) + b
    inner = torch.sum(w * u)
    u = u + (torch.log(1 + torch.exp(inner)) - 1 - inner) * w / torch.sum(w ** 2)
    if act == "tanh":
        h, hp = torch.tanh(lin), 1 / torch.cosh(lin.reshape(-1)) ** 2
    else:
        h = torch.nn.functional.leaky_relu(lin, slope)
        hp = (lin.reshape(-1) < 0) * (slope - 1.0) + 1.0
    return z + u * h, torch.log(torch.abs(1 + torch.sum(w * u) * hp))


def radial_fwd(z, z0, alpha, beta):
    bh = torch.log(1 + torch.exp(beta)) - torch.abs(alpha)
    dz = z - z0
    r = torch.linalg.vector_norm(dz, dim=1, keepdim=True)
    h = bh / (torch.abs(alpha) + r)
    h_ = -bh * r / (torch.abs(alpha) + r) ** 2
    return z + h * dz, ((z.shape[1] - 1) * torch.log(1 + h) + torch.log(1 + h + h_)).reshape(-1)


def sample_restated(layers, z, P):
    """fp64 (x, log_det) of the layers' sampling direction; P maps id(parameter) -> its fp64 leaf."""
    import normflows as nf
    ld = z.new_zeros(z.shape[0])
    for f in layers:
        if isinstance(f, nf.flows.Planar):
            z, l = planar_fwd(z, P[id(f.u)], P[id(f.w)], P[id(f.b)], f.act)
        else:
            z, l = radial_fwd(z, P[id(f.z_0)], P[id(f.alpha)], P[id(f.beta)])
        ld = ld + l
    return z, ld


# ---- element adjoints on the host ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def adjlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "planar_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "planar_adjoint_host_check.cu")])
    return C.CDLL(so)


def _a(v):
    return np.ascontiguousarray(v, dtype=np.float64)


def _P(v):
    return v.ctypes.data_as(C.c_void_p)


def host_planar(lib, act, z, u, w, b, g, gam, use_float=0):
    n, d = z.shape
    z, u, w, g, gam = map(_a, (z, u, w, g, gam))
    gz, gu, gw, gb, cst = np.empty((n, d)), np.empty(d), np.empty(d), np.empty(1), np.empty(2)
    lib.planar_layer_check(C.c_int(use_float), C.c_int(0 if act == "tanh" else 1), C.c_double(0.2), C.c_int(n),
                           C.c_int(d), _P(z), _P(u), _P(w), C.c_double(b), _P(g), _P(gam), _P(gz), _P(gu), _P(gw),
                           _P(gb), _P(cst))
    return gz, gu, gw, gb[0], cst


def host_radial(lib, z, z0, alpha, beta, g, gam, use_float=0):
    n, d = z.shape
    z, z0, g, gam = map(_a, (z, z0, g, gam))
    gz, gz0, gbe, gal, cst = np.empty((n, d)), np.empty(d), np.empty(1), np.empty(1), np.empty(2)
    lib.radial_layer_check(C.c_int(use_float), C.c_int(n), C.c_int(d), _P(z), _P(z0), C.c_double(alpha),
                           C.c_double(beta), _P(g), _P(gam), _P(gz), _P(gz0), _P(gbe), _P(gal), _P(cst))
    return gz, gz0, gbe[0], gal[0], cst


def autograd_planar(act, z, u, w, b, g, gam):
    t = [torch.tensor(_a(v), requires_grad=True) for v in (z, u.reshape(1, -1), w.reshape(1, -1), [b])]
    x, ld = planar_fwd(*t, act)
    (torch.tensor(_a(g)) * x).sum().backward(retain_graph=True)
    (torch.tensor(_a(gam)) * ld).sum().backward()
    return [v.grad.numpy() for v in t]


def autograd_radial(z, z0, alpha, beta, g, gam):
    t = [torch.tensor(_a(v), requires_grad=True) for v in (z, z0.reshape(1, -1), [alpha], [beta])]
    x, ld = radial_fwd(*t)
    ((torch.tensor(_a(g)) * x).sum() + (torch.tensor(_a(gam)) * ld).sum()).backward()
    return [v.grad.numpy() for v in t]


def _loss_planar(act, z, u, w, b, g, gam):
    x, ld = planar_fwd(*[torch.tensor(_a(v)) for v in (z, u.reshape(1, -1), w.reshape(1, -1), [b])], act)
    return float((torch.tensor(g) * x).sum() + (torch.tensor(gam) * ld).sum())


@pytest.mark.parametrize("act", ["tanh", "leaky_relu"])
@pytest.mark.parametrize("d", [1, 2, 5])
def test_planar_adjoint_matches_autograd_and_central_differences(adjlib, act, d):
    rng = np.random.default_rng(d + (act == "tanh"))
    n = 64
    z, g = rng.normal(size=(n, d)), rng.normal(size=(n, d))
    gam = rng.normal(size=n)
    u, w, b = rng.normal(size=d), rng.normal(size=d) * 0.8, 0.3
    gz, gu, gw, gb, _ = host_planar(adjlib, act, z, u, w, b, g, gam)
    az, au, aw, ab = autograd_planar(act, z, u, w, b, g, gam)
    # (the reference forms the leaky h' = (lin < 0)(slope - 1) + 1 in float32, a bool tensor times a Python float, and
    # u_hat's normalisation by |w|^2 amplifies rounding: fp64 agreement to 1e-7 of each scale)
    for got, ref in ((gz, az), (gu, au[0]), (gw, aw[0]), (gb, ab[0])):
        np.testing.assert_allclose(got, ref, rtol=1e-7, atol=1e-7 * np.abs(ref).max())
    h = 1e-4
    for j in range(d if act == "tanh" else 0):   # (leaky: a kinked, badly conditioned loss; autograd above covers it)
        e = np.zeros(d)
        e[j] = h
        fd_u = (_loss_planar(act, z, u + e, w, b, g, gam) - _loss_planar(act, z, u - e, w, b, g, gam)) / (2 * h)
        fd_w = (_loss_planar(act, z, u, w + e, b, g, gam) - _loss_planar(act, z, u, w - e, b, g, gam)) / (2 * h)
        assert abs(fd_u - gu[j]) <= 1e-3 * (1 + abs(fd_u)) and abs(fd_w - gw[j]) <= 1e-3 * (1 + abs(fd_w))
    f32 = host_planar(adjlib, act, z, u, w, b, g, gam, use_float=1)
    for a, r in zip(f32[:4], (gz, gu, gw, gb)):
        np.testing.assert_allclose(a, r, rtol=2e-4, atol=2e-4 * np.abs(r).max())


@pytest.mark.parametrize("d", [1, 2, 5, 40])
def test_radial_adjoint_matches_autograd_and_central_differences(adjlib, d):
    rng = np.random.default_rng(10 + d)
    n = 64
    z, g = rng.normal(size=(n, d)), rng.normal(size=(n, d))
    gam = rng.normal(size=n)
    z0, alpha, beta = rng.normal(size=d), -0.4, 0.3
    gz, gz0, gbe, gal, _ = host_radial(adjlib, z, z0, alpha, beta, g, gam)
    az, az0, aal, abe = autograd_radial(z, z0, alpha, beta, g, gam)
    for got, ref in ((gz, az), (gz0, az0[0]), (gal, aal[0]), (gbe, abe[0])):
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-10)

    def L(a, be):
        x, ld = radial_fwd(*[torch.tensor(_a(v)) for v in (z, z0[None], [a], [be])])
        return float((torch.tensor(g) * x).sum() + (torch.tensor(gam) * ld).sum())
    h = 1e-6
    assert abs((L(alpha + h, beta) - L(alpha - h, beta)) / (2 * h) - gal) <= 1e-5 * (1 + abs(gal))
    assert abs((L(alpha, beta + h) - L(alpha, beta - h)) / (2 * h) - gbe) <= 1e-5 * (1 + abs(gbe))


def test_softplus_overflow_gives_the_reference_values(adjlib):
    """w.u >~ 88.7: log(1 + exp(w.u)) overflows in float32; the constants are the reference's expression's values."""
    u, w = np.array([10.0, 0.0]), np.array([9.5, 0.5])
    _, _, _, _, cst = host_planar(adjlib, "tanh", np.zeros((1, 2)), u, w, 0.0, np.zeros((1, 2)), np.zeros(1),
                                  use_float=1)
    ut, wt = torch.tensor(u, dtype=torch.float32), torch.tensor(w, dtype=torch.float32)
    inner = torch.sum(wt * ut)
    k = (torch.log(1 + torch.exp(inner)) - 1 - inner) / torch.sum(wt ** 2)
    psi = torch.sum(wt * (ut + k * wt))
    for got, ref in zip(cst, (k.item(), psi.item())):
        assert (math.isnan(got) and math.isnan(ref)) or got == ref, (cst, k, psi)
    assert not np.isfinite(cst).all()


def test_saturated_tanh_gives_the_finite_limit(adjlib):
    """|w.z + b| >~ 89: cosh overflows, h' = 0; autograd of 1 / cosh^2 gives NaN, the adjoint the limit (h'' -> 0)."""
    lin = np.array([95.0, -95.0, 200.0, 30.0])
    psi, gu, gam = np.full(4, 0.7), np.full(4, 1.3), np.full(4, 0.9)
    for use_float in (0, 1):
        c, hv, e = np.empty(4), np.empty(4), np.empty(4)
        adjlib.planar_row_check(C.c_int(use_float), C.c_int(0), C.c_double(0.2), C.c_int(4), _P(_a(lin)), _P(_a(psi)),
                                _P(_a(gu)), _P(_a(gam)), _P(c), _P(hv), _P(e))
        assert np.isfinite(c).all() and np.isfinite(e).all()
        np.testing.assert_allclose(hv, np.tanh(lin), rtol=1e-6)
        assert abs(c[0]) < 1e-30 and abs(e[0]) < 1e-30
    t = torch.tensor([95.0], dtype=torch.float32, requires_grad=True)
    (1 / torch.cosh(t) ** 2).sum().backward()
    assert torch.isnan(t.grad).all()   # (why the limit is taken)


def test_leaky_relu_at_zero_uses_one_in_the_log_det_and_the_slope_in_the_map(adjlib):
    lin, psi, gu, gam = _a([0.0]), _a([0.5]), _a([2.0]), _a([3.0])
    c, hv, e = np.empty(1), np.empty(1), np.empty(1)
    adjlib.planar_row_check(C.c_int(0), C.c_int(1), C.c_double(0.2), C.c_int(1), _P(lin), _P(psi), _P(gu), _P(gam),
                            _P(c), _P(hv), _P(e))
    assert hv[0] == 0.0
    assert c[0] == pytest.approx(2.0 * 0.2)            # d leaky(lin) / d lin at 0: the slope (leaky_relu_backward)
    assert e[0] == pytest.approx(3.0 * 1.0 / 1.5)      # h'(0) = 1 in the log-det (planar.py:60)
    # the same through a whole layer, against autograd (z = 0, b = 0: lin = 0 exactly)
    z, u, w, g, gm = np.zeros((3, 2)), np.array([0.4, -0.3]), np.array([0.5, 0.8]), np.ones((3, 2)), np.ones(3)
    got = host_planar(adjlib, "leaky_relu", z, u, w, 0.0, g, gm)
    ref = autograd_planar("leaky_relu", z, u, w, 0.0, g, gm)
    for a, r in zip(got[:4], (ref[0], ref[1][0], ref[2][0], ref[3][0])):
        np.testing.assert_allclose(a, r, rtol=1e-7, atol=1e-7)


def test_radial_at_z0_and_alpha_zero_match_autograd(adjlib):
    z0 = np.array([0.3, -0.2, 0.5])
    z = np.stack([z0, z0 + 0.1, z0 - 0.7])   # row 0: z == z0 exactly
    g, gam = np.ones((3, 3)), np.array([0.5, -1.0, 2.0])
    for alpha in (0.6, 0.0):   # (z = z0 with alpha = 0 divides by zero in the reference as well: rows 1, 2 only)
        if alpha == 0.0:
            z, g, gam = z[1:], g[1:], gam[1:]
        got = host_radial(adjlib, z, z0, alpha, 0.2, g, gam)
        az, az0, aal, abe = autograd_radial(z, z0, alpha, 0.2, g, gam)
        assert np.isfinite(got[0]).all()
        for a, r in zip(got[:4], (az, az0[0], abe[0], aal[0])):
            np.testing.assert_allclose(a, r, rtol=1e-12, atol=1e-12)
        if alpha == 0.0:
            assert got[3] == 0.0


# ---- modules against the reference -----------------------------------------------------------------------------------
GOLDEN = ["r", "s", "t", "u", "v"]


def load_golden(name):
    from helpers import load_npz_parts
    return load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_rkl_{name}.npz"))


@pytest.mark.parametrize("name", GOLDEN)
def test_seeded_construction_matches_the_reference_and_loads_strictly(name):
    import helpers_planar_rkl as H
    import normflows as nf
    gd = load_golden(name)
    model = H.build(nf, name)
    sd = model.state_dict()
    init = {k[6:]: v for k, v in gd.items() if k.startswith("init__")}
    assert list(sd) == list(init)
    for k, v in sd.items():
        assert tuple(v.shape) == init[k].shape and v.dtype == torch.as_tensor(init[k]).dtype, k
        np.testing.assert_array_equal(v.numpy(), init[k], err_msg=k)
    fresh = H.build(nf, name)
    fresh.load_state_dict({k[4:]: torch.as_tensor(v) for k, v in gd.items() if k.startswith("sd__")}, strict=True)


def test_module_attributes_follow_the_reference():
    import normflows as nf
    p = nf.flows.Planar((3,), act="leaky_relu")
    assert [n for n, _ in p.named_parameters()] == ["u", "w", "b"]
    assert [n for n, _ in p.named_modules()] == ["", "h"] and p.h.negative_slope == 0.2
    assert nf.flows.Planar((3,)).h is torch.tanh
    r = nf.flows.Radial((4,))
    assert [n for n, _ in r.named_parameters()] == ["beta", "alpha", "z_0"]
    assert r.d.dim() == 0 and r.d.dtype == torch.int64 and int(r.d) == 4
    with pytest.raises(NotImplementedError, match="Nonlinearity"):
        nf.flows.Planar((2,), act="relu")


def test_targets_match_the_reference_values():
    import helpers_planar_rkl as H
    import normflows as nf
    gd = load_golden("s")
    eps = torch.tensor(gd["eps"]).double()
    for name, t in H.notebook_targets(nf).items():
        np.testing.assert_allclose(t.log_prob(eps).numpy(), gd["p_log_prob__" + name], rtol=1e-12, atol=1e-12)
    # batches of any shape: the last axis holds the coordinates
    t = nf.distributions.Sinusoidal_gap(0.4, 4)
    np.testing.assert_array_equal(t.log_prob(eps[:12].reshape(3, 4, 2)).T.numpy(),
                                  t.log_prob(eps[:12]).reshape(3, 4).T.numpy())


def restated_loss(name, model, eps, x=None):
    """The cases' losses in fp64 torch: the sampling direction by sample_restated, the density direction (t, u) by
    `_autograd.layer_inverse`, the base by its reparameterised formula."""
    import helpers_planar_rkl as H
    from normflows._autograd import layer_inverse
    P = {id(p): p for p in model.parameters()}
    q0 = model.q0

    def base_lp(z):
        ls = q0.log_scale.reshape(-1)
        return -0.5 * z.shape[1] * math.log(2 * math.pi) - ls.sum() - 0.5 * (((z - q0.loc) / torch.exp(ls)) ** 2).sum(1)

    def density(z):
        lq = torch.zeros(z.shape[0], dtype=z.dtype)
        for f in reversed(model.flows):
            z, ld = layer_inverse(f, z)
            lq = lq + ld
        return lq + base_lp(z)
    if name == "u":
        return -torch.mean(density(x))
    z, log_q = H.replay_forward(q0, eps)(eps.shape[0])
    z, ld = sample_restated(model.flows, z, P)
    log_q = log_q - ld
    if name == "t":
        for p in model.parameters():
            p.requires_grad_(False)
        log_q = density(z)
        for p in model.parameters():
            p.requires_grad_(True)
    return torch.mean(log_q) - (0.5 if name == "r" else 1.0) * torch.mean(model.p.log_prob(z))


def golden_model(name):
    import helpers_planar_rkl as H
    import normflows as nf
    gd = load_golden(name)
    model = H.build(nf, name)
    model.load_state_dict({k[4:]: torch.as_tensor(v) for k, v in gd.items() if k.startswith("sd__")})
    return model, torch.tensor(gd["eps"]), (torch.tensor(gd["x"]) if "x" in gd else None), gd


def check_golden(got, gd, name, tol):
    from test_maf_training import check_golden as check
    check(got, gd, name, tol)


@pytest.mark.parametrize("name", GOLDEN)
def test_fp64_restatement_matches_reference_goldens(name):
    model, eps, x, gd = golden_model(name)
    model = model.double()
    loss = restated_loss(name, model, eps.double(), x.double() if x is not None else None)
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    for n, p in model.named_parameters():
        check_golden(p.grad, gd, n, 1e-10)


def test_not_implemented_cases():
    import normflows as nf
    msg = "This flow has no algebraic inverse."
    for f in (nf.flows.Planar((2,)), nf.flows.Radial((2,))):
        with pytest.raises(NotImplementedError, match=msg):
            f.inverse(torch.zeros(3, 2))
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), [nf.flows.Planar((2,), act="leaky_relu"),
                                                                  nf.flows.Radial((2,))])
    for call in (model.log_prob, model.forward_kld, model.inverse):
        with pytest.raises(NotImplementedError, match=msg):
            call(torch.zeros(3, 2))
    with pytest.raises(RuntimeError, match="no CPU/eager fallback"):
        nf.flows.Planar((2,))(torch.zeros(3, 2))


@pytest.mark.gpu
def test_unsupported_shapes_raise_naming_the_limit():
    import normflows as nf
    with pytest.raises(NotImplementedError, match="at most 64 features"):
        nf.flows.Planar((65,)).cuda()(torch.zeros(3, 65, device="cuda"))
    with pytest.raises(NotImplementedError, match="at most 64 features"):
        nf.flows.Radial((80,)).cuda()(torch.zeros(3, 80, device="cuda"))
    with pytest.raises(NotImplementedError, match="image-shaped"):
        nf.flows.Planar((1, 2, 2)).cuda()(torch.zeros(3, 4, device="cuda"))


# ---- GPU: the stack against fp64 autograd of the restatement -----------------------------------------------------------
def make_stack(D, K, seed, kinds=("tanh", "leaky_relu", "radial")):
    import normflows as nf
    torch.manual_seed(seed)
    flows = []
    for i in range(K):
        k = kinds[i % len(kinds)]
        flows.append(nf.flows.Radial((D,)) if k == "radial" else nf.flows.Planar((D,), act=k))
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():   # off the init, tame enough that a deep stack stays finite in float32
        for f in flows:
            for n, p in f.named_parameters():
                if n in ("u", "w"):
                    p.copy_(torch.randn(p.shape, generator=g) * 0.6 / math.sqrt(D))
                elif n == "z_0":
                    p.copy_(torch.randn(p.shape, generator=g) * 0.5)
                else:
                    p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return flows


def _close(got, ref, name, tol=2e-3):
    from test_affine_rkl_training import _close as close
    close(got, ref, name, tol)


def check_stack_gradients(flows, D, rows, seed, layer_loop=False):
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows).cuda()
    g = torch.Generator().manual_seed(seed)
    z0 = torch.randn(rows, D, generator=g).cuda()
    gx = torch.randn(rows, D, generator=g).cuda()
    gld = torch.randn(rows, generator=g).cuda()
    z = z0.clone().requires_grad_(True)
    if layer_loop:
        x, ld = z, torch.zeros(rows, device="cuda")
        for f in model.flows:
            x, l = f(x)
            ld = ld + l
    else:
        x, ld = model.forward_and_log_det(z)
    ((x * gx).sum() + (ld * gld).sum()).backward()
    P = {id(p): p.detach().double().requires_grad_(True) for p in model.flows.parameters()}
    zd = z0.double().requires_grad_(True)
    xr, ldr = sample_restated(model.flows, zd, P)
    ((xr * gx.double()).sum() + (ldr * gld.double()).sum()).backward()
    _close(x.detach(), xr.detach(), "x", 1e-4)
    _close(ld.detach(), ldr.detach(), "log_det", 1e-4)
    _close(z.grad, zd.grad, "g_z")
    for n, p in model.flows.named_parameters():
        assert p.grad is not None, n
        _close(p.grad, P[id(p)].grad, n)
    return model


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,rows", [(1, 6, 129), (2, 12, 127), (2, 32, 5000), (5, 9, 1), (40, 20, 1000),
                                      (64, 12, 129), (64, 3, 5000)])
def test_stack_sampling_backward_matches_fp64_autograd(D, K, rows):
    check_stack_gradients(make_stack(D, K, seed=D + K), D, rows, seed=rows)


@pytest.mark.gpu
@pytest.mark.parametrize("kinds", [("tanh",), ("leaky_relu",), ("radial",)])
def test_single_kind_stacks_match_fp64_autograd(kinds):
    check_stack_gradients(make_stack(5, 8, seed=3, kinds=kinds), 5, 333, seed=4)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 40])
def test_layer_loop_sampling_backward_matches_fp64_autograd(D):
    check_stack_gradients(make_stack(D, 6, seed=7), D, 300, seed=3, layer_loop=True)


@pytest.mark.gpu
def test_rows_beyond_one_workspace_chunk():
    """D = 64, 64 layers: about 25 KB of workspace per row, so 25 000 rows need three chunks."""
    model = check_stack_gradients(make_stack(64, 64, seed=11), 64, 25000, seed=5)
    assert model._stack().launch_count() == 3 * 3 + 1


@pytest.mark.gpu
def test_values_bit_identical_with_and_without_grad_and_reproducible_gradients():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 9, seed=4)).cuda()
    z = torch.randn(777, 5, device="cuda")
    with torch.no_grad():
        x0, l0 = model.forward_and_log_det(z)
    grads = []
    for _ in range(2):
        model.zero_grad()
        x, ld = model.forward_and_log_det(z.clone().requires_grad_(True))
        assert torch.equal(x, x0) and torch.equal(ld, l0)
        (x.square().sum() + ld.sum()).backward()
        grads.append([p.grad.clone() for p in model.flows.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    layer = model.flows[2]
    with torch.no_grad():
        y0, m0 = layer(z)
    y, m = layer(z.clone().requires_grad_(True))
    assert torch.equal(y, y0) and torch.equal(m, m0)


@pytest.mark.gpu
def test_softplus_overflow_values_match_the_reference_expression_on_the_gpu():
    import normflows as nf
    f = nf.flows.Planar((2,), u=torch.tensor([[10.0, 0.0]]), w=torch.tensor([[9.5, 0.5]])).cuda()
    z = torch.randn(16, 2, device="cuda")
    with torch.no_grad():
        x, ld = f(z)
        xr, ldr = planar_fwd(z, f.u, f.w, f.b, "tanh")
    for a, r in ((x, xr), (ld, ldr)):
        assert torch.equal(torch.isnan(a), torch.isnan(r)) and torch.equal(torch.isinf(a), torch.isinf(r))


@pytest.mark.gpu
def test_in_place_change_zero_rows_and_shared_parameters():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 6, seed=2)).cuda()
    x, ld = model.forward_and_log_det(torch.randn(64, 5, device="cuda"))
    with torch.no_grad():
        model.flows[0].u.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        (x.sum() + ld.sum()).backward()
    model.zero_grad()
    x, ld = model.forward_and_log_det(torch.zeros(0, 5, device="cuda", requires_grad=True))
    (x.sum() + ld.sum()).backward()
    for n, p in model.flows.named_parameters():
        assert p.grad is not None and (p.grad == 0).all(), n
    p, r = make_stack(3, 2, seed=9, kinds=("tanh", "radial"))
    check_stack_gradients([p, r, p, r], 3, 300, seed=10)


@pytest.mark.gpu
def test_launch_counts():
    import normflows as nf
    counts = []
    for K in (4, 64):
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), make_stack(2, K, seed=K)).cuda()
        with torch.no_grad():
            model.forward_and_log_det(torch.randn(100, 2, device="cuda"))
        assert model._stack().launch_count() == 1
        x, ld = model.forward_and_log_det(torch.randn(100, 2, device="cuda"))
        (x.sum() + ld.sum()).backward()
        counts.append(model._stack().launch_count())
    assert counts[0] == counts[1] == 4, counts


@pytest.mark.gpu
def test_mixed_planar_and_affine_stacks_still_raise():
    import normflows as nf
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    target = nf.distributions.TwoModes(2, 0.1)
    for flows in ([nf.flows.Planar((2,)), nf.flows.MaskedAffineFlow(torch.tensor([1., 0.]), nf.nets.MLP([2, 4, 2]))],
                  [nf.flows.Radial((2,)), nf.flows.ActNorm(2)]):
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, target).cuda()
        with pytest.raises(NotImplementedError, match=msg):
            model.reverse_kld(64)


@pytest.mark.gpu
def test_leaky_planar_density_direction_matches_the_restatement():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 6, seed=5, kinds=("leaky_relu",))).cuda()
    x = torch.randn(500, 5, device="cuda")
    with torch.no_grad():
        z, ld = model.inverse_and_log_det(x)
    assert model._stack().launch_count() == 1
    from normflows._autograd import layer_inverse
    zr, ldr = x.double(), torch.zeros(500, dtype=torch.float64, device="cuda")
    for f in reversed(model.flows):
        zr, l = layer_inverse(f.double(), zr)
        ldr = ldr + l
    model.float()
    _close(z, zr, "z", 1e-4)
    _close(ld, ldr, "log_det", 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN)
def test_model_gradients_match_reference_goldens(name):
    import helpers_planar_rkl as H
    model, eps, x, gd = golden_model(name)
    model = model.cuda()
    model.q0.forward = H.replay_forward(model.q0, eps.cuda())
    loss = H.loss_of(name, model, eps.shape[0], x.cuda() if x is not None else None)
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    for n, p in model.named_parameters():
        assert p.grad is not None, n
        check_golden(p.grad, gd, n, 2e-3)


# ---- GPU: the notebooks' training cells --------------------------------------------------------------------------------
def _fixed_kl(nfm, beta=1.0):
    """E[log q - beta log p] over a fixed seeded 8 192-sample draw: the reverse KL (beta = 1), or the annealed objective
    the notebooks' training cells minimise at inverse temperature beta."""
    with torch.no_grad():
        torch.manual_seed(123)
        z, log_q = nfm.sample(8192)
        return (log_q - beta * nfm.p.log_prob(z)).mean().item()


def _train(nfm, loss_fn, max_iter, lr, wd):
    """The notebooks' loop: Adam, skip non-finite losses."""
    optimizer = torch.optim.Adam(nfm.parameters(), lr=lr, weight_decay=wd)
    for it in range(max_iter):
        optimizer.zero_grad()
        loss = loss_fn(it)
        if ~(torch.isnan(loss) | torch.isinf(loss)):
            loss.backward()
            optimizer.step()
    for n, p in nfm.named_parameters():
        assert torch.isfinite(p).all(), n
    with torch.no_grad():
        z, log_q = nfm.sample(2 ** 20)
    assert torch.isfinite(z).all()


@pytest.mark.gpu
def test_planar_notebook_trains():
    import normflows as nf
    torch.manual_seed(0)
    nfm = nf.NormalizingFlow(q0=nf.distributions.DiagGaussian(2), flows=[nf.flows.Planar((2,)) for _ in range(16)],
                             p=nf.distributions.TwoModes(2, 0.1)).cuda()
    before = _fixed_kl(nfm)
    _train(nfm, lambda it: nfm.reverse_kld(2 * 20, beta=np.min([1., 0.01 + it / 10000])), 400, 1e-3, 1e-4)
    assert _fixed_kl(nfm) < before


@pytest.mark.gpu
@pytest.mark.parametrize("flow", ["Planar", "Radial"])
def test_comparison_notebook_trains(flow):
    import normflows as nf
    priors = [nf.distributions.TwoModes(2.0, 0.2), nf.distributions.Sinusoidal(0.4, 4),
              nf.distributions.Sinusoidal_gap(0.4, 4), nf.distributions.Sinusoidal_split(0.4, 4),
              nf.distributions.Smiley(0.15)]
    for K in (2, 8, 32):
        for k, prior in enumerate(priors):
            torch.manual_seed(K + k)
            anneal_iter = 10000 if k in (0, 4) else 1
            flows = [nf.flows.Planar((2,)) if flow == "Planar" else nf.flows.Radial((2,)) for _ in range(K)]
            nfm = nf.NormalizingFlow(p=prior, q0=nf.distributions.DiagGaussian(2), flows=flows).cuda()
            n_iter = 150
            beta = float(np.min([1.0, 0.01 + (n_iter - 1) / anneal_iter]))   # (annealed targets: beta ends near 0.025)
            before = _fixed_kl(nfm, beta)
            _train(nfm, lambda it: nfm.reverse_kld(1024, np.min([1.0, 0.01 + it / anneal_iter])), n_iter, 1e-3, 1e-3)
            assert _fixed_kl(nfm, beta) < before, (flow, K, k)
