"""Stochastic normalizing flows and HAIS (reference flows/stochastic.py, distributions/mh_proposal.py,
distributions/linear_interpolation.py, sampling/hais.py): HamiltonianMonteCarlo / MetropolisHastings on native
densities through csrc/nfb_stochastic.cu, with their native backward, and HAIS as one chain launch.

CPU: the reference's state_dict keys; the fp64 restatement (tests/helpers_stochastic.py: the kernels' forward and the
closed-form backward) against the goldens of tests/golden/make_stochastic_grads.py to 1e-10; the host-compiled density
element against central differences.
GPU: every native path against the goldens at 2e-3 of each tensor's scale; native against the generic (reference)
path on the same replayed draws over D, K, leapfrog steps and rows, NaN and overflowing targets included; values
bit-identical with and without grad; seeded runs bit-identical; an in-place change after the forward raises;
invariance of a mixture under 50 HMC transitions; HAIS log Z on a normalised target; a short SNF reverse-KL loop."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import helpers_stochastic as H
from conftest import ROOT, GOLDEN


def golden(name):
    f = np.load(os.path.join(GOLDEN, f"stochastic_{name}.npz"))
    return {k: f[k] for k in f.files}


def gm_terms(g):
    return [(1.0, g["loc"], g["log_scale"], g["weight_scores"])]


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_state_dict_keys_match_reference():
    import normflows as nf
    g = golden("hmc_a")
    gm = nf.distributions.GaussianMixture(3, 4)
    layer = nf.flows.HamiltonianMonteCarlo(gm, 5, torch.zeros(4), torch.zeros(4))
    assert sorted(layer.state_dict().keys()) == list(g["sd_keys"])
    m = golden("mh")
    mh = nf.flows.MetropolisHastings(nf.distributions.DiagGaussian(4), nf.distributions.DiagGaussianProposal((4,), 0.6),
                                     5)
    assert sorted(mh.state_dict().keys()) == list(m["sd_keys"])
    assert np.array_equal(mh.state_dict()["proposal.scale"].numpy(), m["sd_scale"].astype(np.float32))
    sd = {k: torch.tensor(v) for k, v in golden("snf").items() if k.startswith("sd__")}
    model = snf_model(nf)
    model.load_state_dict({k[4:]: v for k, v in sd.items()}, strict=True)


@pytest.mark.parametrize("name", ["hmc_a", "hmc_b"])
def test_restatement_hmc_matches_golden(name):
    g = golden(name)
    args = (g["z"], gm_terms(g), int(g["steps"]), g["log_step_size"], g["log_mass"], float(g["max_abs_grad"]),
            g["noise"], g["unif"])
    z_out, ld, _, _ = H.hmc(*args)
    np.testing.assert_allclose(z_out, g["z_out"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(ld, g["log_det"], rtol=0, atol=1e-10)
    gz, gls, glm, gp = H.hmc_grads(*args, g["w_z"], g["w_ld"])
    for got, key in [(gz, "g_z"), (gls, "g_log_step_size"), (glm, "g_log_mass"), (gp[0][0], "g_loc"),
                     (gp[0][1], "g_log_scale"), (gp[0][2], "g_weight_scores")]:
        np.testing.assert_allclose(got, g[key], rtol=1e-10, atol=1e-10, err_msg=key)


def test_restatement_mh_matches_golden():
    g = golden("mh")
    terms = [(1.0, g["loc"][None], g["log_scale"][None], np.zeros(1))]
    z_out, ld, moved = H.mh(g["z"], terms, int(g["steps"]), float(np.float32(g["scale"])), g["noise"], g["unif"])
    np.testing.assert_allclose(z_out, g["z_out"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(ld, g["log_det"], rtol=0, atol=1e-10)
    gz, gzo, gp = H.log_det_grads(g["z"], z_out, moved.astype(float), terms, g["w_ld"])
    np.testing.assert_allclose(g["w_z"] + gzo + gz, g["g_z"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(gp[0][0][0], g["g_loc"], rtol=1e-10, atol=1e-10)
    np.testing.assert_allclose(gp[0][1][0], g["g_log_scale"], rtol=1e-10, atol=1e-10)


def test_restatement_hais_matches_golden():
    g = golden("hais")
    eps = g["eps"]
    D = eps.shape[1]
    lq0 = -0.5 * D * np.log(2 * np.pi) - 0.5 * (eps ** 2).sum(1)
    prior = [(1.0, np.zeros((1, D)), np.zeros((1, D)), np.zeros(1))]
    z, lw, _ = H.hais(eps, -lq0, gm_terms(g), prior, g["betas"], 5, np.full(D, np.log(0.15)), np.zeros(D), g["noise"],
                      g["unif"])
    np.testing.assert_allclose(z, g["samples"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(lw, g["log_w"], rtol=0, atol=1e-10)


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "stochastic_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "stochastic_host_check.cu")])
    return C.CDLL(so)


@pytest.mark.parametrize("K,D", [(1, 1), (3, 4), (8, 16)])
def test_host_density_element_central_differences(hostlib, K, D):
    rng = np.random.default_rng(K * 100 + D)
    f = lambda v: np.ascontiguousarray(v, dtype=np.float64)
    mu, ls, ws = f(rng.normal(0, 1, (K, D))), f(rng.normal(0, 0.3, (K, D))), f(rng.normal(0, 0.5, K))
    z = f(rng.normal(0, 1.5, (7, D)))
    c = 0.7
    P = lambda v: v.ctypes.data_as(C.c_void_p)

    def run(zz):
        lp, g = np.empty(len(zz)), np.empty(zz.shape)
        hostlib.stochastic_grad_check(C.c_int(K), C.c_int(D), C.c_int(len(zz)), C.c_double(c), P(f(zz)), P(mu), P(ls),
                                      P(ws), P(lp), P(g))
        return lp, g
    lp, g = run(z)
    import helpers_mixture as M
    np.testing.assert_allclose(lp, M.log_prob(z, mu, ls, ws), rtol=1e-12, atol=1e-12)
    h = 1e-6
    for d in range(D):
        e = np.zeros(D)
        e[d] = h
        fd = (run(z + e)[0] - run(z - e)[0]) / (2 * h)
        np.testing.assert_allclose(g[:, d], c * fd, rtol=1e-6, atol=1e-7)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def snf_model(nf, D=4):
    gm = nf.distributions.GaussianMixture(3, D)
    flows = []
    for i in range(2):
        b = torch.tensor([(j + i) % 2 for j in range(D)], dtype=torch.float32)
        flows += [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([D, 16, D], init_zeros=True),
                                            nf.nets.MLP([D, 16, D], init_zeros=True)),
                  nf.flows.ActNorm(D),
                  nf.flows.HamiltonianMonteCarlo(gm, 3, torch.full((D,), float(np.log(0.1))), torch.zeros(D))]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows, p=gm)


def close(got, want, tol=2e-3, what=""):
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got)
    scale = max(np.abs(want).max(), 1e-12)
    err = np.abs(got.reshape(want.shape) - want).max() / scale
    assert err <= tol, f"{what}: {err:.3e}"


def cuda(a, grad=False):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda", requires_grad=grad)


def gm_module(nf, g):
    K, D = g["loc"].shape
    gm = nf.distributions.GaussianMixture(K, D).cuda()
    with torch.no_grad():
        gm.loc.copy_(cuda(g["loc"])[None])
        gm.log_scale.copy_(cuda(g["log_scale"])[None])
        gm.weight_scores.copy_(cuda(g["weight_scores"])[None])
    return gm


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["hmc_a", "hmc_b"])
def test_hmc_native_matches_golden(name):
    import normflows as nf
    g = golden(name)
    gm = gm_module(nf, g)
    mag = float(g["max_abs_grad"]) or None
    layer = nf.flows.HamiltonianMonteCarlo(gm, int(g["steps"]), cuda(g["log_step_size"]), cuda(g["log_mass"]),
                                           max_abs_grad=mag).cuda()
    z = cuda(g["z"], grad=True)
    with torch.enable_grad(), H.Replay([g["noise"][None], g["unif"][None]]):
        z_out, ld = layer(z)
        loss = (cuda(g["w_z"]) * z_out).sum() + (cuda(g["w_ld"]) * ld).sum()
    assert "HmcFn" in type(z_out.grad_fn).__name__
    with torch.enable_grad():
        loss.backward()
    close(z_out, g["z_out"], what="z_out")
    close(ld, g["log_det"], what="log_det")
    for t, key in [(z.grad, "g_z"), (layer.log_step_size.grad, "g_log_step_size"), (layer.log_mass.grad, "g_log_mass"),
                   (gm.loc.grad, "g_loc"), (gm.log_scale.grad, "g_log_scale"),
                   (gm.weight_scores.grad, "g_weight_scores")]:
        close(t, g[key], what=key)


@pytest.mark.gpu
def test_mh_native_matches_golden():
    import normflows as nf
    g = golden("mh")
    dg = nf.distributions.DiagGaussian(4).cuda()
    with torch.no_grad():
        dg.loc.copy_(cuda(g["loc"])[None])
        dg.log_scale.copy_(cuda(g["log_scale"])[None])
    layer = nf.flows.MetropolisHastings(dg, nf.distributions.DiagGaussianProposal((4,), 0.6), int(g["steps"])).cuda()
    z = cuda(g["z"], grad=True)
    with torch.enable_grad(), H.Replay([g["noise"], g["unif"]]):
        z_out, ld = layer(z)
        loss = (cuda(g["w_z"]) * z_out).sum() + (cuda(g["w_ld"]) * ld).sum()
    assert "MhFn" in type(z_out.grad_fn).__name__
    with torch.enable_grad():
        loss.backward()
    close(z_out, g["z_out"], what="z_out")
    close(ld, g["log_det"], what="log_det")
    close(z.grad, g["g_z"], what="g_z")
    close(dg.loc.grad, g["g_loc"], what="g_loc")
    close(dg.log_scale.grad, g["g_log_scale"], what="g_log_scale")


def hais_of(nf, g, prior=None):
    D = g["eps"].shape[1]
    gm = gm_module(nf, g)
    prior = prior or nf.distributions.DiagGaussian(D, trainable=False).cuda()
    return nf.HAIS(torch.tensor(g["betas"], dtype=torch.float32), prior, gm, 5, torch.full((D,), 0.15, device="cuda"),
                   torch.zeros(D, device="cuda"))


def hais_draws(g):
    return [g["eps"], g["noise"], g["unif"]]


@pytest.mark.gpu
def test_hais_chain_matches_golden_in_one_launch():
    import normflows as nf
    from normflows import _stochastic as S
    g = golden("hais")
    h = hais_of(nf, g)
    calls = []
    orig = S.hmc_launch
    S.hmc_launch = lambda *a: calls.append(1) or orig(*a)
    try:
        with H.Replay(hais_draws(g)):
            z, lw = h.sample(len(g["eps"]))
    finally:
        S.hmc_launch = orig
    assert len(calls) == 1
    close(z, g["samples"], what="samples")
    close(lw, g["log_w"], what="log_w")
    # under grad HAIS walks the layers on the same draws: the same bits
    with torch.enable_grad(), H.Replay(hais_draws(g)):
        z2, lw2 = h.sample(len(g["eps"]))
    assert torch.equal(z, z2.detach()) and torch.equal(lw, lw2.detach())


@pytest.mark.gpu
def test_snf_reverse_kld_matches_golden():
    import normflows as nf
    g = golden("snf")
    model = snf_model(nf).cuda()
    model.load_state_dict({k[4:]: torch.tensor(v) for k, v in g.items() if k.startswith("sd__")}, strict=True)
    assert model._takes_layer_loop()
    with torch.enable_grad(), H.Replay([g["eps"], g["n0"][None], g["u0"][None], g["n1"][None], g["u1"][None]]):
        loss = model.reverse_kld(len(g["eps"]))
        loss.backward()
    close(loss, g["loss"], what="loss")
    for k, p in model.named_parameters():
        close(p.grad, g["g__" + k], what=k)


def generic_target(gm):
    """The same density as a non-native Target: forces the generic (reference) path."""
    class T:
        def log_prob(self, z):
            return gm.log_prob(z)
    return T()


CASES = [(D, K, steps, rows) for D in (1, 2, 5, 16, 64) for K in (1, 8) for steps in (0, 1, 10) for rows in (1, 1061)]
CASES += [(5, 8, 10, 0), (2, 1, 1, 65536), (64, 8, 10, 65536)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,steps,rows", CASES)
def test_hmc_native_matches_generic(D, K, steps, rows):
    import normflows as nf
    torch.manual_seed(D * 1000 + K * 10 + steps)
    gm = nf.distributions.GaussianMixture(K, D, loc=np.random.default_rng(D + K).normal(0, 1, (K, D))).cuda()
    ls, lm = torch.full((D,), float(np.log(0.3 / np.sqrt(D)))).cuda(), (0.1 * torch.randn(D)).cuda()
    native = nf.flows.HamiltonianMonteCarlo(gm, steps, ls.clone(), lm.clone(), max_abs_grad=3.0).cuda()
    generic = nf.flows.HamiltonianMonteCarlo(generic_target(gm), steps, ls.clone(), lm.clone(), max_abs_grad=3.0).cuda()
    z = 1.5 * torch.randn(rows, D, device="cuda")
    noise, unif = torch.randn(1, rows, D, device="cuda"), torch.rand(1, rows, device="cuda")
    with H.Replay([noise, unif]):
        za, la = native(z)
    with H.Replay([noise, unif]):
        zb, lb = generic(z)
    assert za.shape == (rows, D) and la.shape == (rows,)
    if rows:
        same = (za == zb).all(1) | ((za - zb).abs().max(1).values < 1e-3)
        assert same.float().mean() > 0.995          # rows at an accept margin may decide differently in float32
        ok = same & torch.isfinite(lb)
        assert torch.allclose(la[ok], lb[ok], rtol=1e-3, atol=1e-3 * max(1.0, float(lb[ok].abs().max())))


@pytest.mark.gpu
@pytest.mark.parametrize("D,K,steps,rows", [(1, 1, 0, 1), (2, 8, 1, 1061), (5, 1, 10, 1061), (64, 8, 10, 1061),
                                            (16, 8, 1, 65536)])
def test_mh_native_matches_generic(D, K, steps, rows):
    import normflows as nf
    torch.manual_seed(7 * D + K + steps)
    gm = nf.distributions.GaussianMixture(K, D).cuda()
    prop = nf.distributions.DiagGaussianProposal((D,), 0.4)
    native = nf.flows.MetropolisHastings(gm, prop, steps).cuda()
    generic = nf.flows.MetropolisHastings(generic_target(gm), prop, steps).cuda()
    z = torch.randn(rows, D, device="cuda")
    noise, unif = torch.randn(steps, rows, D, device="cuda"), torch.rand(steps, rows, device="cuda")
    with H.Replay([noise, unif]):
        za, la = native(z)
    with H.Replay([noise, unif]):
        zb, lb = generic(z)
    same = (za - zb).abs().max(1).values < 1e-4
    assert same.float().mean() > 0.995
    assert torch.allclose(la[same], lb[same], rtol=1e-3, atol=1e-3)


@pytest.mark.gpu
def test_nan_and_overflowing_targets():
    import normflows as nf
    D = 3
    gm = nf.distributions.GaussianMixture(2, D).cuda()
    with torch.no_grad():
        gm.loc[0, 0, 0] = float("nan")       # every row's log p is NaN: every move rejected, log_det NaN
    layer = nf.flows.HamiltonianMonteCarlo(gm, 2, torch.full((D,), -1.0), torch.zeros(D)).cuda()
    z = torch.randn(64, D, device="cuda")
    z_out, ld = layer(z)
    assert torch.equal(z_out, z) and torch.isnan(ld).all()
    # an exponent that overflows exp accepts: start far out in the tail, where log p(z') - log p(z) is huge
    gm2 = nf.distributions.GaussianMixture(1, D, loc=np.zeros((1, D)), scale=np.full((1, D), 1e-3)).cuda()
    layer2 = nf.flows.HamiltonianMonteCarlo(gm2, 1, torch.full((D,), float(np.log(1e-3))), torch.zeros(D)).cuda()
    z = torch.full((64, D), 0.5, device="cuda")
    generic = nf.flows.HamiltonianMonteCarlo(generic_target(gm2), 1, torch.full((D,), float(np.log(1e-3))),
                                             torch.zeros(D)).cuda()
    noise, unif = torch.randn(1, 64, D, device="cuda"), torch.rand(1, 64, device="cuda")
    with H.Replay([noise, unif]):
        za, la = layer2(z)
    with H.Replay([noise, unif]):
        zb, lb = generic(z)
    assert torch.equal(torch.isfinite(la), torch.isfinite(lb))
    assert ((za != z).any(1) == (zb != z).any(1)).all()


@pytest.mark.gpu
def test_bit_identical_with_without_grad_and_seeded():
    import normflows as nf
    torch.manual_seed(0)
    gm = nf.distributions.GaussianMixture(4, 5).cuda()
    layer = nf.flows.HamiltonianMonteCarlo(gm, 4, torch.full((5,), -1.5), torch.zeros(5)).cuda()
    z = torch.randn(3000, 5, device="cuda")
    torch.manual_seed(1)
    a = layer(z)
    torch.manual_seed(1)
    with torch.enable_grad():
        b = layer(z.clone().requires_grad_())
    torch.manual_seed(1)
    c = layer(z)
    for x, y, w in zip(a, b, c):
        assert torch.equal(x, y.detach()) and torch.equal(x, w)
    # the backward: two calls give identical bits
    grads = []
    for _ in range(2):
        layer.zero_grad()
        torch.manual_seed(2)
        with torch.enable_grad():
            zo, ld = layer(z)
            (zo.square().sum() + ld.sum()).backward()
        grads.append([p.grad.clone() for p in layer.parameters()])
    assert all(torch.equal(x, y) for x, y in zip(*grads))


@pytest.mark.gpu
def test_inplace_change_after_forward_raises():
    import normflows as nf
    gm = nf.distributions.GaussianMixture(2, 3).cuda()
    layer = nf.flows.HamiltonianMonteCarlo(gm, 2, torch.full((3,), -1.0), torch.zeros(3)).cuda()
    with torch.enable_grad():
        zo, ld = layer(torch.randn(32, 3, device="cuda"))
        with torch.no_grad():
            layer.log_mass.add_(0.1)
        with pytest.raises(RuntimeError, match="modified in place"):
            (zo.sum() + ld.sum()).backward()


@pytest.mark.gpu
def test_hmc_keeps_mixture_moments():
    import normflows as nf
    torch.manual_seed(3)
    gm = nf.distributions.GaussianMixture(3, 2, loc=[[-1.0, 0.0], [1.0, 0.5], [0.0, -1.0]],
                                          scale=[[0.6, 0.6], [0.5, 0.8], [0.7, 0.4]], weights=[0.3, 0.3, 0.4]).cuda()
    layer = nf.flows.HamiltonianMonteCarlo(gm, 5, torch.full((2,), float(np.log(0.2))), torch.zeros(2)).cuda()
    z0 = gm.sample(1 << 16)
    z = z0
    for _ in range(50):
        z, _ = layer(z)
    # two independent exact samples of 2^16 rows differ in mean by ~0.01 and in second moments by ~0.02 (4 sigma)
    assert (z.mean(0) - z0.mean(0)).abs().max() < 0.03
    assert (torch.cov(z.T) - torch.cov(z0.T)).abs().max() < 0.05


@pytest.mark.gpu
def test_hais_log_z_of_normalised_target():
    import normflows as nf
    torch.manual_seed(4)
    D = 4
    gm = nf.distributions.GaussianMixture(3, D, loc=np.random.default_rng(0).normal(0, 1.5, (3, D))).cuda()
    prior = nf.distributions.DiagGaussian(D, trainable=False).cuda()
    h = nf.HAIS(torch.linspace(1, 0, 200), prior, gm, 5, torch.full((D,), 0.2, device="cuda"),
                torch.zeros(D, device="cuda"))
    with torch.no_grad():
        _, lw = h.sample(1 << 14)
    log_z = torch.logsumexp(lw.double(), 0) - np.log(len(lw))
    # the target is normalised, so log Z = 0; with 198 transitions the weights' spread is small
    assert abs(float(log_z)) < 0.05, float(log_z)


@pytest.mark.gpu
def test_snf_reverse_kld_training_lowers_the_loss():
    import normflows as nf
    torch.manual_seed(5)
    model = snf_model(nf).cuda()
    with torch.no_grad():
        model.p.loc.copy_(torch.tensor([[[2.0, 0, 0, 0], [-2.0, 0, 0, 0], [0, 2.0, 0, 0]]], device="cuda"))
    for p in model.p.parameters():
        p.requires_grad_(False)
    opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=5e-3)
    losses = []
    with torch.enable_grad():
        for _ in range(60):
            opt.zero_grad()
            loss = model.reverse_kld(2048)
            loss.backward()
            opt.step()
            losses.append(float(loss))
    assert np.mean(losses[-10:]) < np.mean(losses[:10]) - 0.05, (losses[:10], losses[-10:])


def _strided(z, layout):
    """A view of z's values that is not contiguous: the first columns of a wider tensor, or a transposed one; -> (leaf
    to differentiate, the view)."""
    if layout == "slice":
        leaf = torch.cat([z, torch.randn(z.shape[0], 3, device=z.device)], 1).requires_grad_()
        return leaf, leaf[:, :z.shape[1]]
    leaf = z.t().contiguous().requires_grad_()
    return leaf, leaf.t()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["hmc", "mh"])
@pytest.mark.parametrize("layout", ["slice", "transpose"])
def test_strided_z_with_and_without_grad(kind, layout):
    import normflows as nf
    torch.manual_seed(11)
    D, rows = 5, 1061
    gm = nf.distributions.GaussianMixture(4, D).cuda()
    if kind == "hmc":
        layer = nf.flows.HamiltonianMonteCarlo(gm, 4, torch.full((D,), -1.2), 0.1 * torch.randn(D)).cuda()
    else:
        layer = nf.flows.MetropolisHastings(gm, nf.distributions.DiagGaussianProposal((D,), 0.5), 4).cuda()
    z = 1.5 * torch.randn(rows, D, device="cuda")
    w = torch.randn(rows, D, device="cuda")

    def run(zz, grad):
        torch.manual_seed(12)
        with torch.set_grad_enabled(grad):
            return layer(zz)
    ref = run(z, False)
    with torch.enable_grad():   # (the view must record its gradient edge to the leaf)
        leaf, zs = _strided(z, layout)
    assert not zs.is_contiguous()
    for got in (run(zs.detach(), False), run(zs, True)):
        assert torch.equal(got[0].detach(), ref[0]) and torch.equal(got[1].detach(), ref[1])
    # gradients from the strided input equal those from a contiguous copy of it
    zo, ld = run(zs, True)
    with torch.enable_grad():
        ((w * zo).sum() + ld.sum()).backward()
    g_strided = [p.grad.clone() for p in layer.parameters()]
    g_z_strided = leaf.grad[:, :D] if layout == "slice" else leaf.grad.t()
    layer.zero_grad()
    zc = z.clone().requires_grad_()
    zo, ld = run(zc, True)
    with torch.enable_grad():
        ((w * zo).sum() + ld.sum()).backward()
    assert all(torch.equal(a, p.grad) for a, p in zip(g_strided, layer.parameters()))
    assert torch.equal(g_z_strided, zc.grad)
    if layout == "slice":
        assert not leaf.grad[:, D:].any()


@pytest.mark.gpu
def test_generic_path_draws_in_z_dtype():
    import normflows as nf
    from normflows import _stochastic as S
    D = 3
    target = torch.distributions.MultivariateNormal(torch.zeros(D, dtype=torch.float64, device="cuda"),
                                                    torch.eye(D, dtype=torch.float64, device="cuda"))
    dtypes = []
    orig = S.draw

    def spy(*a, **k):
        out = orig(*a, **k)
        dtypes.append((out[0].dtype, out[1].dtype))
        return out
    S.draw = spy
    try:
        z = torch.randn(256, D, dtype=torch.float64, device="cuda")
        zo, ld = nf.flows.HamiltonianMonteCarlo(target, 3, torch.full((D,), -1.0), torch.zeros(D)).cuda()(z)
        zm, lm = nf.flows.MetropolisHastings(target, nf.distributions.DiagGaussianProposal((D,), 0.5), 2).cuda()(z)
    finally:
        S.draw = orig
    assert dtypes == [(torch.float64, torch.float64)] * 2
    assert zo.dtype == ld.dtype == zm.dtype == lm.dtype == torch.float64
    assert (zo != z).any() and (zm != z).any()


@pytest.mark.gpu
def test_trainable_alpha_keeps_the_reference_graph():
    import normflows as nf
    torch.manual_seed(13)
    D = 4
    gm = nf.distributions.GaussianMixture(3, D).cuda()
    dg = nf.distributions.DiagGaussian(D, trainable=False).cuda()
    alpha = torch.tensor(0.4, device="cuda", requires_grad=True)
    layer = nf.flows.HamiltonianMonteCarlo(nf.distributions.LinearInterpolation(gm, dg, alpha), 3,
                                           torch.full((D,), -1.0), torch.zeros(D)).cuda()
    with torch.enable_grad():
        zo, ld = layer(torch.randn(512, D, device="cuda"))
        assert "HmcFn" not in type(ld.grad_fn).__name__
        (zo.sum() + ld.sum()).backward()
    assert alpha.grad is not None and torch.isfinite(alpha.grad) and alpha.grad != 0
    # a plain-number alpha stays native
    layer.target = nf.distributions.LinearInterpolation(gm, dg, 0.4)
    with torch.enable_grad():
        zo, ld = layer(torch.randn(512, D, device="cuda"))
    assert "HmcFn" in type(ld.grad_fn).__name__
