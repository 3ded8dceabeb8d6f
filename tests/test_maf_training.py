"""Training of MaskedAffineAutoregressive (examples/conditional_flow.ipynb's third model): the density pass
y = inverse(x, context) solves y = (x - shift(p)) / scale(p), p = MADE(y, context), with the reference's D-pass loop.
Its gradient is the fixed-point adjoint of that loop (nfb_maf_inverse_backward):

    lam = g_y;  repeat D - 1 times: lam = g_y + MADE_dgrad_y(A(lam));  pbar = A(lam);  g_x = lam / scale
    A(lam): pbar_shift = -lam / scale,  pbar_u = -(sig (1 - sig) / scale) (lam y + g_log_det)

which equals the gradient of the unrolled loop exactly, because MADE's Jacobian in y is strictly lower triangular.

CPU: the element adjoint (csrc/nfb_maf_bwd.cuh), compiled for the host, against fp64 autograd and central differences;
a torch fp64 restatement of the layer and of the fixed-point adjoint pinned to gradients minted from the reference's
autograd (tests/golden/make_maf_grads.py cases f and g).
GPU: the layer against fp64 autograd of the restatement, whole models against the goldens, and the notebook's loop."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- element adjoint on the host -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def adjlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "maf_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "maf_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_adjoint(lib, x, u, s, lam, gld, use_float=0):
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
    x, u, s, lam, gld = (f(a) for a in (x, u, s, lam, gld))
    n = x.size
    gu, gs, gx = np.empty(n), np.empty(n), np.empty(n)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    lib.maf_adjoint_check(n, int(use_float), vp(x), vp(u), vp(s), vp(lam), vp(gld), vp(gu), vp(gs), vp(gx))
    return gu, gs, gx


def ref_element(x, u, s):
    """flows/affine/autoregressive.py:114-122, one element: (y, log_det contribution)."""
    scale = torch.sigmoid(u + 2.0) + 1e-3
    return (x - s) / scale, -torch.log(scale)


def element_cases(rng, n=4000):
    x = rng.normal(size=n) * 2.0
    u = rng.normal(size=n) * 3.0
    s = rng.normal(size=n)
    lam = rng.normal(size=n) * 5.0
    gld = rng.normal(size=n)
    u[:40] = -40.0 - rng.uniform(0, 200, 40)   # scale saturated at 1e-3
    u[40:80] = 40.0 + rng.uniform(0, 200, 40)  # scale saturated at 1 + 1e-3
    u[80:120] = -12.0                          # scale just above 1e-3
    gld[120:200] = 0.0
    return x, u, s, lam, gld


def autograd_element(x, u, s, lam, gld):
    ut, st = torch.tensor(u, requires_grad=True), torch.tensor(s, requires_grad=True)
    xt = torch.tensor(x, requires_grad=True)
    y, ld = ref_element(xt, ut, st)
    ((y * torch.tensor(lam)).sum() + (ld * torch.tensor(gld)).sum()).backward()
    return ut.grad.numpy(), st.grad.numpy(), xt.grad.numpy()


def test_maf_element_adjoint_matches_fp64_autograd(adjlib):
    x, u, s, lam, gld = element_cases(np.random.default_rng(0))
    gu, gs, gx = host_adjoint(adjlib, x, u, s, lam, gld)
    ru, rs, rx = autograd_element(x, u, s, lam, gld)
    for got, ref in ((gu, ru), (gs, rs), (gx, rx)):
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-14 * np.abs(ref).max())
    # saturated scales: no gradient into u (exactly 0, not NaN), shift / x gradients of scale 1e-3 and 1 + 1e-3
    assert np.isfinite(gu).all() and (np.abs(gu[:80]) < 1e-6).all()
    np.testing.assert_allclose(gs[:40], -lam[:40] / 1e-3, rtol=1e-12)
    np.testing.assert_allclose(gx[40:80], lam[40:80] / (1 + 1e-3), rtol=1e-12)
    # the float instantiation (what the kernel runs) agrees to fp32 accuracy
    fu, fs, fx = host_adjoint(adjlib, x, u, s, lam, gld, use_float=1)
    for got, ref in ((fu, ru), (fs, rs), (fx, rx)):
        assert np.isfinite(got).all()
        np.testing.assert_allclose(got, ref, rtol=2e-5, atol=1e-6 * np.abs(ref).max())


def test_maf_element_adjoint_matches_finite_differences(adjlib):
    rng = np.random.default_rng(1)
    x, u, s, lam, gld = element_cases(rng, 600)
    u[:120] = rng.normal(size=120)   # FD needs an unsaturated sigmoid to resolve the u gradient
    gu, gs, gx = host_adjoint(adjlib, x, u, s, lam, gld)
    obj = lambda xx, uu, ss: (lambda r: r[0].numpy() * lam + r[1].numpy() * gld)(
        ref_element(torch.tensor(xx), torch.tensor(uu), torch.tensor(ss)))
    eps = 1e-6
    for got, (dx, du, ds) in ((gx, (eps, 0, 0)), (gu, (0, eps, 0)), (gs, (0, 0, eps))):
        fd = (obj(x + dx, u + du, s + ds) - obj(x - dx, u - du, s - ds)) / (2 * eps)
        np.testing.assert_allclose(got, fd, rtol=1e-5, atol=1e-5)


def test_maf_element_adjoint_propagates_nan(adjlib):
    x = np.array([np.nan, 1.0, 1.0, 1.0, 0.5])
    u = np.array([0.3, np.nan, 0.3, 0.3, 0.3])
    s = np.array([0.1, 0.1, np.nan, 0.1, 0.1])
    lam = np.array([1.0, 1.0, 1.0, np.nan, 1.0])
    gld = np.array([0.5, 0.5, 0.5, 0.5, np.nan])
    for use_float in (0, 1):
        gu, gs, gx = host_adjoint(adjlib, x, u, s, lam, gld, use_float)
        ru, rs, rx = autograd_element(x, u, s, lam, gld)
        for got, ref in ((gu, ru), (gs, rs), (gx, rx)):
            assert (np.isnan(got) == np.isnan(ref)).all(), (got, ref)
            np.testing.assert_allclose(got[~np.isnan(ref)], ref[~np.isnan(ref)], rtol=1e-6)


# ---- torch fp64 restatement of the layer and of the fixed-point adjoint ----------------------------------------------
def made_ref(P, pre, y, context, nb):
    """nets/made.py:217-304 with residual blocks (and the blocks' GLU context gate); P: state-dict names -> tensors."""
    lin = lambda n, v: F.linear(v, P[n + ".weight"] * P[n + ".mask"], P[n + ".bias"])
    h = lin(pre + "initial_layer", y)
    if context is not None:
        h = h + F.linear(context, P[pre + "context_layer.weight"], P[pre + "context_layer.bias"])
    for b in range(nb):
        q = f"{pre}blocks.{b}."
        t = lin(q + "linear_layers.1", torch.relu(lin(q + "linear_layers.0", torch.relu(h))))
        if context is not None:
            t = t * torch.sigmoid(F.linear(context, P[q + "context_layer.weight"], P[q + "context_layer.bias"]))
        h = h + t
    return lin(pre + "final_layer", h)


def maf_element(x, p):
    """flows/affine/autoregressive.py:114-128: (y, log_det) of p = [rows, 2 D] interleaved (u, shift)."""
    u, s = p.view(x.shape[0], x.shape[1], 2).unbind(-1)
    y, ld = ref_element(x, u, s)
    return y, ld.sum(1)


def maf_unrolled(P, pre, nb, x, context):
    """The reference's D-pass loop (flows/affine/autoregressive.py:26-33), differentiated by autograd."""
    y, ld = torch.zeros_like(x), None
    for _ in range(x.shape[1]):
        y, ld = maf_element(x, made_ref(P, pre, y, context, nb))
    return y, ld


class MafFixedPoint(torch.autograd.Function):
    """The D-pass loop under no_grad; backward: the fixed-point adjoint (the algorithm nfb_maf_inverse_backward runs)."""

    @staticmethod
    def forward(ctx, P, pre, nb, names, x, context, *params):
        Q = dict(P, **dict(zip(names, params)))
        with torch.no_grad():
            y, ld = maf_unrolled(Q, pre, nb, x, context)
        ctx.P, ctx.pre, ctx.nb, ctx.names = P, pre, nb, names
        ctx.save_for_backward(x, y, context, *params)
        return y, ld

    @staticmethod
    def backward(ctx, g_y, g_ld):
        x, y, context, *params = ctx.saved_tensors
        D = x.shape[1]
        with torch.enable_grad():
            yv = y.detach().requires_grad_(True)
            cv = context.detach().requires_grad_(True) if context is not None else None
            pv = [p.detach().requires_grad_(True) for p in params]
            p = made_ref(dict(ctx.P, **dict(zip(ctx.names, pv))), ctx.pre, yv, cv, ctx.nb)
            u, s = p.detach().view(-1, D, 2).unbind(-1)
            sig = torch.sigmoid(u + 2.0)
            scale = sig + 1e-3

            def A(lam):
                return torch.stack([-(sig * (1 - sig) / scale) * (lam * y + g_ld[:, None]), -lam / scale], -1).view(p.shape)
            lam = g_y
            for _ in range(D - 1):
                lam = g_y + torch.autograd.grad(p, yv, A(lam), retain_graph=True)[0]
            inputs = ([cv] if cv is not None else []) + pv
            grads = list(torch.autograd.grad(p, inputs, A(lam), allow_unused=True))
        g_ctx = grads.pop(0) if cv is not None else None
        return (None, None, None, None, lam / scale, g_ctx, *grads)


def maf_fixed_point(P, pre, nb, x, context):
    names = [n for n in P if n.startswith(pre) and P[n].requires_grad]
    return MafFixedPoint.apply(P, pre, nb, names, x, context, *[P[n] for n in names])


def lu_inverse_ref(P, pre, z):
    """LULinearPermute in the density direction (flows/mixing.py:402-434,514-563): permute, then x U^T L^T + b."""
    n = z.shape[1]
    perm = P[pre + "permutation._permutation"].long()
    il, iu = torch.tril_indices(n, n, -1), torch.triu_indices(n, n, 1)
    lower = torch.eye(n, dtype=z.dtype).index_put((il[0], il[1]), P[pre + "linear.lower_entries"])
    diag = F.softplus(P[pre + "linear.unconstrained_upper_diag"]) + 1e-3
    upper = torch.diag(diag).index_put((iu[0], iu[1]), P[pre + "linear.upper_entries"])
    x = F.linear(F.linear(z[:, perm], upper), lower, P[pre + "linear.bias"])
    return x, torch.log(diag).sum().expand(z.shape[0])


def model_ref_kld(P, n_layers, nb, x, context, fixed_point):
    """forward_kld of cases f / g: n_layers x [MAF, LULinearPermute] on a DiagGaussian."""
    maf = maf_fixed_point if fixed_point else maf_unrolled
    log_q = torch.zeros(x.shape[0], dtype=x.dtype)
    z = x
    for i in range(2 * n_layers - 1, -1, -1):
        if i % 2:
            z, ld = lu_inverse_ref(P, f"flows.{i}.", z)
        else:
            z, ld = maf(P, f"flows.{i}.autoregressive_net.", nb, z, context)
        log_q = log_q + ld
    loc, ls = P["q0.loc"], P["q0.log_scale"]
    d = z.shape[1]
    log_p = -0.5 * d * math.log(2 * math.pi) - ls.sum() - 0.5 * (((z - loc) / torch.exp(ls)) ** 2).sum(1)
    return -(log_q + log_p).mean()


CASES = {"f": dict(layers=4, blocks=2, trainable_base=False), "g": dict(layers=3, blocks=2, trainable_base=True)}


def load_case(name):
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(GOLDEN, f"grads_cond_{name}.npz"))
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    x = torch.tensor(gd["x"])
    ctx = torch.tensor(gd["context"]) if "context" in gd else None
    return gd, sd, x, ctx


def is_param(name, trainable_base):
    return name.endswith((".weight", ".bias", "_entries", "_upper_diag")) or (trainable_base and name.startswith("q0."))


def check_golden(got, gd, name, tol):
    """A gradient against the golden: whole, or through the seeded projections G v, u G and |G|, each within tol of
    its scale."""
    def close(a, b, what):
        a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double()
        scale = b.abs().max().item() + 1e-300
        err = (a - b).abs().max().item()
        assert err <= tol * scale, f"{what}: max err {err:.3e}, scale {scale:.3e}"
    if "g__" + name in gd:
        close(got, gd["g__" + name], name)
        return
    from helpers_glow_grads import grad_projections
    v, u = grad_projections(name, tuple(got.shape))
    G = got.double().cpu().reshape(got.shape[0], -1)
    close(G @ v, gd["gv__" + name], name + " G v")
    close(u @ G, gd["gu__" + name], name + " u G")
    gn = float(gd["gn__" + name])
    assert abs(G.norm().item() - gn) <= tol * gn, name + " |G|"


@pytest.mark.parametrize("name", ["f", "g"])
def test_fp64_fixed_point_adjoint_matches_reference_goldens(name):
    """The restated algorithm in fp64 gives the reference's unrolled-loop autograd gradients to 1e-10 of each scale."""
    gd, sd, x, ctx = load_case(name)
    cfg = CASES[name]
    P = {k: v.double().requires_grad_(is_param(k, cfg["trainable_base"])) for k, v in sd.items()}
    xd = x.double().requires_grad_(True)
    cd = ctx.double().requires_grad_(True) if ctx is not None else None
    loss = model_ref_kld(P, cfg["layers"], cfg["blocks"], xd, cd, fixed_point=True)
    loss.backward()
    # the reference accumulates log_q in a float32 buffer (core.py forward_kld: torch.zeros(len(x)) += log_det), so its
    # loss carries fp32 rounding; its gradients do not
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * abs(float(gd["loss"]))
    names = [k for k, v in P.items() if v.requires_grad]
    minted = {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))} - {"x", "context"}
    assert minted == set(names), minted ^ set(names)
    for n in names:
        check_golden(P[n].grad, gd, n, 1e-10)
    check_golden(xd.grad, gd, "x", 1e-10)
    if cd is not None:
        check_golden(cd.grad, gd, "context", 1e-10)


# ================================================ GPU ================================================================
def _close(got, ref, name, tol=2e-3):
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = ref.abs().max().item() + 1e-12
    err = (got - ref).abs().max().item()
    assert err <= tol * scale, f"{name}: max err {err:.3e} scale {scale:.3e}"


def _perturb(module, seed, s):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.add_(s * torch.randn(p.shape, generator=g))


def build_package_case(name):
    """Model f / g built by this package with the golden's parameters (and MADE masks / degrees); every other buffer
    must equal the reference's."""
    import normflows as nf
    gd, sd, x, ctx = load_case(name)
    torch.manual_seed(0)
    flows = []
    for _ in range(CASES[name]["layers"]):
        if name == "f":
            flows += [nf.flows.MaskedAffineAutoregressive(2, 128, context_features=4, num_blocks=2),
                      nf.flows.LULinearPermute(2)]
        else:
            flows += [nf.flows.MaskedAffineAutoregressive(8, 64, num_blocks=2), nf.flows.LULinearPermute(8)]
    if name == "f":
        model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows)
    else:
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(8), flows)
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    params = {n for n, _ in model.named_parameters()}
    load = {}
    for k, v in own.items():
        ref = sd[k].to(v.dtype)
        if k in params or k.endswith((".mask", ".degrees", "._permutation")):
            load[k] = ref
        else:
            assert torch.equal(v, ref), f"buffer {k} differs from the reference's"
    model.load_state_dict(load, strict=False)
    return model, x, ctx, gd


def _kld(model, x, ctx):
    return model.forward_kld(x, ctx) if ctx is not None else model.forward_kld(x)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["f", "g"])
def test_model_gradients_match_reference_goldens(name):
    """forward_kld(x[, context]).backward() against the reference's fp64 autograd (make_maf_grads.py f, g)."""
    model, x, ctx, gd = build_package_case(name)
    model = model.cuda()
    xc = x.cuda().requires_grad_(True)
    cc = ctx.cuda().requires_grad_(True) if ctx is not None else None
    loss = _kld(model, xc, cc)
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) < 1e-4 * (1 + abs(float(gd["loss"])))
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None, f"{n} got no gradient"
            check_golden(p.grad, gd, n, 2e-3)
    check_golden(xc.grad, gd, "x", 2e-3)
    if cc is not None:
        check_golden(cc.grad, gd, "context", 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("D,H,nb,context,rows", [
    (1, 32, 0, False, 127), (1, 64, 1, True, 1061), (2, 128, 2, True, 1061), (2, 256, 1, False, 1),
    (5, 64, 2, False, 127), (5, 96, 0, True, 1061), (16, 256, 2, False, 1061), (16, 128, 1, True, 127),
    (16, 32, 2, True, 1), (5, 64, 2, True, 0), (2, 32, 0, False, 0)])
def test_layer_backward_matches_fp64_autograd(D, H, nb, context, rows):
    from normflows.flows import MaskedAffineAutoregressive
    torch.manual_seed(D * 100 + H + nb)
    C_ = 3 if context else None
    layer = MaskedAffineAutoregressive(D, H, context_features=C_, num_blocks=nb)
    _perturb(layer, 7 + D, 0.1)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(rows, D, generator=g)
    ctx = torch.randn(rows, 3, generator=g) if context else None
    gy, gld = torch.randn(rows, D, generator=g), torch.randn(rows, generator=g)
    P = {k: v.double().requires_grad_(k.endswith((".weight", ".bias"))) for k, v in layer.state_dict().items()}
    xr = x.double().requires_grad_(True)
    cr = ctx.double().requires_grad_(True) if context else None
    yr, ldr = maf_unrolled(P, "autoregressive_net.", nb, xr, cr)
    ((yr * gy.double()).sum() + (ldr * gld.double()).sum()).backward()
    layer = layer.cuda()
    xc = x.cuda().requires_grad_(True)
    cc = ctx.cuda().requires_grad_(True) if context else None
    y, ld = layer.inverse(xc, cc)
    assert y.requires_grad and ld.requires_grad
    ((y * gy.cuda()).sum() + (ld * gld.cuda()).sum()).backward()
    assert y.shape == (rows, D) and ld.shape == (rows,)
    if rows:
        _close(y.detach(), yr.detach(), "y", 1e-4)
        _close(ld.detach(), ldr.detach(), "log_det", 1e-4)
    for n, p in layer.named_parameters():
        assert p.grad is not None, n
        if rows == 0:
            assert (p.grad == 0).all(), n
        else:
            _close(p.grad, P[n].grad, n)
    if rows:
        _close(xc.grad, xr.grad, "x")
        if context:
            _close(cc.grad, cr.grad, "context")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["f", "g"])
def test_values_bit_identical_with_and_without_grad(name):
    model, x, ctx, _ = build_package_case(name)
    model = model.cuda()
    args = (x.cuda(),) + ((ctx.cuda(),) if ctx is not None else ())
    with torch.no_grad():
        a = model.log_prob(*args)
    b = model.log_prob(*args)
    assert b.requires_grad
    assert torch.equal(a, b.detach())


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    model, x, ctx, _ = build_package_case("f")
    model = model.cuda()
    loss = model.forward_kld(x.cuda(), ctx.cuda())
    with torch.no_grad():
        model.flows[0].autoregressive_net.final_layer.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()


@pytest.mark.gpu
def test_no_context_gradient_formed_unless_wanted(monkeypatch):
    from normflows import _standalone
    seen = []
    real = _standalone.maf_inverse_backward

    def spy(*a, **k):
        out = real(*a, **k)
        seen.append(out[1])
        return out
    monkeypatch.setattr(_standalone, "maf_inverse_backward", spy)
    model, x, ctx, _ = build_package_case("f")
    model = model.cuda()
    model.forward_kld(x.cuda(), ctx.cuda()).backward()
    assert len(seen) == 4 and all(g is None for g in seen)
    seen.clear()
    cc = ctx.cuda().requires_grad_(True)
    model.forward_kld(x.cuda(), cc).backward()
    assert len(seen) == 4 and all(g is not None for g in seen) and cc.grad is not None


@pytest.mark.gpu
def test_notebook_training_loop_trains_every_parameter():
    """examples/conditional_flow.ipynb's MAF model and loop: forward_kld(x, context) + backward + Adam(1e-3, wd 1e-5)."""
    import normflows as nf
    torch.manual_seed(0)
    flows = []
    for _ in range(4):
        flows += [nf.flows.MaskedAffineAutoregressive(2, 128, context_features=4, num_blocks=2),
                  nf.flows.LULinearPermute(2)]
    model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows).cuda()
    start = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-5)
    g = torch.Generator(device="cuda").manual_seed(1)

    def batch(n=128):   # x ~ N(context[:, :2], exp(context[:, 2:]))
        c = torch.rand(n, 4, device="cuda", generator=g) * 2 - 1
        return c[:, :2] + torch.exp(0.5 * c[:, 2:]) * torch.randn(n, 2, device="cuda", generator=g), c
    xe, ce = batch(4096)
    with torch.no_grad():
        first = model.forward_kld(xe, ce).item()
    for _ in range(300):
        x, c = batch()
        opt.zero_grad()
        loss = model.forward_kld(x, c)
        assert torch.isfinite(loss)
        loss.backward()
        opt.step()
    with torch.no_grad():
        last = model.forward_kld(xe, ce).item()
        lp = model.log_prob(xe[:1024], ce[:1024])
    assert math.isfinite(last) and last < first - 0.05, (first, last)
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert not torch.equal(p.detach(), start[n]), f"{n} did not move"
    # the trained model's density against the fp64 restatement
    P = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    with torch.no_grad():
        z, log_q = xe[:1024].double().cpu(), torch.zeros(1024, dtype=torch.float64)
        for i in range(7, -1, -1):
            if i % 2:
                z, ld = lu_inverse_ref(P, f"flows.{i}.", z)
            else:
                z, ld = maf_unrolled(P, f"flows.{i}.autoregressive_net.", 2, z, ce[:1024].double().cpu())
            log_q = log_q + ld
        lp_ref = log_q - math.log(2 * math.pi) - 0.5 * (z ** 2).sum(1)
    np.testing.assert_allclose(lp.double().cpu().numpy(), lp_ref.numpy(), rtol=1e-4)


def test_new_symbols_exported():
    from normflows import _lib
    hdr = open(os.path.join(ROOT, "include", "nfb200.h")).read()
    for name in ("nfb_maf_inverse_backward", "nfb_maf_inverse_backward_workspace_bytes"):
        assert name + "(" in hdr and name in _lib.SYMBOLS, name
        assert hasattr(_lib.lib(), name), name
