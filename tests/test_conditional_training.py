"""Training of the stand-alone layers: the context-conditioned spline layers (examples/conditional_flow.ipynb), the
circular spline layers (examples/circular_nsf.ipynb), the conditioner nets called as modules and ConditionalDiagGaussian.

CPU: the generalised spline adjoint (csrc/nfb_spline_bwd.cuh rqs_adjoint_params), compiled for the host, against
fp64 autograd of a restatement of utils/splines.py:16-219 and against central finite differences.
GPU: every new C ABI adjoint against torch fp64 autograd, and whole models against gradients minted from the reference's
fp64 autograd (tests/golden/make_conditional_grads.py)."""
import copy
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT

CONST = math.log(math.exp(1 - 1e-3) - 1)


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- fp64 restatement of the reference's spline (utils/splines.py:16-219, density direction) -----------------------
def ref_spline(x, uw, uh, ud, tail, mode, circ=None):
    """mode 'linear' (ud: K - 1), 'circular' (K), 'list' (K + 1, circ: bool per feature).  tail: float or per-feature
    tensor.  Returns (y, lad) elementwise."""
    K = uw.shape[-1]
    if mode == "linear":
        pad = torch.full_like(ud[..., :1], CONST)
        udk = torch.cat([pad, ud, pad], -1)
    elif mode == "circular":
        udk = torch.cat([ud, ud[..., :1]], -1)
    else:
        c = torch.as_tensor(circ, dtype=torch.bool, device=x.device).expand(x.shape)[..., None]
        end = torch.where(c, ud[..., :1], torch.full_like(ud[..., :1], CONST))
        udk = torch.cat([end, ud[..., 1:K], end], -1)
    tail = torch.as_tensor(tail, dtype=x.dtype, device=x.device).expand(x.shape)
    inside = (x >= -tail) & (x <= tail)
    xs = torch.where(inside, x, torch.zeros_like(x))
    t = tail[..., None]

    def knots(u):
        s = 1e-3 + (1 - 1e-3 * K) * torch.softmax(u, -1)
        c = F.pad(torch.cumsum(s, -1), (1, 0))
        c = (2 * c - 1) * t
        c = torch.cat([-t, c[..., 1:-1], t], -1)
        return c, c[..., 1:] - c[..., :-1]
    cw, w = knots(uw)
    ch, h = knots(uh)
    d = 1e-3 + F.softplus(udk)
    loc = cw.detach().clone()
    loc[..., -1] += 1e-6
    idx = (torch.sum(xs[..., None] >= loc, -1) - 1).clamp(0, K - 1)[..., None]
    g = lambda a: a.gather(-1, idx)[..., 0]
    in_cw, in_w, in_ch, in_h, d0, d1 = g(cw), g(w), g(ch), g(h), g(d), g(d[..., 1:])
    delta = in_h / in_w
    th = (xs - in_cw) / in_w
    tt = th * (1 - th)
    num = in_h * (delta * th ** 2 + d0 * tt)
    den = delta + (d0 + d1 - 2 * delta) * tt
    y = in_ch + num / den
    dnum = delta ** 2 * (d1 * th ** 2 + 2 * delta * tt + d0 * (1 - th) ** 2)
    lad = torch.log(dnum) - 2 * torch.log(den)
    outside = torch.zeros_like(x) if mode == "list" else x
    return torch.where(inside, y, outside), torch.where(inside, lad, torch.zeros_like(lad))


def ref_spline_params(x, p, K, mode, tail, wh=1.0, circ=None):
    """ref_spline on per-element parameter records [..., 2K + nd]."""
    return ref_spline(x, p[..., :K] * wh, p[..., K:2 * K] * wh, p[..., 2 * K:], tail, mode, circ)


def spline_cases(rng, rows, feats, K, mode, wh=1.0, shared=False):
    """Inputs that hit the interior, the interval ends, interior knots, outside points and NaN.  wh: the width / height
    logit scale the spline will run with; shared: every row uses the parameters of row 0 (a shared table)."""
    nd = {"linear": K - 1, "circular": K, "list": K + 1}[mode]
    P = 2 * K + nd
    params = rng.normal(size=(rows, feats, P)) * 1.5
    if shared:
        params[:] = params[:1]
    tail = rng.uniform(1.5, 4.0, size=feats)
    x = rng.uniform(-1.2, 1.2, size=(rows, feats)) * tail
    x[0, :] = tail
    x[1, :] = -tail
    x[2, 0] = np.nan
    # interior knot hits: x exactly on interior knot min(3, K - 1) of the width partition the spline uses (fp64)
    for r in range(3, 8):
        for f in range(feats):
            u = params[r, f, :K] * wh
            s = np.exp(u - u.max())
            s = 1e-3 + (1 - 1e-3 * K) * s / s.sum()
            x[r, f] = (2 * np.cumsum(s)[min(2, K - 2)] - 1) * tail[f]
    circ = (np.arange(feats) % 2 == 1) if mode == "list" else np.ones(feats, bool)
    return x, params, tail, circ, nd


@pytest.fixture(scope="module")
def adjlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "spline_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "spline_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_adjoint(lib, x, params, tail, circ, K, nd, gy, gl, wh=1.0, use_float=0):
    rows, feats = x.shape
    n = rows * feats
    P = 2 * K + nd
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
    ci = np.ascontiguousarray(np.broadcast_to(circ, (rows, feats)).reshape(-1), dtype=np.int32)
    tb = f(np.broadcast_to(tail, (rows, feats)))
    y, lad, gx, gp = np.empty(n), np.empty(n), np.empty(n), np.empty(n * P)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    xs, ps, gys, gls = f(x), f(params), f(gy), f(np.broadcast_to(np.asarray(gl)[:, None], (rows, feats)))
    lib.spline_adjoint_check(n, K, nd, vp(ci), vp(xs), vp(ps), C.c_double(wh), vp(tb), vp(gys), vp(gls),
                             int(use_float), vp(y), vp(lad), vp(gx), vp(gp))
    sh = (rows, feats)
    return y.reshape(sh), lad.reshape(sh), gx.reshape(sh), gp.reshape(rows, feats, P)


@pytest.mark.parametrize("mode,K", [("linear", 8), ("linear", 5), ("linear", 2), ("circular", 8), ("circular", 3),
                                    ("list", 8), ("list", 6), ("list", 32)])
def test_spline_adjoint_matches_fp64_autograd(adjlib, mode, K):
    rng = np.random.default_rng(11 + K)
    rows, feats = 96, 3
    wh = 0.7
    x, params, tail, circ, nd = spline_cases(rng, rows, feats, K, mode, wh)
    gy, gl = rng.normal(size=(rows, feats)), rng.normal(size=rows)
    y, lad, gx, gp = host_adjoint(adjlib, x, params, tail, circ, K, nd, gy, gl, wh)
    def ref_at(xx):
        xt = torch.tensor(xx, requires_grad=True)
        pt = torch.tensor(params, requires_grad=True)
        yr, lr = ref_spline_params(xt, pt, K, mode, torch.tensor(tail), wh, circ)
        loss = (torch.nan_to_num(yr) * torch.tensor(gy)).sum() + (lr.sum(1) * torch.tensor(gl)).sum()
        gxr, gpr = torch.autograd.grad(loss, [xt, pt])
        return yr.detach().numpy(), lr.detach().numpy(), gxr.numpy(), gpr.numpy()
    yr, lr, gxr, gpr = ref_at(x)
    nan = np.isnan(x)
    knot = np.zeros(rows, bool)
    knot[3:8] = True
    np.testing.assert_allclose(y[~nan], yr[~nan], rtol=1e-7, atol=1e-8)
    np.testing.assert_allclose(lad, lr, rtol=1e-7, atol=1e-8)
    np.testing.assert_allclose(gx[~nan & ~knot[:, None]], gxr[~nan & ~knot[:, None]], rtol=1e-6, atol=1e-8)
    np.testing.assert_allclose(gp[~knot], gpr[~knot], rtol=1e-6, atol=1e-8)
    # on an interior knot the log-det's slope jumps: the gradient is the one of the bin on either side (which side is
    # decided by the last bit of the knot position), so it must equal the reference just left or just right of the knot
    eps = 1e-10 * tail
    sides = [ref_at(x - eps), ref_at(x + eps)]
    for r in range(3, 8):
        for f in range(feats):
            assert any(np.allclose(gx[r, f], sd[2][r, f], rtol=1e-4, atol=1e-6) and
                       np.allclose(gp[r, f], sd[3][r, f], rtol=1e-4, atol=1e-6) for sd in sides), (r, f)
    # semantics the reference fixes exactly
    outside = np.abs(x) > tail
    assert outside.any()
    if mode == "list":
        assert (y[outside] == 0).all() and (gx[outside] == 0).all() and (gp[outside] == 0).all()
        assert (y[nan] == 0).all() and (gx[nan] == 0).all()
        assert (gp[..., 3 * K] == 0).all()                       # derivative K is a copy (circular) or pinned (linear)
        assert (gp[:, ~circ, 2 * K] == 0).all()                  # pinned end of a linear feature
    else:
        assert (y[outside] == x[outside]).all() and np.allclose(gx[outside], gy[outside]) and (gp[outside] == 0).all()
        assert np.isnan(y[nan]).all() and np.allclose(gx[nan], gy[nan])
    # the float instantiation (what the kernels run) agrees to fp32 accuracy
    _, _, gx32, gp32 = host_adjoint(adjlib, x, params, tail, circ, K, nd, gy, gl, wh, use_float=1)
    for got, ref in ((gx32[~nan & ~knot[:, None]], gx[~nan & ~knot[:, None]]), (gp32[~knot], gp[~knot])):
        assert np.mean(np.abs(got - ref) < 2e-4 * np.abs(ref).max() + 1e-5) > 0.995


@pytest.mark.parametrize("mode,K", [("linear", 4), ("circular", 8), ("list", 10)])
def test_spline_adjoint_matches_finite_differences(adjlib, mode, K):
    rng = np.random.default_rng(7)
    rows, feats = 120, 2
    x, params, tail, circ, nd = spline_cases(rng, rows, feats, K, mode)
    x[:8] = rng.uniform(-0.9, 0.9, size=(8, feats)) * tail   # interior points only: FD is meaningless at a knot
    x[8:12] = 1.1 * tail                                     # plus some outside
    eps = 1e-6
    gy, gl = rng.normal(size=(rows, feats)), rng.normal(size=rows)
    obj = lambda xx, pp: (lambda r: (r[0] * gy).sum(1) + r[1].sum(1) * gl)(
        host_adjoint(adjlib, xx, pp, tail, circ, K, nd, gy, gl))
    _, _, gx, gp = host_adjoint(adjlib, x, params, tail, circ, K, nd, gy, gl)
    fd = (obj(x + eps, params) - obj(x - eps, params)) / (2 * eps)
    assert (np.abs(fd[:, None] - gx.sum(1, keepdims=True)) < 1e-4 * (1 + np.abs(gx).sum(1, keepdims=True))).mean() > 0.97
    for k in range(2 * K + nd):
        d = np.zeros_like(params)
        d[..., k] = eps
        fd = (obj(x, params + d) - obj(x, params - d)) / (2 * eps)
        got = gp[..., k].sum(1)
        assert (np.abs(fd - got) < 1e-5 * (1 + np.abs(got))).mean() > 0.97, k


def test_new_symbols_exported():
    from normflows import _lib
    hdr = open(os.path.join(ROOT, "include", "nfb200.h")).read()
    for name in ("nfb_rqs_spline_backward", "nfb_rqs_spline_tails_backward", "nfb_periodic_features_backward",
                 "nfb_glu_residual_backward", "nfb_resnet_backward", "nfb_resnet_backward_workspace_bytes",
                 "nfb_mlp_backward", "nfb_mlp_backward_workspace_bytes"):
        assert name + "(" in hdr and name in _lib.SYMBOLS, name
        assert hasattr(_lib.lib(), name), name


# ================================================ GPU ================================================================
def _close(got, ref, name, tol=2e-3):
    """Every tensor within tol of its scale, or (ReLU kinks resolved differently in fp32 and fp64) >= 97 % of the
    entries within tol and the Frobenius error within 1e-2 of the reference's norm."""
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = ref.abs().max().item() + 1e-12
    err = (got - ref).abs()
    if err.max().item() <= tol * scale:
        return
    frac = (err <= tol * scale).double().mean().item()
    fro = ((got - ref).norm() / (ref.norm() + 1e-30)).item()
    assert frac >= 0.97 and fro <= 1e-2, f"{name}: max err {err.max().item():.3e} scale {scale:.3e} frac {frac:.3f}"


def _perturb(model, seed, s=0.05):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(s * torch.randn(p.shape, generator=g))


def ref_net(net, x, context, masked):
    W = lambda l: l.weight * l.mask if masked else l.weight
    lin = lambda l, v: F.linear(v, W(l), l.bias)
    if net.preprocessing is not None:
        x = ref_periodic(net.preprocessing, x)
    if context is not None and not masked:
        h = lin(net.initial_layer, torch.cat([x, context], 1))
    else:
        h = lin(net.initial_layer, x)
        if context is not None:
            h = h + F.linear(context, net.context_layer.weight, net.context_layer.bias)
    for blk in net.blocks:
        t = lin(blk.linear_layers[1], torch.relu(lin(blk.linear_layers[0], torch.relu(h))))
        if context is not None:
            t = t * torch.sigmoid(F.linear(context, blk.context_layer.weight, blk.context_layer.bias))
        h = h + t
    return lin(net.final_layer, h)


def ref_periodic(pf, x):
    ind = pf.ind
    s = pf.scale if torch.is_tensor(pf.scale) else torch.tensor(float(pf.scale), dtype=x.dtype)
    s = s.to(x)
    v = x[:, ind]
    y = pf.weights[:, 0] * torch.sin(s * v) + pf.weights[:, 1] * torch.cos(s * v)
    if pf.apply_bias:
        y = y + pf.bias
    return x.index_copy(1, ind, y)


def ref_mlp(mlp, x):
    lins = mlp.linear_layers()
    for i, l in enumerate(lins):
        x = F.linear(x, l.weight, l.bias)
        if i + 1 < len(lins):
            x = F.leaky_relu(x, mlp.leaky)
    return x


GOLDEN = os.path.join(ROOT, "tests", "golden")
SEEDS = {"a": 1, "b": 2, "c": 3, "d": 4, "e": 5}


def build_case(name):
    """Model (a)-(e) of tests/golden/make_conditional_grads.py built by this package with the golden's parameters (and
    MADE masks / degrees) loaded; every other buffer (feature splits, tail bounds, periodic-feature scales) is this
    package's own and must equal the reference's.  Returns (model, x, context, golden)."""
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(GOLDEN, f"grads_cond_{name}.npz"))
    torch.manual_seed(SEEDS[name])
    if name in ("a", "b", "c"):
        flows = []
        for _ in range(4 if name != "c" else 2):
            if name == "b":
                flows.append(nf.flows.CoupledRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
            else:
                flows.append(nf.flows.AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
            flows.append(nf.flows.LULinearPermute(2))
        q0 = nf.distributions.DiagGaussian(2, trainable=False) if name != "c" else \
            nf.distributions.ConditionalDiagGaussian(2, nf.nets.MLP([4, 64, 64, 4], leaky=0.01))
        model = nf.ConditionalNormalizingFlow(q0, flows)
    elif name == "d":
        tb = torch.tensor([5.0, math.pi])
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1], tail_bound=tb, permute_mask=True)
                 for _ in range(3)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows)
    else:
        tb = torch.tensor([math.pi, 4.0, 3.0])
        flows = [nf.flows.CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6, tail_bound=tb,
                                                                  reverse_mask=bool(i % 2)) for i in range(2)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(3), flows)
    sd = model.state_dict()
    golden_sd = {k[4:]: v for k, v in gd.items() if k.startswith("sd__")}
    assert set(sd) == set(golden_sd), set(sd) ^ set(golden_sd)
    params = {n for n, _ in model.named_parameters()}
    load = {}
    for k, v in sd.items():
        ref = torch.as_tensor(golden_sd[k]).to(v.dtype)
        if k in params or k.endswith(".mask") or k.endswith(".degrees"):
            load[k] = ref
        else:
            assert torch.equal(v, ref), f"buffer {k} differs from the reference's"
    model.load_state_dict(load, strict=False)
    x = torch.tensor(gd["x"])
    ctx = torch.tensor(gd["context"]) if "context" in gd else None
    return model, x, ctx, gd


def _close_golden(got, gd, name, tol=2e-3):
    """A gradient against the golden: whole, or through the seeded projections G v, u G and |G|."""
    if "g__" + name in gd:
        _close(got, torch.tensor(gd["g__" + name]), name, tol)
        return
    from helpers_glow_grads import grad_projections
    v, u = grad_projections(name, tuple(got.shape))
    G = got.double().cpu().reshape(got.shape[0], -1)
    _close(G @ v, torch.tensor(gd["gv__" + name]), name + " G v", tol)
    _close(u @ G, torch.tensor(gd["gu__" + name]), name + " u G", tol)
    assert abs(G.norm().item() - float(gd["gn__" + name])) <= tol * float(gd["gn__" + name]), name + " |G|"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["a", "b", "c", "d", "e"])
def test_model_gradients_match_reference_goldens(name):
    """forward_kld(x[, context]).backward() against the reference's fp64 autograd (make_conditional_grads.py)."""
    model, x, ctx, gd = build_case(name)
    model = model.cuda()
    xc = x.cuda().requires_grad_(True)
    cc = ctx.cuda().requires_grad_(True) if ctx is not None else None
    loss = model.forward_kld(xc, cc) if cc is not None else model.forward_kld(xc)
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) < 1e-4 * (1 + abs(float(gd["loss"])))
    # (e) is held to 5e-3: the 64-wide conditioners' ReLU kinks make its weight gradients sensitive to fp32 rounding.
    # With the test's fp64 torch restatement evaluated in fp32 and fp64 on the same CPU, the fp32 gradient of
    # flows.1.prqct.transform_net.blocks.1.linear_layers.0.weight is off by 3.4e-2 of its scale at 96 rows and 9.5e-3 at
    # 512 rows, so the spread comes from fp32 itself, not from the kernels; the golden uses 512 rows.
    tol = 5e-3 if name == "e" else 2e-3
    for n, p in model.named_parameters():
        if not p.requires_grad:
            continue
        assert p.grad is not None, f"{n} got no gradient"
        _close_golden(p.grad, gd, n, tol)
    _close_golden(xc.grad, gd, "x", tol)
    if cc is not None:
        _close_golden(cc.grad, gd, "context", tol)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["a", "b", "c", "d", "e"])
def test_values_bit_identical_with_and_without_grad(name):
    model, x, ctx, _ = build_case(name)
    model = model.cuda()
    args = (x.cuda(),) + ((ctx.cuda(),) if ctx is not None else ())
    with torch.no_grad():
        a = model.log_prob(*args)
    b = model.log_prob(*args)
    assert b.requires_grad
    assert torch.equal(a, b.detach())


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    model, x, ctx, _ = build_case("a")
    model = model.cuda()
    loss = model.forward_kld(x.cuda(), ctx.cuda())
    with torch.no_grad():
        model.flows[0].mprqat.autoregressive_net.final_layer.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,K,shared", [("linear", 8, False), ("linear", 5, False), ("linear", 8, True),
                                           ("linear", 11, True), ("list", 8, False), ("list", 6, True),
                                           ("circular", 8, False), ("circular", 32, False)])
def test_spline_backward_kernels(mode, K, shared):
    from normflows._standalone import spline_backward
    rng = np.random.default_rng(K + 3 * shared)
    rows, feats = 1000, 3
    wh = 0.6 if not shared else 1.0
    x, params, tail, circ, nd = spline_cases(rng, rows, feats, K, mode, wh, shared)
    if mode == "linear":   # one scalar bound for nfb_rqs_spline_backward
        x = x / tail * 2.5
        tail = np.full(feats, 2.5)
    x[2, 0] = 0.3   # (NaN semantics are covered on the host)
    if shared:
        params = params[:1]
    gy, gl = rng.normal(size=(rows, feats)), rng.normal(size=rows)
    if shared:   # the table's gradient is a sum over rows: the knot rows (checked per element by the per-row cases) carry no cotangent here
        gy[3:8], gl[3:8] = 0.0, 0.0
    dev = "cuda"
    f32 = lambda a: torch.tensor(np.ascontiguousarray(a), dtype=torch.float32, device=dev)
    xt, pt = f32(x), f32(params.reshape(params.shape[0], -1) if not shared else params[0])
    if mode == "linear":
        gx, gp = spline_backward(xt, pt, shared, K, f32(gy), f32(gl), wh, tail_bound=2.5)
    else:
        gx, gp = spline_backward(xt, pt, shared, K, f32(gy), f32(gl), wh, num_derivatives=nd, tails=f32(tail),
                                 circular=torch.tensor(circ.astype(np.int32), device=dev))
    def ref_at(xx):
        xr = torch.tensor(xx, requires_grad=True)
        pr = torch.tensor(params.astype(np.float32).astype(np.float64), requires_grad=True)
        pe = pr.expand(rows, feats, -1) if shared else pr
        yr, lr = ref_spline_params(xr, pe, K, mode, torch.tensor(tail.astype(np.float32).astype(np.float64)), wh, circ)
        ((yr * torch.tensor(gy)).sum() + (lr.sum(1) * torch.tensor(gl)).sum()).backward()
        return xr.grad, pr.grad
    x64 = x.astype(np.float32).astype(np.float64)
    gxr, gpr = ref_at(x64)
    gx, gp = gx.double().cpu(), gp.reshape(gpr.shape).double().cpu()
    keep = torch.ones(rows, dtype=torch.bool)
    keep[3:8] = False   # interior-knot hits: checked below
    _close(gx[keep], gxr[keep], "gx")
    if not shared:
        _close(gp[keep], gpr[keep], "g_params")
        # knot hits: the gradient of the bin on one side of the knot (fp32 decides the side)
        eps = 1e-7 * tail
        sides = [ref_at(x64 - eps), ref_at(x64 + eps)]
        scale = gpr.abs().max().item()
        for r in range(3, 8):
            for f in range(feats):
                assert any((gp[r, f] - s_[1][r, f]).abs().max().item() < 2e-3 * scale for s_ in sides), (r, f)
    else:
        _close(gp, gpr, "g_table")


@pytest.mark.gpu
def test_glu_and_periodic_adjoints():
    import ctypes
    from normflows import _lib as L
    from normflows._standalone import periodic_backward
    from normflows.utils.nn import PeriodicFeaturesElementwise
    g = torch.Generator().manual_seed(0)
    n = 5000
    h, t, c, go = (torch.randn(n, generator=g).cuda() for _ in range(4))
    gh, gt, gc = torch.empty_like(h), torch.empty_like(h), torch.empty_like(h)
    L.check(L.lib().nfb_glu_residual_backward(L.ptr(go), L.ptr(t), L.ptr(c), n, L.ptr(gh), L.ptr(gt), L.ptr(gc),
                                              L.stream_ptr()))
    hr, tr, cr = (v.double().cpu().requires_grad_(True) for v in (h, t, c))
    (hr + tr * torch.sigmoid(cr)).backward(go.double().cpu())
    for got, ref, nm in ((gh, hr.grad, "gh"), (gt, tr.grad, "gt"), (gc, cr.grad, "gc")):
        _close(got, ref, nm, 1e-5)
    for bias in (False, True):
        pf = PeriodicFeaturesElementwise(4, [1, 3], torch.tensor([0.7, 1.3]), bias=bias)
        with torch.no_grad():
            pf.weights.add_(torch.randn(2, 2, generator=g))
        pf = pf.cuda()
        x = torch.randn(3000, 4, generator=g).cuda()
        gy = torch.randn(3000, 4, generator=g).cuda()
        gx, gmap = periodic_backward(pf, x, gy)
        ref = copy.deepcopy(pf).double().cpu()
        xr = x.double().cpu().requires_grad_(True)
        ref_periodic(ref, xr).backward(gy.double().cpu())
        _close(gx, xr.grad, "gx", 1e-5)
        _close(gmap[pf.weights], ref.weights.grad, "g_weights", 1e-5)
        if bias:
            _close(gmap[pf.bias], ref.bias.grad, "g_bias", 1e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,context,rows", [("resnet", False, 700), ("resnet", True, 700), ("made", False, 700),
                                               ("made", True, 129), ("made", True, 0)])
def test_conditioner_backward(kind, context, rows):
    from normflows.nets import MADE, ResidualNet
    torch.manual_seed(3)
    cf = 5 if context else None
    net = ResidualNet(3, 7, 64, cf, 2) if kind == "resnet" else MADE(4, 64, cf, 2, output_multiplier=3)
    _perturb(net, 9, 0.1)
    d_in = 3 if kind == "resnet" else 4
    x = torch.randn(rows, d_in)
    ctx = torch.randn(rows, 5) if context else None
    ref = copy.deepcopy(net).double()
    net = net.cuda()
    xc = x.cuda().requires_grad_(True)
    cc = ctx.cuda().requires_grad_(True) if context else None
    out = net(xc, cc)
    go = torch.randn(out.shape)
    out.backward(go.cuda())
    xr = x.double().requires_grad_(True)
    cr = ctx.double().requires_grad_(True) if context else None
    ref_net(ref, xr, cr, kind == "made").backward(go.double())
    named = dict(ref.named_parameters())
    for n, p in net.named_parameters():
        assert p.grad is not None, n
        _close(p.grad, named[n].grad, n)
    if rows:
        _close(xc.grad, xr.grad, "x")
        if context:
            _close(cc.grad, cr.grad, "context")


@pytest.mark.gpu
@pytest.mark.parametrize("leaky", [0.0, 0.2])
def test_mlp_backward(leaky):
    from normflows.nets import MLP
    torch.manual_seed(4)
    mlp = MLP([6, 48, 32, 5], leaky=leaky)
    ref = copy.deepcopy(mlp).double()
    mlp = mlp.cuda()
    x = torch.randn(900, 6)
    xc = x.cuda().requires_grad_(True)
    go = torch.randn(900, 5)
    mlp(xc).backward(go.cuda())
    xr = x.double().requires_grad_(True)
    ref_mlp(ref, xr).backward(go.double())
    named = dict(ref.named_parameters())
    for n, p in mlp.named_parameters():
        _close(p.grad, named[n].grad, n)
    _close(xc.grad, xr.grad, "x")


@pytest.mark.gpu
def test_notebook_training_loop_trains_every_parameter():
    """examples/conditional_flow.ipynb's loop: forward_kld(x, context) + backward + Adam(3e-4), batch 128."""
    import normflows as nf
    torch.manual_seed(0)
    flows = []
    for _ in range(4):
        flows += [nf.flows.AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4),
                  nf.flows.LULinearPermute(2)]
    model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows).cuda()
    start = {n: p.detach().clone() for n, p in model.named_parameters()}
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, weight_decay=1e-5)
    g = torch.Generator(device="cuda").manual_seed(1)

    def batch(n=128):   # x ~ N(context[:, :2], exp(context[:, 2:]))
        c = torch.rand(n, 4, device="cuda", generator=g) * 2 - 1
        return c[:, :2] + torch.exp(0.5 * c[:, 2:]) * torch.randn(n, 2, device="cuda", generator=g), c
    xe, ce = batch(4096)
    with torch.no_grad():
        first = model.forward_kld(xe, ce).item()
    for _ in range(200):
        x, c = batch()
        opt.zero_grad()
        loss = model.forward_kld(x, c)
        assert torch.isfinite(loss)
        loss.backward()
        opt.step()
    with torch.no_grad():
        last = model.forward_kld(xe, ce).item()
    assert math.isfinite(last) and last < first - 0.05, (first, last)
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert not torch.equal(p.detach(), start[n]), f"{n} did not move"


@pytest.mark.gpu
def test_conditioner_with_other_preprocessing_module():
    """Any preprocessing module is accepted in front of ResidualNet / MADE, as in the reference: its value is the module's
    call and its gradient comes from torch autograd."""
    from normflows.nets import MADE, ResidualNet
    torch.manual_seed(5)
    for net, masked in ((ResidualNet(3, 4, 32, None, 1, preprocessing=torch.nn.Tanh()), False),
                        (MADE(3, 32, None, 1, output_multiplier=2, preprocessing=torch.nn.Linear(3, 3)), True)):
        _perturb(net, 6, 0.1)
        ref = copy.deepcopy(net).double()
        net = net.cuda()
        x = torch.randn(300, 3)
        with torch.no_grad():
            y0 = net(x.cuda())
        xc = x.cuda().requires_grad_(True)
        out = net(xc)
        assert torch.equal(out.detach(), y0)
        go = torch.randn(out.shape)
        out.backward(go.cuda())
        xr = x.double().requires_grad_(True)
        pre = ref.preprocessing
        ref.preprocessing = None
        ref_net(ref, pre(xr), None, masked).backward(go.double())
        named = dict(ref.named_parameters())
        named.update({"preprocessing." + k: v for k, v in pre.named_parameters()})
        for n, p in net.named_parameters():
            assert p.grad is not None, n
            _close(p.grad, named[n].grad, n)
        _close(xc.grad, xr.grad, "x")
