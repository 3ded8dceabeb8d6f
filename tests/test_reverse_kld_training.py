"""Reverse-KL training (examples/paper_example_nsf.ipynb): gradients through the sampling direction (`forward`) of the
stand-alone spline layers -- the autoregressive ones (context-conditioned, circular), whose sampling pass is the
reference's D-pass loop x = G(z; MADE(pre(x), context)) with G the inverse spline, and the coupling ones (inverse
unconditional CDF, conditioner on its output, inverse spline).

The inverse element's adjoint (csrc/nfb_spline_bwd.cuh rqs_inverse_adjoint_params): with c = g_x - g_ld d_x log f'(x),
    g_z = c / f'(x),   g_theta = -(c / f') d_theta f - g_ld d_theta log f'   (the forward adjoint at x).
The autoregressive layer's backward is the fixed-point adjoint of the loop (nfb_ar_rqs_sampling_backward):
    lam = g_x;  repeat D - 1 times: lam = g_x + pre'(x) MADE_dgrad(pbar(lam));  g_z, g_weights from pbar(lam)

CPU: the element, compiled for the host, against central differences of the oracle's inverse spline and against the
identity above evaluated with the forward element; an fp64 torch restatement of the layers' adjoints pinned to
gradients minted from the reference's autograd (tests/golden/make_reverse_kld_grads.py cases h-l); UniformGaussian /
Target buffers and state_dict keys against the reference's.
GPU: each layer's sampling backward against fp64 autograd of its unrolled sampling loop, models h-l against the goldens,
the reverse_kld gating, and the paper notebook's training loop."""
import copy
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers_rkl as R
from conftest import ROOT
from test_conditional_training import ref_net, ref_spline_params

GOLDEN = os.path.join(ROOT, "tests", "golden")
CONST = math.log(math.exp(1 - 1e-3) - 1)


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- fp64 restatement of the reference's inverse spline (utils/splines.py:16-97, 172-198) ---------------------------
def ref_spline_inverse(z, uw, uh, ud, tail, mode, circ=None):
    """(x, ld) elementwise; modes as test_conditional_training.ref_spline ('linear', 'circular', 'list')."""
    K = uw.shape[-1]
    if mode == "linear":
        pad = torch.full_like(ud[..., :1], CONST)
        udk = torch.cat([pad, ud, pad], -1)
    elif mode == "circular":
        udk = torch.cat([ud, ud[..., :1]], -1)
    else:
        c = torch.as_tensor(circ, dtype=torch.bool, device=z.device).expand(z.shape)[..., None]
        end = torch.where(c, ud[..., :1], torch.full_like(ud[..., :1], CONST))
        udk = torch.cat([end, ud[..., 1:K], end], -1)
    tail = torch.as_tensor(tail, dtype=z.dtype, device=z.device).expand(z.shape)
    inside = (z >= -tail) & (z <= tail)
    zs = torch.where(inside, z, torch.zeros_like(z))
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
    loc = ch.detach().clone()
    loc[..., -1] += 1e-6
    idx = (torch.sum(zs[..., None] >= loc, -1) - 1).clamp(0, K - 1)[..., None]
    g = lambda a: a.gather(-1, idx)[..., 0]
    in_cw, in_w, in_ch, in_h, d0, d1 = g(cw), g(w), g(ch), g(h), g(d), g(d[..., 1:])
    delta = in_h / in_w
    s = d0 + d1 - 2 * delta
    a = (zs - in_ch) * s + in_h * (delta - d0)
    b = in_h * d0 - (zs - in_ch) * s
    cc = -delta * (zs - in_ch)
    root = (2 * cc) / (-b - torch.sqrt(b * b - 4 * a * cc))
    x = root * in_w + in_cw
    tt = root * (1 - root)
    den = delta + s * tt
    dnum = delta ** 2 * (d1 * root ** 2 + 2 * delta * tt + d0 * (1 - root) ** 2)
    ld = -(torch.log(dnum) - 2 * torch.log(den))
    outside = torch.zeros_like(z) if mode == "list" else z
    return torch.where(inside, x, outside), torch.where(inside, ld, torch.zeros_like(ld))


def ref_spline_inverse_params(z, p, K, mode, tail, wh=1.0, circ=None):
    return ref_spline_inverse(z, p[..., :K] * wh, p[..., K:2 * K] * wh, p[..., 2 * K:], tail, mode, circ)


def inverse_element_adjoint(z, p, lam, g_ld, K, mode, tail, wh=1.0, circ=None):
    """(g_z, g_p) of the inverse element by the identity above: the forward spline's autograd at x = g(z)."""
    with torch.no_grad():
        x, _ = ref_spline_inverse_params(z, p, K, mode, tail, wh, circ)
    with torch.enable_grad():
        xx, pp = x.detach().requires_grad_(True), p.detach().requires_grad_(True)
        y, lad = ref_spline_params(xx, pp, K, mode, tail, wh, circ)
        dl = torch.autograd.grad(lad.sum(), xx, retain_graph=True)[0]
        gl = g_ld[:, None].expand_as(lad)
        gz = (lam - gl * dl) * torch.exp(-lad)
        gp = torch.autograd.grad((y * -gz.detach()).sum() + (lad * -gl).sum(), pp)[0]
    tb = torch.as_tensor(tail, dtype=z.dtype).expand(z.shape)
    inside = (z >= -tb) & (z <= tb)
    gz = torch.where(inside, gz, torch.zeros_like(gz) if mode == "list" else lam)
    return gz, torch.where(inside[..., None], gp, torch.zeros_like(gp))


# ---- the element on the host -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def invlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "spline_inverse_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "spline_inverse_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_element(lib, z, params, tail, circ, K, nd, gy, gl, inverse=1, use_float=0, wh=1.0):
    rows, feats = z.shape
    n, P = rows * feats, 2 * K + nd
    f = lambda a: np.ascontiguousarray(a, dtype=np.float64).reshape(-1)
    ci = np.ascontiguousarray(np.broadcast_to(circ, (rows, feats)).reshape(-1), dtype=np.int32)
    tb = f(np.broadcast_to(tail, (rows, feats)))
    y, lad, gx, gp = np.empty(n), np.empty(n), np.empty(n), np.empty(n * P)
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    zs, ps, gys, gls = f(z), f(params), f(gy), f(np.broadcast_to(np.asarray(gl)[:, None], (rows, feats)))
    lib.spline_inverse_adjoint_check(n, K, nd, vp(ci), vp(zs), vp(ps), C.c_double(wh), vp(tb), vp(gys), vp(gls),
                                     int(use_float), int(inverse), vp(y), vp(lad), vp(gx), vp(gp))
    sh = (rows, feats)
    return y.reshape(sh), lad.reshape(sh), gx.reshape(sh), gp.reshape(rows, feats, P)


def oracle_inverse(z, params, tail, circ, K, mode):
    """The oracle's numpy inverse spline: unconstrained_rqs(inverse=True) (linear) or unconstrained_rqs_tails (list;
    'circular' mode = a list of circular features, the same inside the interval)."""
    from oracle import nf_oracle as O
    uw, uh, ud = params[..., :K], params[..., K:2 * K], params[..., 2 * K:]
    if mode == "linear":
        return O.unconstrained_rqs(z, uw, uh, ud, inverse=True, tail_bound=tail[None, :])
    if mode == "circular":
        ud = np.concatenate([ud, ud[..., :1]], -1)
    return O.unconstrained_rqs_tails(z, uw, uh, ud, circ, inverse=True, tail_bound=tail)


def inverse_cases(rng, rows, feats, K, mode):
    nd = {"linear": K - 1, "circular": K, "list": K + 1}[mode]
    params = rng.normal(size=(rows, feats, 2 * K + nd)) * 1.5
    tail = rng.uniform(1.5, 4.0, size=feats)
    z = rng.uniform(-0.98, 0.98, size=(rows, feats)) * tail
    circ = (np.arange(feats) % 2 == 1) if mode == "list" else np.ones(feats, bool)
    return z, params, tail, circ, nd


def height_knots(params, K, tail):
    """Interior height knots (the reference's cumheights) of each element, fp64: [rows, feats, K - 1]."""
    u = params[..., K:2 * K]
    s = np.exp(u - u.max(-1, keepdims=True))
    s = 1e-3 + (1 - 1e-3 * K) * s / s.sum(-1, keepdims=True)
    return (2 * np.cumsum(s, -1)[..., :-1] - 1) * tail[None, :, None]


@pytest.mark.parametrize("mode,K", [("linear", 8), ("linear", 5), ("circular", 8), ("circular", 3), ("list", 10),
                                    ("list", 6), ("list", 8)])
def test_inverse_element_matches_oracle_central_differences(invlib, mode, K):
    rng = np.random.default_rng(K * 7 + len(mode))
    z, params, tail, circ, nd = inverse_cases(rng, 40, 3, K, mode)
    gy, gl = rng.normal(size=z.shape), rng.normal(size=40)
    x, ld, gz, gp = host_element(invlib, z, params, tail, circ, K, nd, gy, gl)
    xo, ldo = oracle_inverse(z, params, tail, circ, K, mode)
    np.testing.assert_allclose(x, xo, rtol=1e-8, atol=1e-8)
    np.testing.assert_allclose(ld, ldo, rtol=1e-7, atol=1e-8)
    obj = lambda zz, pp: (lambda r: r[0] * gy + r[1] * gl[:, None])(oracle_inverse(zz, pp, tail, circ, K, mode))
    eps = 1e-6
    fd = (obj(z + eps, params) - obj(z - eps, params)) / (2 * eps)
    np.testing.assert_allclose(gz, fd, rtol=1e-5, atol=1e-6 * np.abs(fd).max())
    for k in range(2 * K + nd):
        dp = np.zeros_like(params)
        dp[..., k] = eps
        fd = (obj(z, params + dp) - obj(z, params - dp)) / (2 * eps)
        np.testing.assert_allclose(gp[..., k], fd, rtol=1e-5, atol=1e-6 * max(1.0, np.abs(fd).max()),
                                   err_msg=f"parameter {k}")
    # the float instantiation (what the kernels run) agrees to fp32 accuracy
    xf, ldf, gzf, gpf = host_element(invlib, z, params, tail, circ, K, nd, gy, gl, use_float=1)
    np.testing.assert_allclose(gzf, gz, rtol=1e-3, atol=1e-4 * np.abs(gz).max())
    np.testing.assert_allclose(gpf, gp, rtol=1e-3, atol=1e-4 * np.abs(gp).max())


@pytest.mark.parametrize("mode,K", [("linear", 8), ("circular", 8), ("list", 10), ("list", 4)])
def test_inverse_element_is_the_forward_adjoint_at_x(invlib, mode, K):
    """g_theta = forward adjoint at x with cotangents (-g_z, -g_ld); g_z = c / f'(x), c = g_x - g_ld d_x log f'."""
    rng = np.random.default_rng(3 + K)
    z, params, tail, circ, nd = inverse_cases(rng, 64, 4, K, mode)
    gy, gl = rng.normal(size=z.shape), rng.normal(size=64)
    x, ld, gz, gp = host_element(invlib, z, params, tail, circ, K, nd, gy, gl)
    y, lad, _, gpf = host_element(invlib, x, params, tail, circ, K, nd, -gz, -gl, inverse=0)
    np.testing.assert_allclose(y, z, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(lad, -ld, rtol=1e-10, atol=1e-12)
    np.testing.assert_allclose(gpf, gp, rtol=1e-9, atol=1e-12 * np.abs(gp).max())
    _, _, dl, _ = host_element(invlib, x, params, tail, circ, K, nd, np.zeros_like(z), np.ones(64), inverse=0)
    np.testing.assert_allclose(gz, (gy - gl[:, None] * dl) * np.exp(-lad), rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("mode,K", [("linear", 8), ("circular", 5), ("list", 10)])
def test_inverse_element_on_interior_knots_outside_and_nan(invlib, mode, K):
    """z on an interior height knot keeps the bin the inverse spline selects (the reference's: the right one), so the
    gradient is the reference's there; outside the interval: identity (linear, circular) or 0 (list); NaN passes."""
    rng = np.random.default_rng(11)
    rows, feats = 24, 2
    z, params, tail, circ, nd = inverse_cases(rng, rows, feats, K, mode)
    kn = height_knots(params, K, tail)
    for r in range(8):
        z[r, :] = kn[r, np.arange(feats), r % (K - 1)]
    z[8, :], z[9, :] = tail, -tail
    z[10, :], z[11, :] = 1.3 * tail, -2.0 * tail
    z[12, 0] = np.nan
    gy, gl = rng.normal(size=z.shape), rng.normal(size=rows)
    x, ld, gz, gp = host_element(invlib, z, params, tail, circ, K, nd, gy, gl)

    def reference_at(zz):
        zt, pt = torch.tensor(zz, requires_grad=True), torch.tensor(params, requires_grad=True)
        xr, ldr = ref_spline_inverse_params(zt, pt, K, mode, torch.tensor(tail), 1.0, torch.tensor(circ))
        ((xr * torch.tensor(gy)).nan_to_num().sum() + (ldr * torch.tensor(gl)[:, None]).nan_to_num().sum()).backward()
        return xr.detach().numpy(), zt.grad.numpy(), pt.grad.numpy()
    ok = ~np.isnan(z)
    xr, gzr, gpr = reference_at(z)
    np.testing.assert_allclose(x[ok], xr[ok], rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(gz[8:12], gzr[8:12], rtol=1e-8, atol=1e-9 * np.abs(gz[8:12]).max())
    np.testing.assert_allclose(gp[8:12], gpr[8:12], rtol=1e-8, atol=1e-9 * np.abs(gp).max())
    # on a knot, which bin holds z is decided by the last ulp of the knot (the element searches the height knots with
    # rqs_eval_dyn's inverse arithmetic, the fp64 restatement with the reference's): the element's value and gradient
    # must be those of ONE side, the bin on either side of the knot (not a mix, not a re-search on x)
    _, gz_lo, gp_lo = reference_at(np.where(ok, z - 1e-13 * np.abs(tail), z))
    _, gz_hi, gp_hi = reference_at(np.where(ok, z + 1e-13 * np.abs(tail), z))
    for r in range(8):
        for f in range(feats):
            sides = [(gz_lo[r, f], gp_lo[r, f]), (gz_hi[r, f], gp_hi[r, f])]
            assert any(abs(gz[r, f] - a) <= 1e-5 * (1 + abs(a)) and np.allclose(gp[r, f], b, rtol=1e-5, atol=1e-5)
                       for a, b in sides), (r, f, gz[r, f], gp[r, f], sides)
    out = slice(10, 12)
    assert (gp[out] == 0).all() and (ld[out] == 0).all()
    if mode == "list":
        assert (x[out] == 0).all() and (gz[out] == 0).all()
    else:
        assert (x[out] == z[out]).all() and (gz[out] == gy[out]).all()
    assert np.isnan(x[12, 0]) == (mode != "list") and np.isfinite(gz[12, 1])


# ---- fp64 restatement of the layers' sampling passes and of their adjoints ------------------------------------------
def layer_spec(layer):
    from normflows.flows.neural_spline import (CircularAutoregressiveRationalQuadraticSpline,
                                               CircularCoupledRationalQuadraticSpline, _tail_tensors)
    if hasattr(layer, "mprqat"):
        net, D = layer.mprqat.autoregressive_net, layer.features
        if isinstance(layer, CircularAutoregressiveRationalQuadraticSpline):
            tb, circ = _tail_tensors(layer._tail_bound, range(D), layer.ind_circ, D, "cpu")
            return dict(kind="ar", net=net, K=layer.num_bins, mode="list", tail=tb.double(), circ=circ.bool())
        return dict(kind="ar", net=net, K=layer.num_bins, mode="linear", tail=layer.tail_bound, circ=None)
    p = layer.prqct
    spec = dict(kind="coupling", p=p, K=layer.num_bins, wh=1.0 / math.sqrt(p.transform_net.hidden_features))
    if isinstance(layer, CircularCoupledRationalQuadraticSpline):
        (tb_id, c_id), (tb_tr, c_tr) = layer._tails(p, "cpu")
        spec.update(mode="list", id=(tb_id.double(), c_id.bool()), tr=(tb_tr.double(), c_tr.bool()))
    else:
        spec.update(mode="linear", id=(layer.tail_bound, None), tr=(layer.tail_bound, None))
    return spec


def _uncond_table(p):
    u = p.unconditional_transform
    return torch.cat([u.unnormalized_widths, u.unnormalized_heights, u.unnormalized_derivatives], 1)


def _records(out, feats):
    """A conditioner output [rows, feats * P] as per-feature spline records [rows, feats, P] (also for 0 rows)."""
    return out.reshape(out.shape[0], feats, out.shape[1] // feats)


def sampling_unrolled(spec, z, ctx):
    """The reference's sampling pass, differentiable by autograd (the AR layer: its D-pass loop)."""
    K, mode = spec["K"], spec["mode"]
    rows = z.shape[0]
    if spec["kind"] == "ar":
        x, ld = torch.zeros_like(z), None
        for _ in range(z.shape[1]):
            prm = _records(ref_net(spec["net"], x, ctx, True), z.shape[1])
            x, ld = ref_spline_inverse_params(z, prm, K, mode, spec["tail"], 1.0, spec["circ"])
        return x, ld.sum(1)
    p = spec["p"]
    idf, trf = p.identity_features, p.transform_features
    table = _uncond_table(p)
    yi, ldi = ref_spline_inverse_params(z[:, idf], table.expand(rows, -1, -1), K, mode, *spec["id"][:1], 1.0,
                                        spec["id"][1])
    prm = _records(ref_net(p.transform_net, yi, ctx, False), len(trf))
    yt, ld = ref_spline_inverse_params(z[:, trf], prm, K, mode, spec["tr"][0], spec["wh"], spec["tr"][1])
    out = torch.empty_like(z)
    out[:, idf], out[:, trf] = yi, yt
    return out, ld.sum(1) + ldi.sum(1)


class SamplingAdjoint(torch.autograd.Function):
    """The sampling pass under no_grad; backward: the algorithms the native code runs (the AR fixed point with the
    periodic features' adjoint, or the coupling composition), on the inverse element's adjoint restated above."""

    @staticmethod
    def forward(ctx, spec, z, context, *params):
        with torch.no_grad():
            x, ld = sampling_unrolled(spec, z, context)
        ctx.spec, ctx.params = spec, params
        ctx.save_for_backward(z, x, context)
        return x, ld

    @staticmethod
    def backward(ctx, g_x, g_ld):
        z, x, context = ctx.saved_tensors
        spec, params = ctx.spec, ctx.params
        K, mode, rows = spec["K"], spec["mode"], z.shape[0]
        g_x = torch.zeros_like(z) if g_x is None else g_x
        g_ld = torch.zeros(rows, dtype=z.dtype) if g_ld is None else g_ld
        cv = context.detach().requires_grad_(True) if context is not None else None
        with torch.enable_grad():
            if spec["kind"] == "ar":
                xv = x.detach().requires_grad_(True)
                prm = ref_net(spec["net"], xv, cv, True).view(rows, z.shape[1], -1)
                elem = lambda lam: inverse_element_adjoint(z, prm.detach(), lam, g_ld, K, mode, spec["tail"], 1.0,
                                                           spec["circ"])
                lam = g_x
                for _ in range(z.shape[1] - 1):
                    lam = g_x + torch.autograd.grad(prm, xv, elem(lam)[1], retain_graph=True)[0]
                gz, gp = elem(lam)
                ins = ([cv] if cv is not None else []) + list(params)
                grads = list(torch.autograd.grad(prm, ins, gp, allow_unused=True))
                g_ctx = grads.pop(0) if cv is not None else None
                return (None, gz, g_ctx, *grads)
            p = spec["p"]
            idf, trf = p.identity_features, p.transform_features
            table = _uncond_table(p).detach()
            with torch.no_grad():
                yi, _ = ref_spline_inverse_params(z[:, idf], table.expand(rows, -1, -1), K, mode, spec["id"][0], 1.0,
                                                  spec["id"][1])
            yv = yi.requires_grad_(True)
            prm = ref_net(p.transform_net, yv, cv, False).view(rows, len(trf), -1)
            g_tr, gp = inverse_element_adjoint(z[:, trf], prm.detach(), g_x[:, trf], g_ld, K, mode, spec["tr"][0],
                                               spec["wh"], spec["tr"][1])
            net_params = list(p.transform_net.parameters())
            ins = [yv] + ([cv] if cv is not None else []) + net_params
            grads = list(torch.autograd.grad(prm, ins, gp, allow_unused=True))
        g_yi = g_x[:, idf] + grads.pop(0)
        g_ctx = grads.pop(0) if cv is not None else None
        g_id, g_tab = inverse_element_adjoint(z[:, idf], table.expand(rows, -1, -1).contiguous(), g_yi, g_ld, K, mode,
                                              spec["id"][0], 1.0, spec["id"][1])
        g_tab = g_tab.sum(0)
        gz = torch.empty_like(z)
        gz[:, idf], gz[:, trf] = g_id, g_tr
        u = p.unconditional_transform
        gmap = dict(zip(net_params, grads))
        gmap.update({u.unnormalized_widths: g_tab[:, :K], u.unnormalized_heights: g_tab[:, K:2 * K],
                     u.unnormalized_derivatives: g_tab[:, 2 * K:]})
        return (None, gz, g_ctx, *[gmap.get(q) for q in params])


def sampling_fixed_point(layer, z, ctx):
    return SamplingAdjoint.apply(layer_spec(layer), z, ctx, *layer.parameters())


def density_ar(layer, x, ctx):
    """The AR layers' density direction (one MADE pass) in fp64: (z, log_det)."""
    s = layer_spec(layer)
    prm = ref_net(s["net"], x, ctx, True).view(x.shape[0], x.shape[1], -1)
    y, lad = ref_spline_params(x, prm, s["K"], s["mode"], s["tail"], 1.0, s["circ"])
    return y, lad.sum(1)


def base_log_prob(q0, z):
    if hasattr(q0, "inv_perm"):
        s = q0.scale
        g = -0.5 * math.log(2 * math.pi) - torch.log(s[q0.ind_]) - 0.5 * (z[:, q0.ind_] / s[q0.ind_]) ** 2
        return -torch.log(s[q0.ind]).sum() + g.sum(1)
    ls = q0.log_scale.reshape(-1)
    return -0.5 * z.shape[1] * math.log(2 * math.pi) - ls.sum() - 0.5 * (((z - q0.loc) / torch.exp(ls)) ** 2).sum(1)


def restated_loss(name, model, eps, ctx, fixed_point=True):
    """reverse_kld / reverse_alpha_div of cases h-l, restated (core.py:104-165, 337-366)."""
    sample = sampling_fixed_point if fixed_point else (lambda l, z, c: sampling_unrolled(layer_spec(l), z, c))
    if hasattr(model.q0, "inv_perm"):   # UniformGaussian: the replayed draw, the density restated
        z = model.q0.scale * eps
        log_q = base_log_prob(model.q0, z)
    else:
        z, log_q = R.replay_forward(model.q0, eps)(eps.shape[0])
    for f in model.flows:
        z, ld = sample(f, z, ctx)
        log_q = log_q - ld
    target = model.p
    log_p = target.log_prob(z, context=ctx) if ctx is not None else target.log_prob(z)

    def log_q_no_param_grad():
        for q in model.parameters():
            q.requires_grad_(False)
        zz, lq = z, torch.zeros(z.shape[0])   # float32, like the reference's buffer (core.py:123, 151)
        for f in reversed(model.flows):
            zz, ld = density_ar(f, zz, None)
            lq += ld
        lq += base_log_prob(model.q0, zz)
        for q in model.parameters():
            q.requires_grad_(True)
        return lq
    if name == "i":
        log_q = log_q_no_param_grad()
    if name == "j":   # alpha = 1, dreg
        w_const = torch.exp(log_p - log_q).detach()
        log_q = log_q_no_param_grad()
        w = torch.exp(log_p - log_q)
        w_alpha = w_const / torch.mean(w_const)
        return -torch.mean(w_alpha ** 2 * torch.log(w))
    return torch.mean(log_q) - torch.mean(log_p)


def build_case(name):
    """Case h-l built by this package (on the CPU) with the golden's parameters and MADE masks; every other buffer must
    equal the reference's."""
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(GOLDEN, f"grads_rkl_{name}.npz"))
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    torch.manual_seed(0)
    if name in ("h", "i"):
        tb = torch.tensor([5.0, math.pi])
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 64, [1], num_bins=10, tail_bound=tb,
                                                                        permute_mask=True) for _ in range(3)]
        q0 = nf.distributions.UniformGaussian(2, [1], torch.tensor([1.0, 2 * math.pi]))
        model = nf.NormalizingFlow(q0, flows, R.gaussian_von_mises(nf.distributions.Target))
    elif name == "j":
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(5, 2, 64, [1, 3]) for _ in range(2)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows, R.TorusTarget5())
    elif name == "k":
        tb = torch.tensor([math.pi, 4.0, 3.0])
        flows = [nf.flows.CircularCoupledRationalQuadraticSpline(3, 2, 64, [1], num_bins=6, tail_bound=tb,
                                                                  reverse_mask=bool(i % 2)) for i in range(2)]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(3), flows, R.TorusTarget3())
    else:
        flows = [nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 64, num_context_channels=4),
                 nf.flows.CoupledRationalQuadraticSpline(2, 1, 64, num_context_channels=4),
                 nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 64, num_context_channels=4)]
        model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows,
                                              R.ContextTarget())
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    params = {n for n, _ in model.named_parameters()}
    load = {}
    for k, v in own.items():
        ref = sd[k].to(v.dtype)
        if k in params or k.endswith((".mask", ".degrees")):
            load[k] = ref
        else:
            assert torch.allclose(v.double(), ref.double(), rtol=1e-6, atol=0), f"buffer {k} differs from the reference's"
            load[k] = ref
    model.load_state_dict(load, strict=False)
    eps = torch.tensor(gd["eps"])
    ctx = torch.tensor(gd["context"]) if "context" in gd else None
    return model, eps, ctx, gd


def check_golden(got, gd, name, tol):
    from test_maf_training import check_golden as check
    check(got, gd, name, tol)


CASES = ["h", "i", "j", "k", "l"]


@pytest.mark.parametrize("name", CASES)
def test_fp64_sampling_adjoints_match_reference_goldens(name):
    """The restated adjoints (AR fixed point with D - 1 data passes, coupling composition) give the reference's
    unrolled-loop autograd gradients to 1e-10 of each scale."""
    model, eps, ctx, gd = build_case(name)
    model = model.double()
    loss = restated_loss(name, model, eps.double(), ctx.double() if ctx is not None else None)
    loss.backward()
    # the reference accumulates the density pass's log_q in a float32 buffer (core.py:123, 151), so the losses of i and j
    # carry fp32 rounding; their gradients do not
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    minted = {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))}
    assert minted == set(names), minted ^ set(names)
    for n, p in model.named_parameters():
        check_golden(p.grad, gd, n, 1e-10)


def test_h_has_draws_beyond_the_tail_bound():
    eps = R.draws("h")
    assert (eps[:, 0].abs() > 5).sum() >= 4


def test_uniform_gaussian_and_target_match_the_reference_buffers():
    """Case h's golden carries the reference's UniformGaussian(2, [1], [1, 2 pi]) (q0.*) and its GaussianVonMises(Target)
    (p.*) state: same keys, order, dtypes and values."""
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(GOLDEN, "grads_rkl_h.npz"))
    q0 = nf.distributions.UniformGaussian(2, [1], torch.tensor([1.0, 2 * math.pi]))
    target = R.gaussian_von_mises(nf.distributions.Target)
    for pre, mod in (("q0.", q0), ("p.", target)):
        ref = [k for k in gd if k.startswith("sd__" + pre)]
        own = mod.state_dict()
        assert ["sd__" + pre + k for k in own] == ref, (list(own), ref)
        for k, v in own.items():
            r = gd["sd__" + pre + k]
            assert v.numpy().dtype == r.dtype and np.array_equal(v.numpy(), r), k
    assert list(nf.distributions.UniformGaussian(3, 1).state_dict()) == ["ind", "ind_", "inv_perm", "scale"]
    assert isinstance(target, nf.distributions.Target) and list(nf.distributions.Target().state_dict()) == \
        ["prop_scale", "prop_shift"]


def test_new_symbols_exported():
    from normflows import _lib
    hdr = open(os.path.join(ROOT, "include", "nfb200.h")).read()
    for name in ("nfb_rqs_spline_inverse_backward", "nfb_rqs_spline_tails_inverse_backward",
                 "nfb_ar_rqs_sampling_backward", "nfb_ar_rqs_sampling_backward_workspace_bytes"):
        assert name + "(" in hdr and name in _lib.SYMBOLS, name
        assert hasattr(_lib.lib(), name), name


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


def relu_margin(spec, z, x, ctx):
    """Per row, the smallest |ReLU input| of the conditioner at the point the backward linearises it (the MADE at x,
    the coupling net at the identity features' output), relative to the median: where it is tiny, fp32 and fp64 may
    take different sides of the kink and their gradients legitimately differ by that row's whole contribution."""
    if spec["kind"] == "ar":
        net, inp, masked = spec["net"], x, True
    else:
        p = spec["p"]
        rows = z.shape[0]
        table = _uncond_table(p)
        inp, _ = ref_spline_inverse_params(z[:, p.identity_features], table.expand(rows, -1, -1), spec["K"],
                                           spec["mode"], spec["id"][0], 1.0, spec["id"][1])
        net, masked = p.transform_net, False
    from test_conditional_training import ref_periodic
    W = lambda l: l.weight * l.mask if masked else l.weight
    lin = lambda l, v: F.linear(v, W(l), l.bias)
    if net.preprocessing is not None:
        inp = ref_periodic(net.preprocessing, inp)
    if ctx is not None and not masked:
        h = lin(net.initial_layer, torch.cat([inp, ctx], 1))
    else:
        h = lin(net.initial_layer, inp)
        if ctx is not None:
            h = h + F.linear(ctx, net.context_layer.weight, net.context_layer.bias)
    acts = []
    for blk in net.blocks:
        t1 = lin(blk.linear_layers[0], torch.relu(h))
        acts += [h, t1]
        t = lin(blk.linear_layers[1], torch.relu(t1))
        if ctx is not None:
            t = t * torch.sigmoid(F.linear(ctx, blk.context_layer.weight, blk.context_layer.bias))
        h = h + t
    a = torch.cat(acts, 1).abs()
    return a.min(1).values / a.median()


def make_layer(kind, D, K, context):
    import normflows as nf
    C_ = 3 if context else None
    if kind == "ar":
        return nf.flows.AutoregressiveRationalQuadraticSpline(D, 1, 48, num_context_channels=C_, num_bins=K,
                                                              tail_bound=2.5, permute_mask=True)
    if kind == "car":   # circular every other feature, per-feature bounds
        tb = torch.tensor([2.5 + 0.5 * i for i in range(D)])
        return nf.flows.CircularAutoregressiveRationalQuadraticSpline(D, 2, 48, list(range(1, D, 2)) or [0],
                                                                      num_context_channels=C_, num_bins=K, tail_bound=tb)
    if kind == "cc":
        tb = torch.tensor([2.0 + 0.5 * i for i in range(D)])
        return nf.flows.CircularCoupledRationalQuadraticSpline(D, 2, 48, [0], num_context_channels=C_, num_bins=K,
                                                               tail_bound=tb)
    return nf.flows.CoupledRationalQuadraticSpline(D, 2, 48, num_context_channels=C_, num_bins=K, tail_bound=2.5)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,D,K,context,rows", [
    ("ar", 1, 8, True, 127), ("ar", 2, 10, True, 1061), ("ar", 5, 6, True, 1), ("ar", 16, 8, True, 300),
    ("car", 1, 8, False, 127), ("car", 2, 10, False, 1061), ("car", 5, 6, True, 1061), ("car", 16, 8, False, 300),
    ("car", 5, 8, False, 0), ("cc", 2, 8, False, 1061), ("cc", 5, 6, True, 127), ("cc", 16, 10, False, 1),
    ("coupled", 2, 8, True, 1061), ("coupled", 5, 10, True, 127), ("coupled", 16, 6, True, 0)])
def test_layer_sampling_backward_matches_fp64_autograd(kind, D, K, context, rows):
    torch.manual_seed(D * 100 + K + rows)
    layer = make_layer(kind, D, K, context)
    _perturb(layer, 7 + D, 0.1)
    g = torch.Generator().manual_seed(11)
    z = torch.randn(rows, D, generator=g) * 1.2
    ctx = torch.randn(rows, 3, generator=g) if context else None
    gx, gld = torch.randn(rows, D, generator=g), torch.randn(rows, generator=g)
    ref = copy.deepcopy(layer).double()
    if rows:   # leave out the rows that sit on a ReLU kink of the conditioner (within 1e-5 of the median activation)
        with torch.no_grad():
            spec = layer_spec(ref)
            xk, _ = sampling_unrolled(spec, z.double(), ctx.double() if context else None)
            keep = relu_margin(spec, z.double(), xk, ctx.double() if context else None) > 1e-5
        z, gx, gld = z[keep], gx[keep], gld[keep]
        ctx = ctx[keep] if context else None
        assert keep.sum() >= 0.98 * rows
        rows = z.shape[0]
    zr = z.double().requires_grad_(True)
    cr = ctx.double().requires_grad_(True) if context else None
    xr, ldr = sampling_unrolled(layer_spec(ref), zr, cr)
    ((xr * gx.double()).sum() + (ldr * gld.double()).sum()).backward()
    layer = layer.cuda()
    zc = z.cuda().requires_grad_(True)
    cc = ctx.cuda().requires_grad_(True) if context else None
    x, ld = layer(zc, cc) if context else layer(zc)
    assert x.requires_grad and ld.requires_grad
    ((x * gx.cuda()).sum() + (ld * gld.cuda()).sum()).backward()
    assert x.shape == (rows, D) and ld.shape == (rows,)
    if rows:
        _close(x.detach(), xr.detach(), "x", 1e-4)
        _close(ld.detach(), ldr.detach(), "log_det", 1e-4)
    refp = dict(ref.named_parameters())
    for n, p in layer.named_parameters():
        assert p.grad is not None, n
        if rows == 0:
            assert (p.grad == 0).all(), n
        else:
            _close(p.grad, refp[n].grad, n)
    if rows:
        _close(zc.grad, zr.grad, "z")
        if context:
            _close(cc.grad, cr.grad, "context")


def package_loss(name, model, eps, ctx):
    model.q0.forward = R.replay_forward(model.q0, eps)
    n = eps.shape[0]
    if name in ("h", "k"):
        return model.reverse_kld(n)
    if name == "i":
        return model.reverse_kld(n, score_fn=False)
    if name == "j":
        return model.reverse_alpha_div(n, alpha=1, dreg=True)
    return model.reverse_kld(n, context=ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_model_gradients_match_reference_goldens(name):
    model, eps, ctx, gd = build_case(name)
    model = model.cuda()
    loss = package_loss(name, model, eps.cuda(), ctx.cuda() if ctx is not None else None)
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    # h / i: one of the 512 draws sits 1e-6 from a ReLU kink of a first block (a fixed golden cannot leave it out, see
    # test_layer_sampling_backward_matches_fp64_autograd): fp32 takes the other side there, which moves the gradients of
    # the initial layers and first blocks by up to 7e-3 of their scale; every other tensor is held to 2e-3
    kink = ("initial_layer.", "blocks.0.linear_layers.0.") if name in ("h", "i") else ()
    for n, p in model.named_parameters():
        assert p.grad is not None, f"{n} got no gradient"
        check_golden(p.grad, gd, n, 1e-2 if any(k in n for k in kink) else 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["h", "k", "l"])
def test_values_bit_identical_with_and_without_grad(name):
    model, eps, ctx, _ = build_case(name)
    model = model.cuda()
    args = (ctx.cuda(),) if ctx is not None else ()
    model.q0.forward = R.replay_forward(model.q0, eps.cuda())
    with torch.no_grad():
        a = model.sample(eps.shape[0], *args)
    b = model.sample(eps.shape[0], *args)
    assert b[0].requires_grad and b[1].requires_grad
    assert torch.equal(a[0], b[0].detach()) and torch.equal(a[1], b[1].detach())


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    model, eps, ctx, _ = build_case("h")
    model = model.cuda()
    loss = package_loss("h", model, eps.cuda(), None)
    with torch.no_grad():
        model.flows[0].mprqat.autoregressive_net.final_layer.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()


@pytest.mark.gpu
def test_no_context_gradient_formed_unless_wanted(monkeypatch):
    from normflows import _standalone
    seen = []
    for fn in ("ar_rqs_sampling_backward", "conditioner_backward"):
        real = getattr(_standalone, fn)

        def spy(*a, _real=real, **k):
            out = _real(*a, **k)
            seen.append(out[1])
            return out
        monkeypatch.setattr(_standalone, fn, spy)
    model, eps, ctx, _ = build_case("l")
    model = model.cuda()
    package_loss("l", model, eps.cuda(), ctx.cuda()).backward()
    assert len(seen) == 3 and all(g is None for g in seen)
    seen.clear()
    cc = ctx.cuda().requires_grad_(True)
    package_loss("l", model, eps.cuda(), cc).backward()
    assert len(seen) == 3 and all(g is not None for g in seen) and cc.grad is not None


@pytest.mark.gpu
def test_uniform_gaussian_log_prob_and_gradient():
    import normflows as nf
    scale = torch.tensor([1.5, 2 * math.pi, 0.7, 3.0])
    q0 = nf.distributions.UniformGaussian(4, [1, 3], scale).cuda()
    z = (torch.randn(1061, 4, generator=torch.Generator().manual_seed(5)) * 2).cuda().requires_grad_(True)
    lp = q0.log_prob(z)
    g = torch.randn(1061, generator=torch.Generator().manual_seed(6)).cuda()
    (lp * g).sum().backward()
    zr = z.detach().double().cpu().requires_grad_(True)
    qr = copy.deepcopy(q0).double().cpu()
    lr = base_log_prob(qr, zr)
    (lr * g.double().cpu()).sum().backward()
    _close(lp.detach(), lr.detach(), "log_prob", 1e-6)
    _close(z.grad, zr.grad, "z", 1e-6)
    zz, lq = q0(4096)
    assert zz.shape == (4096, 4) and (zz[:, [1, 3]].abs() <= scale[[1, 3]].cuda() / 2).all()
    _close(lq, base_log_prob(qr, zz.double().cpu()), "forward log_prob", 1e-6)


@pytest.mark.gpu
def test_stacks_without_a_differentiable_sampling_direction_still_raise():
    import normflows as nf
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    target = nf.distributions.TwoMoons()
    stacks = [
        [nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 32), nf.flows.LULinearPermute(2)],   # fused
        [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 32, [1]), nf.flows.LULinearPermute(2)],
        [nf.flows.MaskedAffineAutoregressive(2, 32), nf.flows.CircularCoupledRationalQuadraticSpline(2, 1, 32, [1])],
    ]
    for flows in stacks:
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, target).cuda()
        for call in (lambda: model.reverse_kld(64), lambda: model.reverse_alpha_div(64, dreg=True)):
            with pytest.raises(NotImplementedError, match=msg):
                call()
        with torch.no_grad():
            assert torch.isfinite(model.reverse_kld(64))
    model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2), [
        nf.flows.MaskedAffineAutoregressive(2, 32, context_features=4)], R.ContextTarget()).cuda()
    with pytest.raises(NotImplementedError, match=msg):
        model.reverse_kld(64, context=torch.zeros(64, 4, device="cuda"))


@pytest.mark.gpu
def test_paper_notebook_training_loop_trains_every_parameter():
    """examples/paper_example_nsf.ipynb's model and training cell, verbatim but for max_iter = 300 and no plotting:
    12 x CircularAutoregressiveRationalQuadraticSpline(2, 1, 512, [1], num_bins=10) on UniformGaussian,
    reverse_kld(2**14), Adam(5e-4) with cosine annealing."""
    import normflows as nf
    torch.manual_seed(0)
    target = R.gaussian_von_mises(nf.distributions.Target)
    base = nf.distributions.UniformGaussian(2, [1], torch.tensor([1., 2 * np.pi]))
    flow_layers = []
    for i in range(12):
        flow_layers += [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 512, [1], num_bins=10,
                                                                               tail_bound=torch.tensor([5., np.pi]),
                                                                               permute_mask=True)]
    model = nf.NormalizingFlow(base, flow_layers, target).cuda()
    start = {n: p.detach().clone() for n, p in model.named_parameters()}

    def dead_feature(n):   # the periodic weights of a feature with the last MADE degree feed no output (reference too)
        return n.endswith("preprocessing.weights") and not model.get_submodule(
            n[:-len("preprocessing.weights")] + "initial_layer").mask[:, 1].any()
    max_iter, num_samples = 300, 2 ** 14
    optimizer = torch.optim.Adam(model.parameters(), lr=5e-4)
    scheduler = torch.optim.lr_scheduler.CosineAnnealingLR(optimizer, max_iter)
    loss_hist = []
    for it in range(max_iter):
        optimizer.zero_grad()
        loss = model.reverse_kld(num_samples)
        if ~(torch.isnan(loss) | torch.isinf(loss)):
            loss.backward()
            if it == max_iter - 1:   # (at the identity init only the final layers have a gradient)
                for n, p in model.named_parameters():
                    assert p.grad is not None and torch.isfinite(p.grad).all(), n
                    assert (p.grad.abs().max() > 0) != dead_feature(n), n
            optimizer.step()
        loss_hist.append(loss.item())
        scheduler.step()
    first, last = np.mean(loss_hist[:20]), np.mean(loss_hist[-20:])
    assert np.isfinite(last) and last < first - 0.05, (first, last)
    for n, p in model.named_parameters():
        if dead_feature(n):
            continue
        assert not torch.equal(p.detach(), start[n]), f"{n} did not move"
