"""Forward-KL training of affine-coupling flows (examples/real_nvp_colab.ipynb, the first model of
change_base_distribution.ipynb, the ActNorms of residual.ipynb): gradients through the density direction of the affine
family -- MaskedAffineFlow, AffineConstFlow / ActNorm, AffineCouplingBlock, Permute -- which runs as one
affine_stack_kernel launch (direction 0) and is differentiated by affine_density_bwd_rows_kernel + the fixed-order
weight reduction: nfb_flow_density_backward for a stack or a layer on its own, and inside nfb_flow_log_prob_backward for
affine groups anywhere in a stack.

Per-op density adjoints (csrc/nfb_affine_bwd.cuh), row cotangents g of the output and gam of the log-det:
    MaskedAffineFlow   s_hat = -(1-b)(g (z-t) e^-s + gam),  t_hat = -(1-b) g e^-s,  g_z = (b + (1-b) e^-s) g + b J^T (...)
    AffineConstFlow    g_z = g e^-s,  g_s = -sum_rows (g (z-t) e^-s + gam),  g_t = -sum_rows g e^-s
    AffineCouplingBlock  exp: x2 = (v - shift) e^-sc;  sigmoid: (v - shift) sg;  sigmoid_inv: (v - shift) / sg
    Permute            g_z[i] = g[fwd[i]]

CPU: the element adjoints, compiled for the host, against fp64 autograd and central differences (non-finite s / t
included); an fp64 restatement of forward_kld against the reference's goldens.
GPU: log_prob / inverse_and_log_det / the layer loop against fp64 autograd over the sampling tests' shape grid, the
goldens, zero rows and several workspace chunks, bit-identical values and gradients, the in-place refusal, a launch count
independent of depth, shared parameters, no use of the torch restatement, and the real_nvp_colab training cell."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT
from test_affine_rkl_training import _close, _randomise, make_stack, real_nvp


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- element adjoints on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def adjlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "affine_density_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "affine_density_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_adjoint(lib, op, a, b, c, d, g, gam, scale=1, smap=0, use_float=0):
    f = lambda v: np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
    a, b, c, d, g, gam = (f(v) for v in (a, b, c, d, g, gam))
    n = a.size
    outs = [np.empty(n) for _ in range(3)]
    P = lambda v: v.ctypes.data_as(C.c_void_p)
    lib.affine_density_adjoint_check(C.c_int(op), C.c_int(scale), C.c_int(smap), C.c_int(n), C.c_int(use_float),
                                     P(a), P(b), P(c), P(d), P(g), P(gam), *[P(o) for o in outs])
    return outs


def _vjp(fn, inputs, g, gam):
    """fp64 autograd of sum(g * x + gam * ld) for (x, ld) = fn(*inputs), elementwise."""
    xs = [torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in inputs]
    x, ld = fn(*xs)
    (torch.as_tensor(g) * x + torch.as_tensor(gam) * ld).sum().backward()
    return [v.grad.numpy() for v in xs]


def masked_elem(z, b, s, t):
    nan = torch.tensor(float("nan"), dtype=z.dtype)
    s, t = torch.where(torch.isfinite(s), s, nan), torch.where(torch.isfinite(t), t, nan)
    return b * z + (1 - b) * (z - t) * torch.exp(-s), -(1 - b) * s


def coupling_elem(scale, smap):
    def fn(v, shift, sc):
        if not scale:
            return v - shift, 0 * sc
        if smap == 0:
            return (v - shift) * torch.exp(-sc), -sc
        sg = torch.sigmoid(sc + 2)
        return ((v - shift) * sg, torch.log(sg)) if smap == 1 else ((v - shift) / sg, -torch.log(sg))
    return fn


def _fd(fn, args, k, g, gam, h=1e-6):
    hi = [torch.tensor(a + (h if i == k else 0)) for i, a in enumerate(args)]
    lo = [torch.tensor(a - (h if i == k else 0)) for i, a in enumerate(args)]
    L = lambda xs: (lambda x, ld: g * x.numpy() + gam * ld.numpy())(*fn(*xs))
    return (L(hi) - L(lo)) / (2 * h)


def test_masked_density_element_matches_autograd_and_central_differences(adjlib):
    rng = np.random.default_rng(10)
    n = 400
    z, s, t, g, gam = (rng.normal(size=n) for _ in range(5))
    b = (rng.random(n) < 0.5).astype(np.float64)
    sh, th, gz = host_adjoint(adjlib, 0, z, b, s, t, g, gam)
    gz_a, _, gs_a, gt_a = _vjp(masked_elem, [z, b, s, t], g, gam)
    np.testing.assert_allclose(gz, gz_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(sh, gs_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(th, gt_a, rtol=1e-12, atol=1e-12)
    for k, got in ((0, gz), (2, sh), (3, th)):
        np.testing.assert_allclose(got, _fd(masked_elem, [z, b, s, t], k, g, gam), rtol=1e-6, atol=1e-6)
    f32 = host_adjoint(adjlib, 0, z, b, s, t, g, gam, use_float=1)
    for a, r in zip(f32, (sh, th, gz)):
        np.testing.assert_allclose(a, r, rtol=1e-5, atol=1e-5)


def test_masked_density_element_non_finite_s_or_t_passes_no_gradient_to_the_nets(adjlib):
    z = np.array([0.5, -1.0, 2.0, 0.3, 0.7])
    b = np.array([0.0, 0.0, 1.0, 0.0, 0.0])
    s = np.array([np.inf, 0.2, np.nan, 0.1, -np.inf])
    t = np.array([0.1, -np.inf, 0.3, np.nan, 0.2])
    g, gam = np.ones(5), np.full(5, 0.5)
    sh, th, gz = host_adjoint(adjlib, 0, z, b, s, t, g, gam)
    assert sh[0] == 0 and sh[2] == 0 and sh[4] == 0 and th[1] == 0 and th[3] == 0
    gz_a, _, gs_a, gt_a = _vjp(masked_elem, [z, b, s, t], g, gam)
    np.testing.assert_array_equal(np.isnan(gz), np.isnan(gz_a))
    np.testing.assert_allclose(sh, gs_a, rtol=1e-12, equal_nan=True)
    np.testing.assert_allclose(th, gt_a, rtol=1e-12, equal_nan=True)


def test_const_density_element_matches_autograd_and_central_differences(adjlib):
    rng = np.random.default_rng(11)
    z, s, t, g, gam = (rng.normal(size=300) for _ in range(5))
    gz, cs, ct = host_adjoint(adjlib, 1, z, z, s, t, g, gam)
    fn = lambda z, s, t: ((z - t) * torch.exp(-s), -s)
    gz_a, gs_a, gt_a = _vjp(fn, [z, s, t], g, gam)
    for a, r in ((gz, gz_a), (cs, gs_a), (ct, gt_a)):
        np.testing.assert_allclose(a, r, rtol=1e-12, atol=1e-12)
    for k, got in ((0, gz), (1, cs), (2, ct)):
        np.testing.assert_allclose(got, _fd(fn, [z, s, t], k, g, gam), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("scale,smap", [(1, 0), (1, 1), (1, 2), (0, 0)])
def test_coupling_density_element_matches_autograd_and_central_differences(adjlib, scale, smap):
    rng = np.random.default_rng(20 + smap + 3 * scale)
    n = 300
    v, shift, g, gam = (rng.normal(size=n) for _ in range(4))
    sc = rng.normal(size=n) * 3
    sc[:4] = [60.0, -60.0, 300.0, -300.0]   # saturated sigmoid: exact limits, no inf * 0
    gv, gsh, gsc = host_adjoint(adjlib, 2, v, shift, sc, sc, g, gam, scale=scale, smap=smap)
    if smap == 1:
        assert np.isfinite(gv).all() and np.isfinite(gsc).all()
    fn = coupling_elem(scale, smap)
    gv_a, gsh_a, gsc_a = _vjp(fn, [v, shift, sc], g, gam)
    ok = slice(4, None)
    np.testing.assert_allclose(gv[ok], gv_a[ok], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gsh[ok], gsh_a[ok], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gsc[ok], gsc_a[ok], rtol=1e-10, atol=1e-12)
    for k, got in ((0, gv), (1, gsh), (2, gsc)):
        np.testing.assert_allclose(got[ok], _fd(fn, [v, shift, sc], k, g, gam)[ok], rtol=1e-5, atol=1e-6)


# ---- goldens: fp64 autograd of the reference's forward_kld (tests/golden/make_affine_fkl_grads.py) --------------------
def build_golden_case(name):
    """The case built by this package (on the CPU) with the golden's parameters and buffers."""
    import helpers_affine_fkl as A
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_fkl_{name}.npz"))
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    model = A.build(nf, name)
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    model.load_state_dict({k: sd[k].to(v.dtype) for k, v in own.items()})
    x = torch.tensor(gd["x"])
    ctx = torch.tensor(gd["context"]) if "context" in gd else None
    return model, x, ctx, gd


def restated_fkl(model, x, ctx):
    """forward_kld (core.py:40-53, 246-258) in fp64 torch: each layer's density direction by _autograd.layer_inverse,
    the context spline layer of case cond by test_reverse_kld_training's density restatement."""
    from normflows._autograd import layer_inverse
    from normflows.flows import neural_spline as ns
    from test_reverse_kld_training import base_log_prob, density_ar
    z, lq = x, x.new_zeros(x.shape[0])
    for f in reversed(list(model.flows)):
        ar_ctx = ctx is not None and isinstance(f, ns.AutoregressiveRationalQuadraticSpline)
        z, ld = density_ar(f, z, ctx) if ar_ctx else layer_inverse(f, z)
        lq = lq + ld
    return -torch.mean(lq + base_log_prob(model.q0, z))


def check_golden(got, gd, name, tol):
    from test_maf_training import check_golden as check
    check(got, gd, name, tol)


GOLDEN_CASES = ["colab", "realnvp", "every", "mixed", "cond"]


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_fp64_restatement_matches_reference_goldens(name):
    """The restated density direction and loss give the reference's fp64 autograd gradients to 1e-10 of each scale."""
    model, x, ctx, gd = build_golden_case(name)
    model = model.double()
    loss = restated_fkl(model, x.double(), ctx.double() if ctx is not None else None)
    loss.backward()
    # (the reference sums log_q into a float32 buffer, core.py:47-52)
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    minted = {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))}
    assert minted == set(names), minted ^ set(names)
    for n, p in model.named_parameters():
        check_golden(p.grad, gd, n, 1e-10)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_model_gradients_match_reference_goldens(name):
    model, x, ctx, gd = build_golden_case(name)
    model = model.cuda()
    loss = model.forward_kld(x.cuda(), context=ctx.cuda()) if ctx is not None else model.forward_kld(x.cuda())
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None, f"{n} got no gradient"
            check_golden(p.grad, gd, n, 2e-3)


# ---- GPU: the stack against fp64 autograd of a torch restatement of the density direction --------------------------
def _mlp64(net, x, P, slope, margins=None):
    """The MLP on the leaves P; appends each row's smallest |pre-activation| of a LeakyReLU to `margins` if given."""
    lins = net.linear_layers()
    for i, lin in enumerate(lins):
        x = F.linear(x, P[id(lin.weight)], P[id(lin.bias)])
        if i + 1 < len(lins):
            if margins is not None:
                margins.append(x.detach().abs().min(1).values)
            x = F.leaky_relu(x, slope)
    return x


def density_restated(layers, x, P, margins=None):
    """fp64 (z, log_det) of the layers' density direction (ops last-to-first); P maps id(parameter) -> its fp64 leaf."""
    from normflows.flows import affine, mixing
    _mlp = lambda net, v, slope: _mlp64(net, v, P, slope, margins)
    ld = x.new_zeros(x.shape[0])
    z = x
    for layer in reversed(list(layers)):
        if isinstance(layer, affine.MaskedAffineFlow):
            b = layer.b.to(x.dtype)
            zm = b * z
            s = _mlp(layer.s, zm, layer.s.leaky) if layer.s is not None else torch.zeros_like(z)
            t = _mlp(layer.t, zm, layer.t.leaky) if layer.t is not None else torch.zeros_like(z)
            nan = torch.tensor(float("nan"), dtype=z.dtype, device=z.device)
            s, t = torch.where(torch.isfinite(s), s, nan), torch.where(torch.isfinite(t), t, nan)
            z = zm + (1 - b) * (z - t) * torch.exp(-s)
            ld = ld - torch.sum((1 - b) * s, 1)
        elif isinstance(layer, affine.AffineConstFlow):
            s = P.get(id(layer.s), layer.s.to(x.dtype)).reshape(1, -1)
            t = P.get(id(layer.t), layer.t.to(x.dtype)).reshape(1, -1)
            z = (z - t) * torch.exp(-s)
            ld = ld - torch.sum(s)
        elif isinstance(layer, affine.AffineCouplingBlock):
            a, c = z.chunk(2, dim=1)
            z1, z2 = (a, c) if layer.split_mode == "channel" else (c, a)
            pm = layer.flows[1].param_map
            param = _mlp(pm, z1, pm.leaky)
            if not layer.scale:
                z2 = z2 - param
            else:
                shift, sc = param[:, 0::2], param[:, 1::2]
                if layer.scale_map == "exp":
                    z2, ld = (z2 - shift) * torch.exp(-sc), ld - sc.sum(1)
                else:
                    sg = torch.sigmoid(sc + 2)
                    if layer.scale_map == "sigmoid":
                        z2, ld = (z2 - shift) * sg, ld + torch.log(sg).sum(1)
                    else:
                        z2, ld = (z2 - shift) / sg, ld - torch.log(sg).sum(1)
            z = torch.cat([z1, z2] if layer.split_mode == "channel" else [z2, z1], 1)
        else:
            assert isinstance(layer, mixing.Permute)
            _, inv = layer._index_lists()
            z = z[:, torch.tensor(inv, device=z.device)]
    return z, ld


def _run(model, x, gz, gld, mode):
    """The loss sum(gz * z + gld * log_det) of the density direction, by `mode`: log_prob (gz unused: the base's
    log-density is part of the output), inverse_and_log_det, or the layer loop (each layer's inverse on its own)."""
    if mode == "log_prob":
        lq = model.log_prob(x)
        return lq, (lq * gld).sum()
    if mode == "inverse":
        z, ld = model.inverse_and_log_det(x)
    else:
        z, ld = x, torch.zeros(x.shape[0], device=x.device)
        for f in reversed(list(model.flows)):
            z, l = f.inverse(z)
            ld = ld + l
    return (z, ld), (z * gz).sum() + (ld * gld).sum()


def check_density_gradients(flows, D, rows, seed, mode="log_prob", kink=0.0):
    """kink > 0: rows with a LeakyReLU pre-activation within `kink` of 0 (in fp64) get zero cotangents.  There the
    float32 recompute may take the other side of the kink than fp64 does, which moves that row's contribution to the
    unit's weights by O(1); at 13 000 rows of the widest, deepest stack a few rows come within 1e-8."""
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows).cuda()
    _randomise(model.q0, seed + 77, 0.3)
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(rows, D, generator=g).cuda()
    gz = torch.randn(rows, D, generator=g).cuda()
    gld = torch.randn(rows, generator=g).cuda()
    if kink > 0:
        margins = []
        with torch.no_grad():
            density_restated(model.flows, x0.double(), {id(p): p.double() for p in model.parameters()}, margins)
        near = torch.stack(margins).min(0).values < kink
        gz[near], gld[near] = 0.0, 0.0
    x = x0.clone().requires_grad_(True)
    out, loss = _run(model, x, gz, gld, mode)
    loss.backward()
    params = list(model.parameters())
    P = {id(p): p.detach().double().requires_grad_(True) for p in params}
    xd = x0.double().requires_grad_(True)
    zr, ldr = density_restated(model.flows, xd, P)
    if mode == "log_prob":
        ls, loc = P[id(model.q0.log_scale)].reshape(-1), P[id(model.q0.loc)].reshape(-1)
        lqr = ldr - 0.5 * D * np.log(2 * np.pi) - ls.sum() - 0.5 * (((zr - loc) / torch.exp(ls)) ** 2).sum(1)
        (lqr * gld.double()).sum().backward()
        _close(out.detach(), lqr.detach(), "log_q", 1e-4)
    else:
        ((zr * gz.double()).sum() + (ldr * gld.double()).sum()).backward()
        _close(out[0].detach(), zr.detach(), "z", 1e-4)
        _close(out[1].detach(), ldr.detach(), "log_det", 1e-4)
    _close(x.grad, xd.grad, "g_x")
    for n, p in model.named_parameters():
        if mode != "log_prob" and n.startswith("q0."):
            continue
        assert p.grad is not None, n
        _close(p.grad, P[id(p)].grad, n)
    return model


GRID = [(1, 8, 2, 0.0, 129), (2, 4, 2, 0.0, 127), (2, 32, 3, 0.2, 5000), (5, 16, 2, 0.2, 128), (5, 128, 6, 0.0, 129),
        (16, 64, 3, 0.0, 1), (16, 128, 2, 0.2, 1000), (5, 8, 1, 0.0, 128)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["log_prob", "inverse"])
@pytest.mark.parametrize("D,width,n_lin,slope,rows", GRID)
def test_stack_density_backward_matches_fp64_autograd(D, width, n_lin, slope, rows, mode):
    check_density_gradients(make_stack(D, width, n_lin, slope, seed=D + n_lin), D, rows, seed=rows, mode=mode)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 5])
def test_layer_loop_density_backward_matches_fp64_autograd(D):
    """Each NativeFlow's inverse called on its own under grad (LayerInverseFn) goes through nfb_flow_density_backward."""
    check_density_gradients(make_stack(D, 16, 2, 0.2, seed=7), D, 300, seed=3, mode="layer")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["log_prob", "inverse", "layer"])
def test_zero_rows_give_zero_gradients(mode):
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 16, 2, 0.0, seed=1)).cuda()
    x = torch.zeros(0, 5, device="cuda", requires_grad=True)
    _, loss = _run(model, x, torch.zeros(0, 5, device="cuda"), torch.zeros(0, device="cuda"), mode)
    loss.backward()
    for n, p in model.flows.named_parameters():
        assert p.grad is not None and (p.grad == 0).all(), n


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["log_prob", "inverse"])
def test_rows_beyond_one_workspace_chunk(mode):
    """Wide, deep nets at 13 000 rows need three workspace chunks: the chunk offsets and the cross-chunk accumulation
    of the weight gradients against fp64 autograd (rows next to a ReLU kink left out, see check_density_gradients)."""
    model = check_density_gradients(make_stack(16, 128, 6, 0.0, seed=22), 16, 13000, seed=5, mode=mode, kink=1e-5)
    assert model._stack().launch_count() >= 6   # 3 launches per chunk


@pytest.mark.gpu
def test_values_bit_identical_with_and_without_grad_and_reproducible_gradients():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 32, 3, 0.2, seed=4)).cuda()
    x = torch.randn(777, 5, device="cuda")
    with torch.no_grad():
        z0, l0 = model.inverse_and_log_det(x)
        q0 = model.log_prob(x)
    grads = []
    for _ in range(2):
        model.zero_grad()
        z, ld = model.inverse_and_log_det(x.clone().requires_grad_(True))
        assert torch.equal(z, z0) and torch.equal(ld, l0)
        lq = model.log_prob(x.clone().requires_grad_(True))
        assert torch.equal(lq, q0)
        (z.square().sum() + ld.sum() + lq.sum()).backward()
        grads.append([p.grad.clone() for p in model.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)
    layer = model.flows[0]
    with torch.no_grad():
        y0, m0 = layer.inverse(x)
    y, m = layer.inverse(x.clone().requires_grad_(True))
    assert torch.equal(y, y0) and torch.equal(m, m0)


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 16, 2, 0.0, seed=2)).cuda()
    z, ld = model.inverse_and_log_det(torch.randn(64, 5, device="cuda"))
    y, m = model.flows[0].inverse(torch.randn(64, 5, device="cuda", requires_grad=True))
    with torch.no_grad():
        model.flows[0].s.net[0].weight.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        (z.sum() + ld.sum()).backward()
    with pytest.raises(RuntimeError, match="modified in place"):
        (y.sum() + m.sum()).backward()


def _fresh_real_nvp(K):
    torch.manual_seed(0)
    model = real_nvp(K)
    for f in model.flows:
        if hasattr(f, "_mark_done"):
            f._mark_done()
    _randomise(model.flows, K)
    return model.cuda()


@pytest.mark.gpu
def test_launch_count_does_not_depend_on_depth():
    counts = []
    for K in (4, 64):
        model = _fresh_real_nvp(K)
        z, ld = model.inverse_and_log_det(torch.randn(20, 2, device="cuda"))
        (z.sum() + ld.sum()).backward()
        n_inverse = model._stack().launch_count()
        model.log_prob(torch.randn(20, 2, device="cuda")).sum().backward()
        counts.append((n_inverse, model._stack().launch_count()))
    assert counts[0] == counts[1] and counts[0][0] <= 3, counts


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["log_prob", "inverse", "layer"])
def test_a_parameter_shared_by_two_layers_gets_the_sum_of_its_gradients(mode):
    import normflows as nf
    b = torch.tensor([1.0, 0.0])
    s, t = nf.nets.MLP([2, 8, 2], leaky=0.2), nf.nets.MLP([2, 8, 2])
    _randomise(s, 1), _randomise(t, 2)
    check_density_gradients([nf.flows.MaskedAffineFlow(b, t, s), nf.flows.MaskedAffineFlow(1 - b, t, s)], 2, 300,
                            seed=9, mode=mode)
    act = nf.flows.AffineConstFlow(2)
    _randomise(act, 3)
    check_density_gradients([act, nf.flows.Permute(2, "swap"), act], 2, 300, seed=10, mode=mode)


@pytest.mark.gpu
def test_the_torch_restatement_is_not_reached(monkeypatch):
    """All-affine, mixed (affine groups between spline / LU groups) and per-layer backward run on the native kernels."""
    import normflows as nf
    import normflows._autograd as AG

    def refuse(*a, **k):
        raise AssertionError("the torch restatement was reached")
    all_affine = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 16, 2, 0.2, seed=3)).cuda()
    mixed, x, _, _ = build_golden_case("mixed")
    mixed = mixed.cuda()
    monkeypatch.setattr(AG, "layer_inverse", refuse)
    for model, D in ((all_affine, 5), (mixed, 2)):
        model.forward_kld(torch.randn(300, D, device="cuda")).backward()
        for n, p in model.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), n
    x = torch.randn(300, 2, device="cuda", requires_grad=True)
    z, ld = mixed.flows[0].inverse(x)
    z, l2 = mixed.flows[1].inverse(z)
    (z.sum() + ld.sum() + l2.sum()).backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()


@pytest.mark.gpu
def test_real_nvp_colab_training_cell_trains():
    """examples/real_nvp_colab.ipynb's training cell, 150 of its 4 000 iterations."""
    import helpers_affine_fkl as A
    import normflows as nf
    torch.manual_seed(0)
    model = A.colab(nf).cuda()
    target = nf.distributions.TwoMoons()
    optimizer = torch.optim.Adam(model.parameters(), lr=5e-4, weight_decay=1e-5)
    start = {n: p.detach().clone() for n, p in model.named_parameters()}
    hist = []
    for it in range(150):
        optimizer.zero_grad()
        x = target.sample(2 ** 9).cuda()
        loss = model.forward_kld(x)
        if ~(torch.isnan(loss) | torch.isinf(loss)):
            loss.backward()
            if it == 149:
                for n, p in model.named_parameters():
                    assert p.grad is not None and torch.isfinite(p.grad).all(), n
            optimizer.step()
        hist.append(loss.item())
    h = np.array(hist)
    assert np.isfinite(h).all() and h[:10].mean() > h[-10:].mean() + 0.1, (h[:10].mean(), h[-10:].mean())
    for n, p in model.named_parameters():
        assert torch.isfinite(p).all() and not torch.equal(p.detach(), start[n]), n
