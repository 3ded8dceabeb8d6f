"""Reverse-KL training of Real NVP flows (examples/real_nvp.ipynb, examples/augmented_flow.ipynb): gradients through the
sampling direction of the affine family -- MaskedAffineFlow, AffineConstFlow / ActNorm, AffineCouplingBlock, Permute --
which runs as one affine_stack_kernel launch and is differentiated by one nfb_flow_sampling_backward call.

Per-op adjoints (csrc/nfb_affine_bwd.cuh), row cotangents g of the output and gam of the log-det:
    MaskedAffineFlow   s_hat = (1-b)(g z e^s + gam),  t_hat = (1-b) g,  g_z = (b + (1-b) e^s) g + b (J_S^T s_hat + J_T^T t_hat)
    AffineConstFlow    g_z = g e^s,  g_s = sum_rows (g z e^s + gam),  g_t = sum_rows g
    AffineCouplingBlock  exp: x2 = z2 e^sc + shift;  sigmoid: z2 / sig(sc + 2) + shift;  sigmoid_inv: z2 sig(sc + 2) + shift
    Permute            gather with the inverse index list

CPU: the element adjoints, compiled for the host, against fp64 autograd and central differences (including non-finite s
and t); TwoModes / TwoIndependent against the reference's values and state_dict keys.
GPU: stacks of every op variant against fp64 autograd of a torch restatement of the sampling direction, bit-identical
values with and without grad, the in-place refusal, reproducible gradients, a launch count independent of depth, the
reverse_kld gating, and the two notebooks' training cells."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import ROOT


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- element adjoints on the host ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def adjlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "affine_adjoint_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "affine_adjoint_host_check.cu")])
    return C.CDLL(so)


def host_adjoint(lib, op, a, b, c, d, g, gam, scale=1, smap=0, use_float=0):
    f = lambda v: np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
    a, b, c, d, g, gam = (f(v) for v in (a, b, c, d, g, gam))
    n = a.size
    outs = [np.empty(n) for _ in range(3)]
    P = lambda v: v.ctypes.data_as(C.c_void_p)
    lib.affine_adjoint_check(C.c_int(op), C.c_int(scale), C.c_int(smap), C.c_int(n), C.c_int(use_float),
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
    return b * z + (1 - b) * (z * torch.exp(s) + t), (1 - b) * s


def coupling_elem(scale, smap):
    def fn(v, shift, sc):
        if not scale:
            return v + shift, 0 * sc
        if smap == 0:
            return v * torch.exp(sc) + shift, sc
        sg = torch.sigmoid(sc + 2)
        return (v / sg + shift, -torch.log(sg)) if smap == 1 else (v * sg + shift, torch.log(sg))
    return fn


def test_masked_element_matches_autograd_and_central_differences(adjlib):
    rng = np.random.default_rng(0)
    n = 400
    z, s, t, g, gam = (rng.normal(size=n) for _ in range(5))
    b = (rng.random(n) < 0.5).astype(np.float64)
    sh, th, gz = host_adjoint(adjlib, 0, z, b, s, t, g, gam)
    gz_a, _, gs_a, gt_a = _vjp(masked_elem, [z, b, s, t], g, gam)
    # the direct part of g_z is the elementwise derivative; the MLP part (b J^T ...) is the autograd of s, t
    np.testing.assert_allclose(gz, gz_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(sh, gs_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(th, gt_a, rtol=1e-12, atol=1e-12)
    h = 1e-6
    for k, v in ((0, z), (2, s), (3, t)):
        args = [z, b, s, t]
        hi = [torch.tensor(a + (h if i == k else 0)) for i, a in enumerate(args)]
        lo = [torch.tensor(a - (h if i == k else 0)) for i, a in enumerate(args)]
        L = lambda xs: (lambda x, ld: (g * x.numpy() + gam * ld.numpy()))(*masked_elem(*xs))
        fd = (L(hi) - L(lo)) / (2 * h)
        np.testing.assert_allclose({0: gz, 2: sh, 3: th}[k], fd, rtol=1e-6, atol=1e-6)
    f32 = host_adjoint(adjlib, 0, z, b, s, t, g, gam, use_float=1)
    for a, r in zip(f32, (sh, th, gz)):
        np.testing.assert_allclose(a, r, rtol=1e-5, atol=1e-5)


def test_masked_element_non_finite_s_or_t_passes_no_gradient_to_the_nets(adjlib):
    z = np.array([0.5, -1.0, 2.0, 0.3])
    b = np.array([0.0, 0.0, 1.0, 0.0])
    s = np.array([np.inf, 0.2, np.nan, 0.1])
    t = np.array([0.1, -np.inf, 0.3, np.nan])
    g, gam = np.ones(4), np.full(4, 0.5)
    sh, th, gz = host_adjoint(adjlib, 0, z, b, s, t, g, gam)
    assert sh[0] == 0 and sh[2] == 0 and th[1] == 0 and th[3] == 0
    assert sh[1] != 0 and th[0] != 0
    gz_a, _, gs_a, gt_a = _vjp(masked_elem, [z, b, s, t], g, gam)
    np.testing.assert_array_equal(np.isnan(gz), np.isnan(gz_a))
    np.testing.assert_allclose(sh, gs_a, rtol=1e-12, equal_nan=True)
    np.testing.assert_allclose(th, gt_a, rtol=1e-12, equal_nan=True)


def test_const_element_matches_autograd(adjlib):
    rng = np.random.default_rng(1)
    z, s, g, gam = (rng.normal(size=300) for _ in range(4))
    gz, cs, ct = host_adjoint(adjlib, 1, z, z, s, s, g, gam)
    gz_a, gs_a, gt_a = _vjp(lambda z, s, t: (z * torch.exp(s) + t, s), [z, s, np.zeros_like(z)], g, gam)
    for a, r in ((gz, gz_a), (cs, gs_a), (ct, gt_a)):
        np.testing.assert_allclose(a, r, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("scale,smap", [(1, 0), (1, 1), (1, 2), (0, 0)])
def test_coupling_element_matches_autograd_and_central_differences(adjlib, scale, smap):
    rng = np.random.default_rng(2 + smap + 3 * scale)
    n = 300
    v, shift, g, gam = (rng.normal(size=n) for _ in range(4))
    sc = rng.normal(size=n) * 3
    sc[:4] = [60.0, -60.0, 300.0, -300.0]   # saturated sigmoid: exact limits, no inf * 0
    gv, gsh, gsc = host_adjoint(adjlib, 2, v, v, sc, sc, g, gam, scale=scale, smap=smap)
    assert np.isfinite(gv[4:]).all() and np.isfinite(gsc).all() if smap != 0 else True
    fn = coupling_elem(scale, smap)
    gv_a, gsh_a, gsc_a = _vjp(fn, [v, shift, sc], g, gam)
    ok = slice(4, None)
    np.testing.assert_allclose(gv[ok], gv_a[ok], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gsh, gsh_a, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(gsc[ok], gsc_a[ok], rtol=1e-10, atol=1e-12)
    h = 1e-6
    L = lambda vv, ss: (lambda x, ld: g * x.numpy() + gam * ld.numpy())(*fn(torch.tensor(vv), torch.tensor(shift),
                                                                            torch.tensor(ss)))
    np.testing.assert_allclose(gsc[ok], ((L(v, sc + h) - L(v, sc - h)) / (2 * h))[ok], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(gv[ok], ((L(v + h, sc) - L(v - h, sc)) / (2 * h))[ok], rtol=1e-5, atol=1e-6)


# ---- targets -------------------------------------------------------------------------------------------------------
# log_prob of the reference (normflows/distributions/prior.py TwoModes, target.py TwoIndependent) at fixed points
PTS = np.array([[0.0, 0.0], [2.0, 0.0], [-1.9, 0.3], [0.5, -2.2], [3.0, 1.0]])


def twomodes_formula(z, loc, scale):
    a = np.abs(z[:, 0])
    return (-0.5 * ((np.linalg.norm(z, axis=1) - loc) / (2 * scale)) ** 2 - 0.5 * ((a - abs(loc)) / (3 * scale)) ** 2
            + np.log(1 + np.exp(-2 * a * abs(loc) / (3 * scale) ** 2)))


def test_two_modes_log_prob_matches_the_reference_formula():
    import normflows as nf
    for loc, scale in ((2.0, 0.1), (1.5, 0.4), (-1.0, 0.3)):
        got = nf.distributions.TwoModes(loc, scale).log_prob(torch.tensor(PTS, dtype=torch.float64)).numpy()
        np.testing.assert_allclose(got, twomodes_formula(PTS, loc, scale), rtol=1e-13)


def test_two_independent_state_dict_matches_the_reference():
    import normflows as nf
    t = nf.distributions.TwoIndependent(nf.distributions.TwoMoons(), nf.distributions.DiagGaussian(2))
    assert list(t.state_dict().keys()) == ['prop_scale', 'prop_shift', 'target1.prop_scale', 'target1.prop_shift',
                                           'target2.loc', 'target2.log_scale']
    assert isinstance(t, nf.distributions.Target)
    assert {n for n, _ in t.named_parameters()} == {"target2.loc", "target2.log_scale"}
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(4), [nf.flows.ActNorm(4)], t)
    assert any(p is t.target2.loc for p in model.parameters())


# ---- GPU: the stack against fp64 autograd of a torch restatement of the sampling direction --------------------------
def _mlp64(net, x, P, slope):
    lins = net.linear_layers()
    for i, lin in enumerate(lins):
        x = F.linear(x, P[id(lin.weight)], P[id(lin.bias)])
        if i + 1 < len(lins):
            x = F.leaky_relu(x, slope)
    return x


def sample_restated(layers, z, P):
    """fp64 (x, log_det) of the layers' sampling direction; P maps id(parameter) -> its fp64 leaf."""
    from normflows.flows import affine, mixing
    ld = z.new_zeros(z.shape[0])
    for layer in layers:
        if isinstance(layer, affine.MaskedAffineFlow):
            b = layer.b.double()
            zm = b * z
            s = _mlp64(layer.s, zm, P, layer.s.leaky) if layer.s is not None else torch.zeros_like(z)
            t = _mlp64(layer.t, zm, P, layer.t.leaky) if layer.t is not None else torch.zeros_like(z)
            nan = torch.tensor(float("nan"), dtype=z.dtype, device=z.device)
            s, t = torch.where(torch.isfinite(s), s, nan), torch.where(torch.isfinite(t), t, nan)
            z = zm + (1 - b) * (z * torch.exp(s) + t)
            ld = ld + torch.sum((1 - b) * s, 1)
        elif isinstance(layer, affine.AffineConstFlow):
            s = P.get(id(layer.s), layer.s.double()).reshape(1, -1)
            t = P.get(id(layer.t), layer.t.double()).reshape(1, -1)
            z = z * torch.exp(s) + t
            ld = ld + torch.sum(s)
        elif isinstance(layer, affine.AffineCouplingBlock):
            a, c = z.chunk(2, dim=1)
            z1, z2 = (a, c) if layer.split_mode == "channel" else (c, a)
            pm = layer.flows[1].param_map
            param = _mlp64(pm, z1, P, pm.leaky)
            if not layer.scale:
                z2 = z2 + param
            else:
                shift, sc = param[:, 0::2], param[:, 1::2]
                if layer.scale_map == "exp":
                    z2, ld = z2 * torch.exp(sc) + shift, ld + sc.sum(1)
                else:
                    sg = torch.sigmoid(sc + 2)
                    if layer.scale_map == "sigmoid":
                        z2, ld = z2 / sg + shift, ld - torch.log(sg).sum(1)
                    else:
                        z2, ld = z2 * sg + shift, ld + torch.log(sg).sum(1)
            z = torch.cat([z1, z2] if layer.split_mode == "channel" else [z2, z1], 1)
        else:
            assert isinstance(layer, mixing.Permute)
            fwd, _ = layer._index_lists()
            z = z[:, torch.tensor(fwd, device=z.device)]
    return z, ld


def _randomise(module, seed, sigma=0.3):
    """Weights ~ N(0, (sigma / sqrt(fan_in))^2), every other parameter ~ N(0, (sigma / 3)^2): off the identity init,
    but tame enough that a deep stack stays finite in float32."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            sd = sigma / math.sqrt(p.shape[1]) if p.dim() == 2 and p.shape[0] > 1 else sigma / 3
            p.copy_(torch.randn(p.shape, generator=g) * sd)


def make_stack(D, width, n_lin, slope, seed):
    """Every op variant at dimension D: MaskedAffineFlow with both nets / s only / t only, ActNorm (initialised), an
    AffineConstFlow with s as a buffer, AffineCouplingBlocks over every scale map, no scale and channel_inv, Permute
    shuffle and swap."""
    import normflows as nf
    torch.manual_seed(seed)
    sizes = lambda i, o: [i] + [width] * (n_lin - 1) + [o]
    mlp = lambda i, o: nf.nets.MLP(sizes(i, o), leaky=slope)
    b = torch.tensor([float(j % 2 == 0) for j in range(D)])
    flows = [nf.flows.MaskedAffineFlow(b, mlp(D, D), mlp(D, D)), nf.flows.ActNorm(D)]
    flows[1]._mark_done()
    flows += [nf.flows.MaskedAffineFlow(1 - b, None, mlp(D, D)), nf.flows.Permute(D, "shuffle"),
              nf.flows.MaskedAffineFlow(b, mlp(D, D), None), nf.flows.AffineConstFlow(D, scale=False)]
    if D >= 2:
        h = (D + 1) // 2
        for k, (scale, smap, split) in enumerate([(True, "exp", "channel"), (True, "sigmoid", "channel_inv"),
                                                  (True, "sigmoid_inv", "channel"), (False, "exp", "channel_inv")]):
            n1 = h if split == "channel" else D - h
            flows.append(nf.flows.AffineCouplingBlock(mlp(n1, (2 if scale else 1) * (D - n1)), scale, smap, split))
            if k == 1:
                flows.append(nf.flows.Permute(D, "swap"))
    flows.append(nf.flows.AffineConstFlow(D))
    for i, f in enumerate(flows):
        _randomise(f, 1000 * seed + i, 0.35)
    return flows


def _close(got, ref, name, tol=2e-3):
    scale = ref.abs().max().item()
    err = (got.double() - ref).abs().max().item() if ref.numel() else 0.0
    assert err <= tol * max(scale, 1e-6), (name, err, scale)


def check_stack_gradients(flows, D, rows, seed, layer_loop=False):
    import normflows as nf
    from normflows._standalone import affine_slot_tensors
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
    slots = [p for p in affine_slot_tensors(model.flows) if isinstance(p, torch.nn.Parameter)]
    P = {id(p): p.detach().double().requires_grad_(True) for p in slots}
    zd = z0.double().requires_grad_(True)
    xr, ldr = sample_restated(model.flows, zd, P)
    ((xr * gx.double()).sum() + (ldr * gld.double()).sum()).backward()
    _close(x.detach(), xr.detach(), "x", 1e-4)
    _close(ld.detach(), ldr.detach(), "log_det", 1e-4)
    _close(z.grad, zd.grad, "g_z")
    for n, p in model.flows.named_parameters():
        assert p.grad is not None, n
        _close(p.grad, P[id(p)].grad, n)


@pytest.mark.gpu
@pytest.mark.parametrize("D,width,n_lin,slope,rows", [
    (1, 8, 2, 0.0, 129), (2, 4, 2, 0.0, 127), (2, 32, 3, 0.2, 5000), (5, 16, 2, 0.2, 128), (5, 128, 6, 0.0, 129),
    (16, 64, 3, 0.0, 1), (16, 128, 2, 0.2, 1000), (5, 8, 1, 0.0, 128)])
def test_stack_sampling_backward_matches_fp64_autograd(D, width, n_lin, slope, rows):
    check_stack_gradients(make_stack(D, width, n_lin, slope, seed=D + n_lin), D, rows, seed=rows)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [2, 5])
def test_layer_loop_sampling_backward_matches_fp64_autograd(D):
    """Each NativeFlow called on its own under grad (the layer-loop path) goes through the same backward."""
    check_stack_gradients(make_stack(D, 16, 2, 0.2, seed=7), D, 300, seed=3, layer_loop=True)


@pytest.mark.gpu
def test_zero_rows_give_zero_gradients():
    import normflows as nf
    flows = make_stack(5, 16, 2, 0.0, seed=1)
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows).cuda()
    z = torch.zeros(0, 5, device="cuda", requires_grad=True)
    x, ld = model.forward_and_log_det(z)
    (x.sum() + ld.sum()).backward()
    for n, p in model.flows.named_parameters():
        assert p.grad is not None and (p.grad == 0).all(), n


def real_nvp(K, latent_size=2, hidden=2, target=None):
    """examples/real_nvp.ipynb's model (augmented_flow.ipynb's with latent_size 4, hidden 4)."""
    import normflows as nf
    b = torch.Tensor([1 if i % 2 == 0 else 0 for i in range(latent_size)]) if latent_size == 2 else \
        torch.Tensor([1] * (latent_size // 2) + [0] * (latent_size // 2))
    flows = []
    for i in range(K):
        s = nf.nets.MLP([latent_size, hidden * latent_size, latent_size], init_zeros=True)
        t = nf.nets.MLP([latent_size, hidden * latent_size, latent_size], init_zeros=True)
        flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
        flows += [nf.flows.ActNorm(latent_size)]
    return nf.NormalizingFlow(q0=nf.distributions.DiagGaussian(latent_size), flows=flows, p=target)


@pytest.mark.gpu
def test_values_bit_identical_with_and_without_grad_and_reproducible_gradients():
    flows = make_stack(5, 32, 3, 0.2, seed=4)
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), flows).cuda()
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
    layer = model.flows[0]
    with torch.no_grad():
        y0, m0 = layer(z)
    y, m = layer(z.clone().requires_grad_(True))
    assert torch.equal(y, y0) and torch.equal(m, m0)


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(5), make_stack(5, 16, 2, 0.0, seed=2)).cuda()
    x, ld = model.forward_and_log_det(torch.randn(64, 5, device="cuda"))
    with torch.no_grad():
        model.flows[0].s.net[0].weight.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        (x.sum() + ld.sum()).backward()


@pytest.mark.gpu
def test_launch_count_does_not_depend_on_depth():
    counts = []
    for K in (4, 64):
        torch.manual_seed(0)
        model = real_nvp(K)
        for f in model.flows:
            if hasattr(f, "_mark_done"):
                f._mark_done()
        _randomise(model.flows, K)
        model = model.cuda()
        x, ld = model.forward_and_log_det(torch.randn(20, 2, device="cuda"))
        (x.sum() + ld.sum()).backward()
        counts.append(model._stack().launch_count())
    assert counts[0] == counts[1] and counts[0] <= 3, counts


@pytest.mark.gpu
def test_mixed_stacks_still_raise_and_affine_stacks_are_admitted():
    import normflows as nf
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    target = nf.distributions.TwoModes(2, 0.1)
    for flows in ([nf.flows.MaskedAffineFlow(torch.tensor([1., 0.]), nf.nets.MLP([2, 4, 2])), nf.flows.LULinearPermute(2)],
                  [nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 32), nf.flows.ActNorm(2)]):
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows, target).cuda()
        with pytest.raises(NotImplementedError, match=msg):
            model.reverse_kld(64)
    model = real_nvp(4, target=target).cuda()
    loss = model.reverse_kld(64)
    loss.backward()
    assert all(p.grad is not None for p in model.flows.parameters())


def _train_notebook(model, loss_fn, max_iter=300, loss_trend=True):
    """The notebooks' training cell (Adam lr 1e-4, weight decay 1e-6, skip non-finite losses), 300 iterations."""
    start = {n: p.detach().clone() for n, p in model.named_parameters()}
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-4, weight_decay=1e-6)
    loss_hist = []
    for it in range(max_iter):
        optimizer.zero_grad()
        loss = loss_fn(it)
        if ~(torch.isnan(loss) | torch.isinf(loss)):
            loss.backward()
            if it == max_iter - 1:
                for n, p in model.named_parameters():
                    assert p.grad is not None and torch.isfinite(p.grad).all(), n
            optimizer.step()
        loss_hist.append(loss.item())
    # (in float32 a batch of 20 can make every importance weight of reverse_alpha_div underflow: a non-finite loss,
    # which the notebook skips as well)
    h = np.array(loss_hist)
    first, last = h[:20][np.isfinite(h[:20])], h[-20:][np.isfinite(h[-20:])]
    assert len(first) >= 15 and len(last) >= 15, h
    assert first.mean() > last.mean() or not loss_trend, (first.mean(), last.mean())
    for n, p in model.named_parameters():
        assert torch.isfinite(p).all() and not torch.equal(p.detach(), start[n]), n


@pytest.mark.gpu
@pytest.mark.parametrize("annealing", [True, False])
def test_real_nvp_notebook_trains(annealing):
    import normflows as nf
    torch.manual_seed(0)
    nfm = real_nvp(64, target=nf.distributions.TwoModes(2, 0.1)).cuda()
    z, _ = nfm.sample(num_samples=2 ** 7)   # initialises ActNorm
    num_samples, anneal_iter = 2 * 10, 10000
    if annealing:
        fn = lambda it: nfm.reverse_kld(num_samples, beta=np.min([1., 0.001 + it / anneal_iter]))
        _train_notebook(nfm, fn)
        return
    # the DReG surrogate's value is too noisy at 20 samples to show a trend in 300 steps: the reverse KL of a fixed
    # 8 192-sample draw must fall instead
    def kl():
        with torch.no_grad():
            torch.manual_seed(123)
            z, log_q = nfm.sample(8192)
            return (log_q - nfm.p.log_prob(z)).mean().item()
    before = kl()
    _train_notebook(nfm, lambda it: nfm.reverse_alpha_div(num_samples, dreg=True, alpha=1), loss_trend=False)
    after = kl()
    assert after < before, (before, after)


@pytest.mark.gpu
def test_augmented_flow_notebook_trains():
    import normflows as nf
    torch.manual_seed(0)
    target = nf.distributions.TwoIndependent(nf.distributions.TwoMoons(), nf.distributions.DiagGaussian(2))
    nfm = real_nvp(32, latent_size=4, hidden=4, target=target).cuda()
    z, _ = nfm.sample(num_samples=2 ** 7)
    _train_notebook(nfm, lambda it: nfm.reverse_kld(2 * 10, beta=np.min([1., 0.01 + it / 10000])))


# ---- goldens m-q: fp64 autograd of the reference (tests/golden/make_affine_rkl_grads.py) -----------------------------
GOLDEN_CASES = ["m", "n", "o", "p", "q"]


def build_golden_case(name):
    """Case m-q built by this package (on the CPU) with the golden's parameters and buffers."""
    import helpers_affine_rkl as A
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_rkl_{name}.npz"))
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    model = A.build(nf, name)
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    model.load_state_dict({k: sd[k].to(v.dtype) for k, v in own.items()})
    eps = torch.tensor(gd["eps"])
    ctx = torch.tensor(gd["context"]) if "context" in gd else None
    return model, eps, ctx, gd


def _target_log_prob64(name, model, x, ctx):
    """The target's log-density in fp64 on the CPU; the DiagGaussian of case o's TwoIndependent is restated here (the
    package's density kernel is CUDA-only)."""
    if name == "o":
        t = model.p
        x1, x2 = x.chunk(2, dim=1)
        ls = t.target2.log_scale.reshape(-1)
        g = -math.log(2 * math.pi) - ls.sum() - 0.5 * (((x2 - t.target2.loc.reshape(-1)) / torch.exp(ls)) ** 2).sum(1)
        return t.target1.log_prob(x1) + g
    return model.p.log_prob(x, context=ctx) if ctx is not None else model.p.log_prob(x)


def restated_affine_loss(name, model, eps, ctx):
    """reverse_kld / reverse_alpha_div of cases m-q (core.py:104-165, 337-366) in fp64 torch: the affine layers by
    sample_restated, the context spline layer of q by the restated fixed-point sampling adjoint of
    test_reverse_kld_training."""
    import helpers_rkl as R
    from normflows._autograd import layer_inverse
    from test_reverse_kld_training import base_log_prob, sampling_fixed_point
    P = {id(p): p for p in model.parameters()}
    z, log_q = R.replay_forward(model.q0, eps)(eps.shape[0])
    for f in model.flows:
        z, ld = sample_restated([f], z, P) if getattr(f, "_affine_family", False) else sampling_fixed_point(f, z, ctx)
        log_q = log_q - ld
    log_p = _target_log_prob64(name, model, z, ctx)

    def log_q_no_param_grad():   # the reference sums the density pass into a float32 buffer (core.py:123, 151)
        for q in model.parameters():
            q.requires_grad_(False)
        zz, lq = z, torch.zeros(z.shape[0])
        for f in reversed(model.flows):
            zz, ld = layer_inverse(f, zz)
            lq += ld
        lq += base_log_prob(model.q0, zz)
        for q in model.parameters():
            q.requires_grad_(True)
        return lq
    if name == "n":
        w_const = torch.exp(log_p - log_q).detach()
        log_q = log_q_no_param_grad()
        w = torch.exp(log_p - log_q)
        w_alpha = w_const / torch.mean(w_const)
        return -torch.mean(w_alpha ** 2 * torch.log(w))
    if name == "o":
        log_q = log_q_no_param_grad()
    return torch.mean(log_q) - (0.5 if name == "m" else 1.0) * torch.mean(log_p)


def check_golden(got, gd, name, tol):
    from test_maf_training import check_golden as check
    check(got, gd, name, tol)


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_fp64_restatement_matches_reference_goldens(name):
    """The restated sampling direction and loss give the reference's fp64 autograd gradients to 1e-10 of each scale."""
    model, eps, ctx, gd = build_golden_case(name)
    model = model.double()
    loss = restated_affine_loss(name, model, eps.double(), ctx.double() if ctx is not None else None)
    loss.backward()
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    minted = {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))}
    assert minted == set(names), minted ^ set(names)
    for n, p in model.named_parameters():
        check_golden(p.grad, gd, n, 1e-10)


@pytest.mark.parametrize("name", ["m", "o"])
def test_targets_match_the_reference_log_prob_stored_in_the_goldens(name):
    model, eps, ctx, gd = build_golden_case(name)
    model = model.double()
    got = _target_log_prob64(name, model, eps.double(), None).detach().numpy()
    np.testing.assert_allclose(got, gd["p_log_prob"], rtol=1e-12, atol=1e-12)


def package_affine_loss(name, model, eps, ctx):
    import helpers_rkl as R
    model.q0.forward = R.replay_forward(model.q0, eps)
    n = eps.shape[0]
    if name == "m":
        return model.reverse_kld(n, beta=0.5)
    if name == "n":
        return model.reverse_alpha_div(n, alpha=1, dreg=True)
    if name == "o":
        return model.reverse_kld(n, score_fn=False)
    if name == "p":
        return model.reverse_kld(n)
    return model.reverse_kld(n, context=ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_model_gradients_match_reference_goldens(name):
    model, eps, ctx, gd = build_golden_case(name)
    model = model.cuda()
    loss = package_affine_loss(name, model, eps.cuda(), ctx.cuda() if ctx is not None else None)
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None, f"{n} got no gradient"
            check_golden(p.grad, gd, n, 2e-3)


@pytest.mark.gpu
def test_rows_beyond_one_workspace_chunk():
    """Wide, deep nets at 13 000 rows need three workspace chunks: the chunk offsets and the cross-chunk accumulation
    of the weight gradients against fp64 autograd."""
    import normflows as nf
    flows = make_stack(16, 128, 6, 0.0, seed=22)
    check_stack_gradients(flows, 16, 13000, seed=5)
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(16), flows).cuda()
    x, ld = model.forward_and_log_det(torch.randn(13000, 16, device="cuda"))
    (x.sum() + ld.sum()).backward()
    assert model._stack().launch_count() >= 6   # 3 launches per chunk


@pytest.mark.gpu
def test_a_parameter_shared_by_two_layers_gets_the_sum_of_its_gradients():
    import normflows as nf
    b = torch.tensor([1.0, 0.0])
    s, t = nf.nets.MLP([2, 8, 2], leaky=0.2), nf.nets.MLP([2, 8, 2])
    _randomise(s, 1), _randomise(t, 2)
    flows = [nf.flows.MaskedAffineFlow(b, t, s), nf.flows.MaskedAffineFlow(1 - b, t, s)]
    check_stack_gradients(flows, 2, 300, seed=9)
    act = nf.flows.AffineConstFlow(2)
    _randomise(act, 3)
    check_stack_gradients([act, nf.flows.Permute(2, "swap"), act], 2, 300, seed=10)
