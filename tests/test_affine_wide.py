"""The affine family's wide path: a group of MaskedAffineFlow / AffineCouplingBlock / AffineConstFlow (ActNorm) /
Permute layers with more than 16 features or a net wider than 128 runs layer by layer, its nets on the tensor-core GEMM
and its coupling arithmetic in csrc/nfb_affine_wide.cu (element formulas: csrc/nfb_affine_wide.cuh), in both directions
and both backwards.  A group within both limits keeps running on affine_stack_kernel.

CPU: the host-compiled element formulas against fp64 torch and, by central differences, against the adjoints the wide
backward pairs them with (non-finite s / t included); the cases' state_dicts rebuilt from the goldens' digests; an fp64
restatement pinned to the reference's goldens (tests/golden/make_affine_wide_grads.py, cases in
tests/helpers_affine_wide.py) at 1e-10.
GPU: values (log_prob, forward_kld, forward_kld_host, inverse_and_log_det, forward_and_log_det, one wide layer's forward /
inverse) and gradients (forward KL, reverse KL, a mixed stack, the flow-VAE) against the goldens; every entry point
against fp64 autograd over a shape grid, zero rows, several workspace chunks, nets 2 048 wide, bit-identical values with
and without grad, the in-place refusal, shared nets, per-layer launch budgets, and the notebooks' loops."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from test_affine_fkl_training import check_density_gradients
from test_affine_rkl_training import _close, _randomise, make_stack, sample_restated


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- element formulas on the host -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def elemlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("native") / "affine_wide_host_check.so")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "affine_wide_host_check.cu")])
    return C.CDLL(so)


def host_elem(lib, op, direction, a, b, c, d=None, scale=1, smap=0, use_float=0):
    """op 0 masked (z, b, s, t), 1 const (z, s, t), 2 coupling (v, shift, sc): (x, log-det term) per element."""
    f = lambda v: np.ascontiguousarray(v, dtype=np.float64).reshape(-1)
    a, b, c = f(a), f(b), f(c)
    d = f(d) if d is not None else np.zeros_like(a)
    x, ld = np.empty(a.size), np.empty(a.size)
    P = lambda v: v.ctypes.data_as(C.c_void_p)
    lib.affine_wide_elem_check(C.c_int(op), C.c_int(direction), C.c_int(scale), C.c_int(smap), C.c_int(a.size),
                               C.c_int(use_float), P(a), P(b), P(c), P(d), P(x), P(ld))
    return x, ld


def torch_masked(direction, z, b, s, t):
    nan = torch.tensor(float("nan"), dtype=torch.float64)
    s, t = torch.where(torch.isfinite(s), s, nan), torch.where(torch.isfinite(t), t, nan)
    if direction:
        return b * z + (1 - b) * (z * torch.exp(s) + t), (1 - b) * s
    return b * z + (1 - b) * (z - t) * torch.exp(-s), -(1 - b) * s


def torch_coupling(direction, scale, smap, v, shift, sc):
    if not scale:
        return (v + shift if direction else v - shift), torch.zeros_like(v)
    if smap == 0:
        return (v * torch.exp(sc) + shift, sc) if direction else ((v - shift) * torch.exp(-sc), -sc)
    sg = torch.sigmoid(sc + 2)
    div = (smap == 1) == bool(direction)
    if direction:
        x = v / sg + shift if div else v * sg + shift
    else:
        x = (v - shift) / sg if div else (v - shift) * sg
    return x, (-torch.log(sg) if div else torch.log(sg))


def _draw(n, seed, *scales):
    g = np.random.default_rng(seed)
    return [g.standard_normal(n) * s for s in scales]


@pytest.mark.parametrize("direction", [0, 1])
def test_masked_element_matches_fp64_torch_and_non_finite_nets_give_nan(elemlib, direction):
    z, s, t = _draw(400, 1 + direction, 1.5, 1.0, 1.0)
    b = (np.arange(400) % 2).astype(np.float64)
    s[:3], t[3:6], s[6], t[6] = np.inf, -np.inf, np.nan, np.nan
    x, ld = host_elem(elemlib, 0, direction, z, b, s, t)
    T = lambda v: torch.tensor(v, dtype=torch.float64)
    xr, ldr = torch_masked(direction, T(z), T(b), T(s), T(t))
    np.testing.assert_allclose(x, xr.numpy(), rtol=1e-13, atol=1e-13, equal_nan=True)
    np.testing.assert_allclose(ld, ldr.numpy(), rtol=1e-13, atol=1e-13, equal_nan=True)
    # a NaN in s or t stays NaN even where b = 1 masks its term out (0 * NaN), as in the reference
    assert np.isnan(x[:7]).all() and np.isfinite(x[7:]).all()
    xf, _ = host_elem(elemlib, 0, direction, z, b, s, t, use_float=1)
    np.testing.assert_allclose(xf[7:], x[7:], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("direction", [0, 1])
def test_const_element_matches_fp64_torch(elemlib, direction):
    z, s, t = _draw(300, 7, 1.0, 0.5, 1.0)
    x, ld = host_elem(elemlib, 1, direction, z, s, t)
    xr = z * np.exp(s) + t if direction else (z - t) * np.exp(-s)
    np.testing.assert_allclose(x, xr, rtol=1e-13)
    np.testing.assert_allclose(ld, s if direction else -s, rtol=0)


@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("scale,smap", [(1, 0), (1, 1), (1, 2), (0, 0)])
def test_coupling_element_matches_fp64_torch(elemlib, direction, scale, smap):
    v, shift, sc = _draw(300, 11 + smap, 1.5, 1.0, 1.5)
    x, ld = host_elem(elemlib, 2, direction, v, shift, sc, scale=scale, smap=smap)
    T = lambda a: torch.tensor(a, dtype=torch.float64)
    xr, ldr = torch_coupling(direction, scale, smap, T(v), T(shift), T(sc))
    np.testing.assert_allclose(x, xr.numpy(), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(ld, ldr.numpy(), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("op,scale,smap", [(0, 1, 0), (1, 1, 0), (2, 1, 0), (2, 1, 1), (2, 1, 2), (2, 0, 0)])
def test_element_formulas_agree_with_the_adjoints_by_central_differences(elemlib, direction, op, scale, smap):
    """The existing adjoints (nfb_affine_bwd.cuh), which the wide backward calls, are the derivatives of the new formulas:
    central differences of host_elem in every input, for MaskedAffineFlow, AffineConstFlow and AffineCouplingBlock
    (exp, sigmoid, sigmoid_inv, no scale)."""
    from test_affine_fkl_training import host_adjoint as dens_adj
    from test_affine_rkl_training import host_adjoint as samp_adj
    adj = dens_adj if direction == 0 else samp_adj
    so_name = "affine_density_adjoint_host_check.cu" if direction == 0 else "affine_adjoint_host_check.cu"
    so = os.path.join(os.path.dirname(elemlib._name), so_name.replace(".cu", ".so"))
    if not os.path.exists(so):
        subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-shared", "-Xcompiler", "-fPIC", "-o", so,
                               os.path.join(ROOT, "tests", "native", so_name)])
    alib = C.CDLL(so)
    n = 64
    z, s, t, g, gam = _draw(n, 21 + direction + 3 * op + smap, 1.0, 0.7, 0.7, 1.0, 1.0)
    b = (np.arange(n) % 2).astype(np.float64)
    h = 1e-6
    if op == 0:      # inputs (z, s, t); adjoint outputs (s_hat, t_hat, g_z)
        ins = [z, s, t]
        elem = lambda a: host_elem(elemlib, 0, direction, a[0], b, a[1], a[2])
        sh, th, gz = adj(alib, 0, z, b, s, t, g, gam)
        want = [gz, sh, th]
    elif op == 1:    # inputs (z, s, t); adjoint outputs (g_z, per-row g_s, per-row g_t)
        ins = [z, s, t]
        elem = lambda a: host_elem(elemlib, 1, direction, a[0], a[1], a[2])
        want = list(adj(alib, 1, z, b, s, t, g, gam))
    else:            # inputs (v, shift, sc); adjoint outputs (g_v, g_shift, g_sc)
        ins = [z, s, t]
        elem = lambda a: host_elem(elemlib, 2, direction, a[0], a[1], a[2], scale=scale, smap=smap)
        # (density: (a, b, c) = (v, shift, sc); sampling: (a, c) = (v, sc), the shift enters additively)
        want = list(adj(alib, 2, z, s, t, t, g, gam, scale=scale, smap=smap))
        if not scale:
            want[2] = np.zeros(n)
    for k in range(3):
        p_, m_ = [v.copy() for v in ins], [v.copy() for v in ins]
        p_[k] += h
        m_[k] -= h
        (xp, lp), (xm, lm) = elem(p_), elem(m_)
        fd = (g * (xp - xm) + gam * (lp - lm)) / (2 * h)
        np.testing.assert_allclose(want[k], fd, rtol=1e-5, atol=1e-6, err_msg=f"input {k}")


# ---- GPU: the stacks against fp64 autograd of the torch restatements --------------------------------------------------
WIDE_GRID = [(17, 32, 2, 0.2, 300), (2, 256, 3, 0.0, 513), (40, 40, 1, 0.0, 129), (64, 256, 3, 0.0, 1000),
             (17, 200, 2, 0.2, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("D,width,n_lin,slope,rows", WIDE_GRID)
def test_wide_sampling_backward_matches_fp64_autograd(D, width, n_lin, slope, rows):
    """forward_and_log_det (StackSamplingFn -> nfb_flow_sampling_backward) over every op variant."""
    check_sampling(make_stack(D, width, n_lin, slope, seed=D + n_lin), D, rows, seed=rows)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["log_prob", "inverse"])
@pytest.mark.parametrize("D,width,n_lin,slope,rows", WIDE_GRID)
def test_wide_density_backward_matches_fp64_autograd(D, width, n_lin, slope, rows, mode):
    """log_prob (nfb_flow_log_prob_backward) and inverse_and_log_det (nfb_flow_density_backward)."""
    check_density_gradients(make_stack(D, width, n_lin, slope, seed=D + n_lin), D, rows, seed=rows, mode=mode,
                            kink=1e-5 if n_lin > 1 else 0.0)


@pytest.mark.gpu
def test_a_single_wide_layer_in_both_directions():
    """Each layer called on its own (nfb_flow_layer_apply, LayerInverseFn) in both directions."""
    check_sampling(make_stack(17, 32, 2, 0.2, seed=7), 17, 300, seed=3, layer_loop=True)
    check_density_gradients(make_stack(17, 32, 2, 0.2, seed=7), 17, 300, seed=3, mode="layer")


@pytest.mark.gpu
def test_wide_groups_around_a_spline_block_and_lu():
    """Wide affine groups on both sides of a spline block + LULinearPermute: nfb_flow_log_prob_backward dispatches each
    affine group to the wide backward.  forward_kld and every gradient against test_affine_fkl_training's fp64
    restatement."""
    import normflows as nf
    from test_affine_fkl_training import restated_fkl
    model = mixed64(nf).cuda()
    x = torch.randn(700, 64, generator=torch.Generator().manual_seed(4)) * 0.8
    loss = model.forward_kld(x.cuda())
    loss.backward()
    md = mixed64(nf).double()
    md.load_state_dict({k: v.double().cpu() for k, v in model.state_dict().items()})
    ref = restated_fkl(md, x.double(), None)
    ref.backward()
    assert abs(loss.item() - ref.item()) < 1e-4 * (1 + abs(ref.item()))
    for (n, p), (_, q) in zip(model.named_parameters(), md.named_parameters()):
        assert p.grad is not None, n
        _close(p.grad, q.grad.cuda(), n)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sampling", "log_prob", "inverse", "layer"])
def test_zero_rows_give_zero_gradients(mode):
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(17), make_stack(17, 16, 2, 0.0, seed=1)).cuda()
    if mode == "sampling":
        z = torch.zeros(0, 17, device="cuda", requires_grad=True)
        x, ld = model.forward_and_log_det(z)
        (x.sum() + ld.sum()).backward()
    else:
        from test_affine_fkl_training import _run
        x = torch.zeros(0, 17, device="cuda", requires_grad=True)
        _, loss = _run(model, x, torch.zeros(0, 17, device="cuda"), torch.zeros(0, device="cuda"), mode)
        loss.backward()
    for n, p in model.flows.named_parameters():
        assert p.grad is not None and (p.grad == 0).all(), n


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sampling", "inverse"])
def test_rows_spanning_three_workspace_chunks(mode):
    """64 features and 512-wide, 4-Linear nets: 30 000 rows need three chunks of the 256 MiB workspace; the weight
    gradients accumulate across them (rows next to a ReLU kink left out, see check_density_gradients)."""
    from normflows import _lib
    flows = make_stack(64, 512, 4, 0.0, seed=22)
    if mode == "inverse":
        model = check_density_gradients(flows, 64, 30000, seed=5, mode="inverse", kink=1e-5)
    else:
        model = check_sampling(flows, 64, 30000, seed=5)
    per_row = _lib.lib().nfb_flow_density_backward_workspace_bytes(model._stack()._h, 1024) / 1024
    assert 30000 * per_row > 2.05 * (256 << 20), per_row


def sample_restated_margins(layers, z, P, margins):
    """sample_restated, recording each row's smallest |pre-activation| of a hidden layer in `margins`."""
    import torch.nn.functional as F
    import test_affine_rkl_training as R
    orig = R._mlp64

    def spy(net, x, P_, slope):
        lins = net.linear_layers()
        for i, lin in enumerate(lins):
            x = F.linear(x, P_[id(lin.weight)], P_[id(lin.bias)])
            if i + 1 < len(lins):
                margins.append(x.detach().abs().min(1).values)
                x = F.leaky_relu(x, slope)
        return x
    R._mlp64 = spy
    try:
        with torch.no_grad():
            sample_restated(layers, z, P)
    finally:
        R._mlp64 = orig


def check_sampling(flows, D, rows, seed, kink=1e-5, layer_loop=False):
    """test_affine_rkl_training's check_stack_gradients with rows next to a ReLU kink given zero cotangents (see
    check_density_gradients: with 256-wide nets a few float32 rows land on the other side of a kink than fp64)."""
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows).cuda()
    g = torch.Generator().manual_seed(seed)
    z0 = torch.randn(rows, D, generator=g).cuda()
    gx = torch.randn(rows, D, generator=g).cuda()
    gld = torch.randn(rows, generator=g).cuda()
    margins = []
    sample_restated_margins(model.flows, z0.double(), {id(p): p.detach().double() for p in model.parameters()}, margins)
    if margins:
        near = torch.stack(margins).min(0).values < kink
        gx[near], gld[near] = 0.0, 0.0
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
def test_values_bit_identical_with_and_without_grad_and_in_place_change_raises():
    import normflows as nf
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(17), make_stack(17, 160, 3, 0.2, seed=4)).cuda()
    x = torch.randn(777, 17, device="cuda")
    with torch.no_grad():
        z0, l0 = model.inverse_and_log_det(x)
        q0 = model.log_prob(x)
        s0, m0 = model.forward_and_log_det(x)
        y0, n0 = model.flows[0].inverse(x)
    z, ld = model.inverse_and_log_det(x.clone().requires_grad_(True))
    assert torch.equal(z, z0) and torch.equal(ld, l0)
    assert torch.equal(model.log_prob(x.clone().requires_grad_(True)), q0)
    s, m = model.forward_and_log_det(x.clone().requires_grad_(True))
    assert torch.equal(s, s0) and torch.equal(m, m0)
    y, n = model.flows[0].inverse(x.clone().requires_grad_(True))
    assert torch.equal(y, y0) and torch.equal(n, n0)
    with torch.no_grad():
        model.flows[0].s.net[0].weight.add_(1.0)
    for out in ((z, ld), (s, m), (y, n)):
        with pytest.raises(RuntimeError, match="modified in place"):
            (out[0].sum() + out[1].sum()).backward()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sampling", "log_prob", "inverse", "layer"])
def test_a_net_shared_by_two_layers_gets_the_sum_of_its_gradients(mode):
    import normflows as nf
    b = torch.tensor([float(j % 2) for j in range(20)])
    s, t = nf.nets.MLP([20, 160, 20], leaky=0.2), nf.nets.MLP([20, 160, 20])
    _randomise(s, 1), _randomise(t, 2)
    flows = [nf.flows.MaskedAffineFlow(b, t, s), nf.flows.MaskedAffineFlow(1 - b, t, s)]
    if mode == "sampling":
        check_sampling(flows, 20, 300, seed=9)
    else:
        check_density_gradients(flows, 20, 300, seed=9, mode=mode, kink=1e-5)


# ---- launch counts ----------------------------------------------------------------------------------------------------
def rnvp64(nf, K=8, D=64, hidden=256):
    """8 x [MaskedAffineFlow(alternating b, MLP([64, 256, 256, 64]) for s and t), ActNorm(64)]."""
    b = torch.tensor([float(j % 2) for j in range(D)])
    flows = []
    for i in range(K):
        s, t = nf.nets.MLP([D, hidden, hidden, D]), nf.nets.MLP([D, hidden, hidden, D])
        flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(D)]
    return flows


def mixed64(nf):
    torch.manual_seed(64)
    b = torch.tensor([float(j % 2) for j in range(64)])
    flows = [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([64, 160, 64]), nf.nets.MLP([64, 160, 64], leaky=0.2)),
             nf.flows.ActNorm(64), nf.flows.AutoregressiveRationalQuadraticSpline(64, 1, 64),
             nf.flows.LULinearPermute(64), nf.flows.AffineCouplingBlock(nf.nets.MLP([32, 200, 64]), True, "sigmoid"),
             nf.flows.Permute(64, "shuffle")]
    for i, f in enumerate(flows):
        if isinstance(f, nf.flows.ActNorm):
            f._mark_done()
        if not isinstance(f, (nf.flows.AutoregressiveRationalQuadraticSpline, nf.flows.LULinearPermute)):
            _randomise(f, 500 + i, 0.3)
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(64), flows)


def _counts(model, D, rows=256):
    x = torch.randn(rows, D, device="cuda")
    st = model._stack()
    with torch.no_grad():
        model.inverse_and_log_det(x)
        inv = st.launch_count()
        model.forward_and_log_det(x)
        fwd = st.launch_count()
    z, ld = model.inverse_and_log_det(x.clone().requires_grad_(True))
    (z.sum() + ld.sum()).backward()
    dbwd = st.launch_count()
    z, ld = model.forward_and_log_det(x.clone().requires_grad_(True))
    (z.sum() + ld.sum()).backward()
    return inv, fwd, dbwd, st.launch_count()


def _per_block(make, D):
    """Launches per block (difference between 4 and 2 blocks, halved) of inverse, forward, density backward and sampling
    backward, after checking that the counts are linear in depth (the fixed part does not grow)."""
    import normflows as nf
    counts = {}
    for K in (2, 4, 6):
        torch.manual_seed(0)
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), make(K)).cuda()
        counts[K] = _counts(model, D)
    per = [(b - a) / 2 for a, b in zip(counts[2], counts[4])]
    assert [(c - b) / 2 for b, c in zip(counts[4], counts[6])] == per, counts
    return per


@pytest.mark.gpu
def test_launch_count_within_the_per_layer_budget_and_linear_in_depth():
    """DESIGN §3.13's budget.  Per [MaskedAffineFlow with 3-Linear s and t nets, ActNorm] block: forward 6 GEMMs + their
    6 weight packs + 2 element launches (masked input, coupling) + 1 (ActNorm) = 15.  Backward: the recompute of the
    block's input (15), the nets again (mask + 6 GEMMs + 6 packs = 13), 1 adjoint, per net and Linear a wgrad GEMM, a
    bias memset and colsum, and per net 3 dgrad GEMMs + packs (2 x 15), ActNorm 1 adjoint + 2 x (memset, colsum) = 64.
    Per [AffineCouplingBlock(MLP([32, 256, 64])), Permute] block: forward 2 GEMMs + 2 packs + 1 element + 1 gather = 6;
    backward 6 (recompute) + 4 (net again) + 1 adjoint + 2 x 3 (wgrad, memset, colsum) + 2 x 2 (dgrad, pack) + 1 gather
    = 22."""
    import normflows as nf

    def masked(K):
        flows = rnvp64(nf, K)
        for f in flows:
            if isinstance(f, nf.flows.ActNorm):
                f._mark_done()
        return flows

    def coupling(K):
        flows = []
        for _ in range(K):
            flows += [nf.flows.AffineCouplingBlock(nf.nets.MLP([32, 256, 64])), nf.flows.Permute(64, "swap")]
        for i, f in enumerate(flows):
            _randomise(f, i, 0.2)
        return flows
    inv, fwd, dbwd, sbwd = _per_block(masked, 64)
    assert inv <= 15 and fwd <= 15 and dbwd <= 64 and sbwd <= 64, (inv, fwd, dbwd, sbwd)
    inv, fwd, dbwd, sbwd = _per_block(coupling, 64)
    assert inv <= 6 and fwd <= 6 and dbwd <= 22 and sbwd <= 22, (inv, fwd, dbwd, sbwd)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["sampling", "log_prob"])
def test_nets_2048_wide(mode):
    """A hidden layer 2 048 wide at 512 rows: few output tiles and K >= 2 048, where the GEMM would split K; with a bias /
    ReLU epilogue it runs unsplit."""
    import normflows as nf
    torch.manual_seed(3)
    b = torch.tensor([float(j % 2) for j in range(64)])
    flows = [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([64, 2048, 64]), nf.nets.MLP([64, 2048, 64])),
             nf.flows.MaskedAffineFlow(1 - b, nf.nets.MLP([64, 2048, 2048, 64]), None)]
    for i, f in enumerate(flows):
        _randomise(f, 70 + i, 0.3)
    if mode == "sampling":
        check_sampling(flows, 64, 512, seed=8)
    else:
        check_density_gradients(flows, 64, 512, seed=8, mode=mode, kink=1e-5)


@pytest.mark.gpu
def test_a_narrow_stack_still_runs_affine_stack_kernel_once():
    """real_nvp_colab's 64 blocks fit the narrow limits: log_prob is the log-det fill, ONE affine_stack_kernel launch and
    the base density, whatever the batch."""
    import helpers_affine_fkl as A
    import normflows as nf
    torch.manual_seed(0)
    model = A.colab(nf).cuda()
    for rows in (512, 65536):
        with torch.no_grad():
            model.log_prob(torch.randn(rows, 2, device="cuda"))
        assert model._stack().launch_count() == 3


# ---- notebooks --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_vae_notebook_realnvp_cell_as_written_runs_a_step():
    """examples/vae.ipynb with flow_type = 'RealNVP': 40 features, 40 MaskedAffineFlows with MLP([40, 40]) nets.  As
    written (default initialisation) exp(s) overflows in the first forward and the prior's argument check raises, as in
    the reference's float32 run; with the nets scaled down so every value is finite, the notebook's step runs through
    the wide sampling backward."""
    from torch import optim
    from test_vae_training import _notebook, synthetic_mnist
    torch.manual_seed(0)
    nfm = _notebook("RealNVP")
    x = synthetic_mnist(64).cuda()
    with pytest.raises(ValueError, match="support"):
        nfm(x, 32)
    with torch.no_grad():
        for f in nfm.flows:
            for p in f.parameters():
                p.mul_(0.05)
    optimizer = optim.Adam(nfm.parameters(), lr=1e-4, weight_decay=1e-4)
    optimizer.zero_grad()
    z, log_q, log_p = nfm(x, 32)
    assert z.shape == (64, 32, 40) and torch.isfinite(z).all()
    loss = torch.mean(log_q) - torch.mean(log_p)
    loss.backward()
    optimizer.step()
    assert np.isfinite(loss.item())
    for n, p in nfm.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n


@pytest.mark.gpu
def test_rnvp64_forward_kld_loop_lowers_the_loss():
    import normflows as nf
    torch.manual_seed(0)
    flows = rnvp64(nf)
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(64), flows).cuda()
    A = torch.randn(64, 64, generator=torch.Generator().manual_seed(1)).cuda() * 0.3
    optimizer = torch.optim.Adam(model.parameters(), lr=1e-4)
    hist = []
    for it in range(100):
        x = torch.randn(512, 64, device="cuda") @ A + 1.0
        optimizer.zero_grad()
        loss = model.forward_kld(x)
        loss.backward()
        optimizer.step()
        hist.append(loss.item())
    h = np.array(hist)
    assert np.isfinite(h).all() and h[-10:].mean() < h[:10].mean() - 1.0, (h[:10].mean(), h[-10:].mean())


# ---- goldens: fp64 autograd of the reference (tests/golden/make_affine_wide_grads.py) ---------------------------------
def _golden(name):
    from helpers import load_npz_parts
    return load_npz_parts(os.path.join(ROOT, "tests", "golden", f"grads_wide_{name}.npz"))


def build_golden_case(name):
    """Case `name` built by this package on the CPU with the golden's parameters: rebuilt by the shared constructors and
    perturbation, checked bit for bit against the golden's digests (w17 also loads its stored state_dict)."""
    import json
    import helpers_affine_wide as W
    import normflows as nf
    gd = _golden(name)
    model = W.build(nf, name)
    W.perturb(model, name)
    if name == "w17":
        own = model.state_dict()
        sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
        assert set(own) == set(sd), set(own) ^ set(sd)
        model.load_state_dict({k: sd[k].to(v.dtype) for k, v in own.items()})
    ref = json.loads(str(gd["sd_sha256"]))
    own = json.loads(W.digests(model))
    assert set(own) == set(ref), set(own) ^ set(ref)
    bad = [k for k in own if own[k] != ref[k]]
    assert not bad, f"{name}: rebuilt entries differ from the reference's: {bad[:5]}"
    return model, gd


def _mixture_log_prob64(p, z):
    """GaussianMixture.log_prob (distributions/base.py of the reference) in fp64 torch."""
    loc, ls = p.loc.double().reshape(1, -1, z.shape[1]), p.log_scale.double().reshape(1, -1, z.shape[1])
    w = torch.softmax(p.weight_scores.double().reshape(1, -1), 1)
    eps = (z[:, None, :] - loc) / torch.exp(ls)
    lp = (-0.5 * z.shape[1] * np.log(2 * np.pi) + torch.log(w) - 0.5 * torch.sum(eps ** 2, 2) - torch.sum(ls, 2))
    return torch.logsumexp(lp, 1)


def _vae_restated(P, x, eps):
    """NormalizingFlowVAE.forward of case vae40 in fp64 (helpers_vae's pieces: NN encoder, MaskedAffineFlows, standard
    normal prior, Bernoulli decoder) and the notebook's loss."""
    import helpers_vae as V
    B, S, d = eps.shape
    z, log_q = V.encoder_draw("a", P, x, eps)
    z, log_q = z.reshape(B * S, d), log_q.reshape(-1)
    for i in range(40):
        z, ld = V.masked_affine(z, P, f"flows.{i}.")
        log_q = log_q - ld
    log_p = V.prior_log_prob("a", P, z) + V.decoder_log_prob("e", P, x, z)
    log_q, log_p = log_q.view(B, S), log_p.view(B, S)
    return z.view(B, S, d), log_q, log_p, torch.mean(log_q) - torch.mean(log_p)


def _check(got, gd, name, tol):
    from test_maf_training import check_golden
    check_golden(got, gd, name, tol)


def _minted(gd):
    return {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))}


@pytest.mark.parametrize("name", ["w17", "w2wide", "rnvp64", "rnvp64_rkl", "mixed64", "vae40"])
def test_fp64_restatement_matches_reference_goldens(name):
    """The restated directions and losses give the reference's fp64 autograd gradients to 1e-10 of each scale."""
    import helpers_rkl as R
    from test_affine_fkl_training import restated_fkl
    model, gd = build_golden_case(name)
    model = model.double()
    if name == "vae40":
        P = {k: v.detach().double().clone().requires_grad_(True) for k, v in model.named_parameters()}
        P.update({k: v.double() for k, v in model.named_buffers()})
        z, log_q, log_p, loss = _vae_restated(P, torch.tensor(gd["x"]).double(), torch.tensor(gd["eps"]).double())
        for key, got in (("z", z), ("log_q", log_q), ("log_p", log_p)):
            np.testing.assert_allclose(got.detach().numpy(), gd[key], rtol=1e-10, atol=1e-10, err_msg=key)
        loss.backward()
        grads = {k: v.grad for k, v in P.items() if v.requires_grad}
    else:
        if name == "rnvp64_rkl":
            eps = torch.tensor(gd["eps"]).double()
            P = {id(p): p for p in model.parameters()}
            z, log_q = R.replay_forward(model.q0, eps)(eps.shape[0])
            x, ld = sample_restated(model.flows, z, P)
            loss = torch.mean(log_q - ld) - torch.mean(_mixture_log_prob64(model.p, x))
        else:
            loss = restated_fkl(model, torch.tensor(gd["x"]).double(), None)
        loss.backward()
        grads = {n: p.grad for n, p in model.named_parameters() if p.requires_grad}
    # (the reference sums log_q into a float32 buffer in forward_kld / reverse_kld)
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    assert _minted(gd) == set(grads), _minted(gd) ^ set(grads)
    for n, g in grads.items():
        _check(g, gd, n, 1e-10)


def _gpu_case(name):
    model, gd = build_golden_case(name)
    return model.cuda(), gd


def _vclose(got, ref, what, tol=1e-4):
    ref = torch.as_tensor(np.asarray(ref)).double()
    assert tuple(got.shape) == tuple(ref.shape), (what, got.shape, ref.shape)
    _close(got.detach().double().cpu(), ref, what, tol)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w17", "w2wide", "rnvp64", "mixed64"])
def test_values_match_reference_goldens(name):
    """log_prob, forward_kld, forward_kld_host, inverse_and_log_det, forward_and_log_det and the first (wide) layer's
    inverse / forward on its own, against the reference's fp64 values at 1e-4 of each scale."""
    model, gd = _gpu_case(name)
    x = torch.tensor(gd["x"])
    xc = x.cuda()
    with torch.no_grad():
        _vclose(model.log_prob(xc), gd["log_q"], "log_prob")
        ref = -float(np.mean(gd["log_q"]))
        for what, got in (("forward_kld", model.forward_kld(xc).item()), ("forward_kld_host", model.forward_kld_host(x))):
            got = float(got)
            assert abs(got - ref) <= 1e-4 * max(1.0, abs(ref)), (what, got, ref)
        z, ld = model.inverse_and_log_det(xc)
        _vclose(z, gd["inv_z"], "inverse z")
        _vclose(ld, gd["inv_ld"], "inverse log_det")
        if "fwd_x" in gd:
            y, ld = model.forward_and_log_det(xc)
            _vclose(y, gd["fwd_x"], "forward x")
            _vclose(ld, gd["fwd_ld"], "forward log_det")
        for key, fn in (("l0_inv", model.flows[0].inverse), ("l0_fwd", model.flows[0].forward)):
            y, ld = fn(xc)
            _vclose(y, gd[key + ("_z" if key == "l0_inv" else "_x")], key)
            _vclose(ld, gd[key + "_ld"], key + " log_det")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w17", "w2wide", "rnvp64", "rnvp64_rkl", "mixed64", "vae40"])
def test_model_gradients_match_reference_goldens(name):
    """Forward KL (w17, w2wide, rnvp64, mixed64), reverse KL against a native 64-D GaussianMixture (rnvp64_rkl) and the
    flow-VAE loss (vae40): loss and every gradient against the reference's fp64 autograd at 2e-3 of each scale."""
    import helpers_rkl as R
    model, gd = _gpu_case(name)
    if name == "rnvp64_rkl":
        eps = torch.tensor(gd["eps"]).cuda()
        model.q0.forward = R.replay_forward(model.q0, eps)
        loss = model.reverse_kld(eps.shape[0])
    elif name == "vae40":
        import helpers_affine_wide as W
        eps = torch.tensor(gd["eps"]).cuda()
        model.q0._draw_eps = lambda shape, device: eps.reshape(shape).clone()
        model.prior = torch.distributions.MultivariateNormal(torch.zeros(40, device="cuda"),
                                                             torch.eye(40, device="cuda"))
        z, log_q, log_p = model(torch.tensor(gd["x"]).cuda(), W.VAE_S)
        for key, got in (("z", z), ("log_q", log_q), ("log_p", log_p)):
            _vclose(got, gd[key], key, 2e-3)
        loss = torch.mean(log_q) - torch.mean(log_p)
    else:
        loss = model.forward_kld(torch.tensor(gd["x"]).cuda())
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    names = set()
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None, f"{n} got no gradient"
            _check(p.grad.cpu(), gd, n, 2e-3)
            names.add(n)
    assert names == _minted(gd), names ^ _minted(gd)
