"""Reverse-KL training of coupling spline flows: gradients through the sampling direction of an all-native stack of
CoupledRationalQuadraticSpline and LULinearPermute layers (nfb_flow_sampling_backward).

The LU layer's sampling map and its adjoint (W = L U, perm the layer's permutation):
    t = W^-1 (y - b),  x = t[:, inv_perm],  log_det = -sum log diag U
    g_t = g_x[:, perm],  g_y = W^-T g_t,  dW = -sum_rows g_y t^T,  g_b = -colsum(g_y),  d log|det W| = -sum g_ld
and dW, d log|det W| go through W = L U to the factors.  A coupled block's sampling adjoint is the stand-alone layer's
(tests/test_reverse_kld_training.py SamplingAdjoint): the inverse spline's adjoint on the transform features, the
conditioner's backward at the identity features' output, the unconditional CDF's inverse adjoint on g_x[id] plus the
conditioner's data gradient.

CPU: an fp64 restatement of both adjoints pinned to gradients minted from the reference's autograd
(tests/golden/make_coupled_rkl_grads.py, cases w-z) at 1e-10; which stacks are admitted.
GPU: stack backward against fp64 autograd of the sampling pass over stack shapes, both execution paths and zero rows;
models w-z against the goldens; bit-identical values with and without grad; the in-place refusal; a lone coupled layer;
NormalizingFlowVAE; a short training loop."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import helpers_coupled_rkl as H
import helpers_rkl as R
from conftest import ROOT
from test_conditional_training import ref_net, ref_spline_params
from test_maf_training import check_golden
from test_reverse_kld_training import (_records, _uncond_table, base_log_prob, layer_spec, relu_margin,
                                       sampling_fixed_point, sampling_unrolled)

GOLDEN = os.path.join(ROOT, "tests", "golden")
CASES = ["w", "x", "y", "z"]


@pytest.fixture(autouse=True)
def _grad_on():
    with torch.enable_grad():
        yield


# ---- fp64 restatement ----------------------------------------------------------------------------------------------
def lu_weight(lin):
    """(W = L U, log|det W|) of an LULinearPermute's factors (flows/mixing.py:402-412, 514-532), differentiable."""
    n = lin.features
    il, iu = torch.tril_indices(n, n, -1), torch.triu_indices(n, n, 1)
    dt = lin.unconstrained_upper_diag.dtype
    lower = torch.eye(n, dtype=dt).index_put((il[0], il[1]), lin.lower_entries)
    diag = F.softplus(lin.unconstrained_upper_diag) + lin.eps
    upper = torch.diag(diag).index_put((iu[0], iu[1]), lin.upper_entries)
    return lower @ upper, torch.log(diag).sum()


def lu_sampling_unrolled(layer, y):
    """LULinearPermute.forward (the sampling direction), differentiable by autograd."""
    W, lad = lu_weight(layer.linear)
    t = torch.linalg.solve(W, (y - layer.linear.bias).T).T
    inv = torch.argsort(layer.permutation._permutation)
    return t[:, inv], -lad.expand(y.shape[0])


class LUSamplingAdjoint(torch.autograd.Function):
    """The sampling map under no_grad; backward: the adjoint in the module docstring, as the native code runs it."""

    @staticmethod
    def forward(ctx, layer, y, *params):
        with torch.no_grad():
            x, ld = lu_sampling_unrolled(layer, y)
            W, _ = lu_weight(layer.linear)
            t = torch.linalg.solve(W, (y - layer.linear.bias).T).T
        ctx.layer, ctx.params = layer, params
        ctx.save_for_backward(t)
        return x, ld

    @staticmethod
    def backward(ctx, g_x, g_ld):
        (t,) = ctx.saved_tensors
        lin = ctx.layer.linear
        g_x = torch.zeros_like(t) if g_x is None else g_x
        g_ld = torch.zeros(t.shape[0], dtype=t.dtype) if g_ld is None else g_ld
        with torch.no_grad():
            W, _ = lu_weight(lin)
            g_t = g_x[:, ctx.layer.permutation._permutation]
            g_y = g_t @ torch.linalg.inv(W)
            dW = -(g_y.T @ t)
            g_b = -g_y.sum(0)
        with torch.enable_grad():
            factors = [lin.lower_entries, lin.upper_entries, lin.unconstrained_upper_diag]
            W_, lad_ = lu_weight(lin)
            gf = torch.autograd.grad([W_, lad_], factors, [dW, -g_ld.sum()], allow_unused=True)
        gmap = dict(zip(map(id, factors), gf))
        gmap[id(lin.bias)] = g_b
        return (None, g_y, *[gmap.get(id(q)) for q in ctx.params])


def sample_layer(layer, z):
    if hasattr(layer, "prqct"):
        return sampling_fixed_point(layer, z, None)
    return LUSamplingAdjoint.apply(layer, z, *layer.parameters())


def density_layer(layer, x):
    """The density direction (`inverse`) in fp64: (z, log_det)."""
    if hasattr(layer, "prqct"):
        p, K, tb = layer.prqct, layer.num_bins, layer.tail_bound
        idf, trf = p.identity_features, p.transform_features
        rows = x.shape[0]
        yi, ldi = ref_spline_params(x[:, idf], _uncond_table(p).expand(rows, -1, -1), K, "linear", tb)
        prm = _records(ref_net(p.transform_net, x[:, idf], None, False), len(trf))
        yt, ld = ref_spline_params(x[:, trf], prm, K, "linear", tb, 1.0 / np.sqrt(p.transform_net.hidden_features))
        out = torch.empty_like(x)
        out[:, idf], out[:, trf] = yi, yt
        return out, ld.sum(1) + ldi.sum(1)
    W, lad = lu_weight(layer.linear)
    return x[:, layer.permutation._permutation] @ W.T + layer.linear.bias, lad.expand(x.shape[0])


def restated_loss(name, model, eps):
    """reverse_kld / reverse_alpha_div of cases w-z (core.py:104-165), on the restated adjoints."""
    z, log_q = R.replay_forward(model.q0, eps)(eps.shape[0])
    for f in model.flows:
        z, ld = sample_layer(f, z)
        log_q = log_q - ld
    log_p = model.p.log_prob(z)

    def log_q_no_param_grad():
        for q in model.parameters():
            q.requires_grad_(False)
        zz, lq = z, torch.zeros(z.shape[0])   # float32, like the reference's buffer (core.py:123, 151)
        for f in reversed(model.flows):
            zz, ld = density_layer(f, zz)
            lq += ld
        lq += base_log_prob(model.q0, zz)
        for q in model.parameters():
            q.requires_grad_(True)
        return lq
    if name == "x":   # alpha = 1, dreg
        w_const = torch.exp(log_p - log_q).detach()
        log_q = log_q_no_param_grad()
        w = torch.exp(log_p - log_q)
        w_alpha = w_const / torch.mean(w_const)
        return -torch.mean(w_alpha ** 2 * torch.log(w))
    if name == "z":
        log_q = log_q_no_param_grad()
    return torch.mean(log_q) - torch.mean(log_p)


def build_case(name):
    """Case w-z built by this package (on the CPU) with the golden's state (parameters and buffers)."""
    import normflows as nf
    from helpers import load_npz_parts
    gd = load_npz_parts(os.path.join(GOLDEN, f"grads_rkl_{name}.npz"))
    sd = {k[4:]: torch.tensor(v) for k, v in gd.items() if k.startswith("sd__")}
    model = H.build(nf, name)
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    model.load_state_dict({k: sd[k].to(v.dtype) for k, v in own.items()})
    return model, torch.tensor(gd["eps"]), gd


@pytest.mark.parametrize("name", CASES)
def test_fp64_restatement_matches_reference_goldens(name):
    """The restated LU and coupled-block sampling adjoints give the reference's autograd gradients to 1e-10."""
    model, eps, gd = build_case(name)
    model = model.double()
    loss = restated_loss(name, model, eps.double())
    loss.backward()
    # (x and z re-evaluate log_q in the reference's float32 buffer: their losses carry fp32 rounding)
    assert abs(loss.item() - float(gd["loss"])) <= 1e-6 * max(1.0, abs(float(gd["loss"])))
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    minted = {k.split("__", 1)[1] for k in gd if k.startswith(("g__", "gn__"))}
    assert minted == set(names), minted ^ set(names)
    for n, p in model.named_parameters():
        check_golden(p.grad, gd, n, 1e-10)


def test_w_has_draws_beyond_the_tail_bound():
    eps = H.draws("w")
    assert ((eps.abs() > 3).sum(1) == 6).sum() == 8


def test_admission_is_a_stack_level_rule():
    """Coupled (8 bins, no context) + LU stacks are admitted; an LU layer alone stays without a sampling backward, and
    so do stacks with an autoregressive block or another bin count."""
    import normflows as nf
    Cq, LU = nf.flows.CoupledRationalQuadraticSpline, nf.flows.LULinearPermute
    ok = lambda flows: nf.NormalizingFlow(nf.distributions.DiagGaussian(4), flows)._flows_sampling_differentiable()
    assert ok([Cq(4, 1, 16), LU(4)]) and ok([LU(4)]) and ok([LU(4), Cq(4, 1, 16), LU(4), LU(4)])
    assert not ok([nf.flows.AutoregressiveRationalQuadraticSpline(4, 1, 16), LU(4)])
    assert not ok([Cq(4, 1, 16, num_bins=6), LU(4)])
    assert not ok([nf.flows.CircularAutoregressiveRationalQuadraticSpline(4, 1, 16, [1]), LU(4)])
    assert not LU(4)._sampling_differentiable() and Cq(4, 1, 16)._sampling_differentiable()


def test_layer_loops_with_an_lu_layer_still_raise_under_grad():
    """The stack rule holds only where the stack runs: a conditional flow walks its layers one by one, and so does an
    all-native stack whose base draws are not [rows, features]; an LU layer there has no sampling backward."""
    import normflows as nf
    Cq, LU = nf.flows.CoupledRationalQuadraticSpline, nf.flows.LULinearPermute
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    for flows in ([Cq(4, 1, 16), LU(4)], [LU(4)]):
        model = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(4), flows, R.ContextTarget())
        with pytest.raises(NotImplementedError, match=msg):
            model.reverse_kld(8)
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian((4, 1)), [Cq(4, 1, 16), LU(4)])
    with pytest.raises(NotImplementedError, match=msg):
        model.reverse_kld(8)
    cond = nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(4), [Cq(4, 1, 16)], R.ContextTarget())
    assert cond._flows_sampling_differentiable()   # the coupled layer alone carries its own backward


# ================================================ GPU ================================================================
def _close(got, ref, name, tol=2e-3):
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = ref.abs().max().item() + 1e-12
    err = (got - ref).abs().max().item()
    assert err <= tol * scale, f"{name}: max err {err:.3e} scale {scale:.3e}"


def make_stack(kinds, D, hidden, blocks, seed, first_reverse=False):
    import normflows as nf
    torch.manual_seed(seed)
    flows, i = [], 0
    for k in kinds:
        if k == "C":
            flows.append(nf.flows.CoupledRationalQuadraticSpline(D, blocks, hidden, tail_bound=2.5,
                                                                 reverse_mask=bool((i + first_reverse) % 2)))
            i += 1
        else:
            flows.append(nf.flows.LULinearPermute(D))
    # off the identity init by 0.1 at width 32, less for wider nets: at 0.1 a 256-wide conditioner makes splines so steep
    # that float32 torch itself misses the fp64 gradients by 4e-3
    s = 0.1 * min(1.0, (32 / max(hidden, 1)) ** 0.5)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for f in flows:
            for p in f.parameters():
                p.add_(s * torch.randn(p.shape, generator=g))
    return flows


def stack_unrolled(flows, z):
    x, ld = z, torch.zeros(z.shape[0], dtype=z.dtype)
    for f in flows:
        x, l = sampling_unrolled(layer_spec(f), x, None) if hasattr(f, "prqct") else lu_sampling_unrolled(f, x)
        ld = ld + l
    return x, ld


def stack_margin(flows, z):
    """Per row, the smallest relative ReLU margin of any coupled block's conditioner along the fp64 sampling pass."""
    m = torch.full((z.shape[0],), float("inf"), dtype=z.dtype)
    x = z
    for f in flows:
        if hasattr(f, "prqct"):
            spec = layer_spec(f)
            xo, _ = sampling_unrolled(spec, x, None)
            if len(f.prqct.transform_net.blocks):   # (a net without blocks has no ReLU)
                m = torch.minimum(m, relu_margin(spec, x, xo, None))
            x = xo
        else:
            x, _ = lu_sampling_unrolled(f, x)
    return m


STACKS = [   # kinds, D, hidden, blocks, rows, tensor cores (False: the layer-by-layer path), first reverse_mask
    ("C", 2, 32, 0, 127, True, False),
    ("C", 5, 64, 1, 1061, True, True),
    ("C", 17, 128, 2, 1, False, False),
    ("CL", 2, 48, 1, 1061, True, True),
    ("CL", 17, 64, 2, 127, True, False),
    ("CL", 5, 32, 1, 0, True, False),
    ("L", 17, 0, 0, 127, True, False),
    ("LL", 5, 0, 0, 1061, True, False),
    ("CLCL", 64, 256, 2, 1061, True, False),
    ("CLCL", 64, 256, 1, 127, False, True),
    ("LCLC", 17, 128, 1, 1061, True, False),
    ("LCLCL", 5, 32, 2, 1, True, True),
    ("CLLC", 5, 32, 0, 127, True, False),
    ("CCLCCL", 2, 256, 2, 1061, True, False),
    ("CLCLCLCL", 64, 64, 1, 0, True, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kinds,D,hidden,blocks,rows,tc,rev", STACKS)
def test_stack_sampling_backward_matches_fp64_autograd(kinds, D, hidden, blocks, rows, tc, rev):
    import normflows as nf
    flows = make_stack(kinds, D, hidden, blocks, 31 * D + len(kinds) + rows, rev)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(rows, D, generator=g) * 1.3
    gx, gld = torch.randn(rows, D, generator=g), torch.randn(rows, generator=g)
    ref = [copy.deepcopy(f).double() for f in flows]
    if rows:   # leave out rows on a conditioner ReLU kink (within 1e-5 of the median activation)
        with torch.no_grad():
            keep = stack_margin(ref, z.double()) > 1e-5
        z, gx, gld = z[keep], gx[keep], gld[keep]
        assert keep.sum() >= 0.9 * rows
        rows = z.shape[0]
    zr = z.double().requires_grad_(True)
    xr, ldr = stack_unrolled(ref, zr)
    ((xr * gx.double()).sum() + (ldr * gld.double()).sum()).backward()
    old = nf.flows.base.NativeFlow.use_tensor_cores
    nf.flows.base.NativeFlow.use_tensor_cores = tc
    try:
        flows = [f.cuda() for f in flows]
        zc = z.cuda().requires_grad_(True)
        if len(flows) == 1 and kinds == "C":   # the layer on its own
            x, ld = flows[0](zc)
        else:
            x, ld = nf.NormalizingFlow(None, flows).forward_and_log_det(zc)
        assert x.requires_grad and ld.requires_grad
        ((x * gx.cuda()).sum() + (ld * gld.cuda()).sum()).backward()
    finally:
        nf.flows.base.NativeFlow.use_tensor_cores = old
    if rows:
        _close(x.detach(), xr.detach(), "x", 1e-4)
        _close(ld.detach(), ldr.detach(), "log_det", 1e-4)
        _close(zc.grad, zr.grad, "z")
    for k, (f, fr) in enumerate(zip(flows, ref)):
        refp = dict(fr.named_parameters())
        for n, p in f.named_parameters():
            assert p.grad is not None, (k, n)
            if rows == 0:
                assert (p.grad == 0).all(), (k, n)
            else:
                _close(p.grad, refp[n].grad, f"layer {k} {n}")


def package_loss(name, model, eps):
    model.q0.forward = R.replay_forward(model.q0, eps)
    return H.loss_of(name, model, eps.shape[0])


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_model_gradients_match_reference_goldens(name):
    model, eps, gd = build_case(name)
    model = model.cuda()
    loss = package_loss(name, model, eps.cuda())
    loss.backward()
    ref = float(gd["loss"])
    assert abs(loss.item() - ref) < 1e-4 * (1 + abs(ref)), (loss.item(), ref)
    for n, p in model.named_parameters():
        assert p.grad is not None, f"{n} got no gradient"
        check_golden(p.grad, gd, n, 2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["w", "y"])
def test_values_bit_identical_with_and_without_grad(name):
    model, eps, _ = build_case(name)
    model = model.cuda()
    model.q0.forward = R.replay_forward(model.q0, eps.cuda())
    with torch.no_grad():
        a = model.sample(eps.shape[0])
        ka = model.reverse_kld(eps.shape[0])
    b = model.sample(eps.shape[0])
    kb = model.reverse_kld(eps.shape[0])
    assert b[0].requires_grad and b[1].requires_grad and kb.requires_grad
    assert torch.equal(a[0], b[0].detach()) and torch.equal(a[1], b[1].detach())
    assert torch.equal(ka, kb.detach())


@pytest.mark.gpu
def test_in_place_parameter_change_after_forward_raises():
    model, eps, _ = build_case("w")
    model = model.cuda()
    loss = package_loss("w", model, eps.cuda())
    with torch.no_grad():
        model.flows[1].linear.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified in place"):
        loss.backward()


@pytest.mark.gpu
def test_vae_with_coupled_flows_trains_one_step():
    import helpers_vae as V
    import normflows as nf
    torch.manual_seed(0)
    d = 4
    flows = [nf.flows.CoupledRationalQuadraticSpline(d, 1, 16), nf.flows.LULinearPermute(d),
             nf.flows.CoupledRationalQuadraticSpline(d, 1, 16, reverse_mask=True), nf.flows.LULinearPermute(d)]
    enc = nf.distributions.NNDiagGaussian(nf.nets.MLP([12, 16, 2 * d]))
    dec = nf.distributions.NNBernoulliDecoder(nf.nets.MLP([d, 16, 12]))
    model = nf.NormalizingFlowVAE(V.mvn(d, "cuda"), enc, flows, dec).cuda()
    _perturb_all(model, 3)
    x = (torch.rand(6, 12, device="cuda") > 0.5).float()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    z, log_q, log_p = model(x, 2)
    loss = torch.mean(log_q) - torch.mean(log_p)
    loss.backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    assert all(p.grad.abs().max() > 0 for p in model.flows.parameters())
    opt.step()


def _perturb_all(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.add_(0.05 * torch.randn(p.shape, generator=g).to(p.device))


@pytest.mark.gpu
def test_training_loop_of_model_w_lowers_the_loss():
    import normflows as nf
    model = H.build(nf, "w").cuda()
    _perturb_all(model, 4)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    hist = []
    for _ in range(150):
        opt.zero_grad()
        loss = model.reverse_kld(1024)
        loss.backward()
        opt.step()
        hist.append(loss.item())
    first, last = np.mean(hist[:10]), np.mean(hist[-10:])
    assert np.isfinite(last) and last < first - 0.1, (first, last)
