"""The native sampling backward of coupled-spline / LU stacks (nfb_flow_sampling_backward -> coupled_lu_sampling_backward,
csrc/nfb_api.cu) across the configuration space of tests/test_fused_configs.py, against the fp64 gradient oracle
(oracle/nf_oracle_grad.py sampling_grads).

Configurations: every forward-sweep entry with D >= 2 as a coupling stack (the autoregressive entries re-kinded, so that
the admitted set still covers D x H and H x nb; a Permute layout becomes SLLS), coupled_h320 (no fused plan), coupling
stacks at D = 65, 128, 490 and 784 (layer by layer, up to 392 identity features), LLS, SLLS and LU-only stacks, and a
trainable DiagGaussian base on every third configuration.  Each runs with the whole-stack plan where eligible and layer
by layer, at 1 061 rows and, with an LU map or H >= 256, 4 133 rows (K = rows >= 2048: launch_gemm_tc splits the LU's
dW and the conditioners' weight gradients).  Cotangents g_x and g_ld carry per-row signs and two decades of magnitude;
rows within round-off of an inverse-spline knot, a tail bound or a conditioner ReLU kink along the fp64 sampling pass
get weight 0.  The bars are test_spline_backward_configs.check_grads', scaled by the error of fp32 torch autograd of the
restated sampling pass on the same rows, with this backward's own multiples.

On the CPU: sampling_grads against torch fp64 autograd of the restatement and against goldens w and y; the bars reject
sampling-specific slips; the admitted configurations cover what they claim."""
import itertools

import numpy as np
import pytest
import torch

import helpers_rkl as R
import normflows as nf
from normflows._standalone import StackSamplingFn
from normflows.flows.base import NativeFlow
from oracle import nf_oracle as O
from oracle import nf_oracle_grad as G
from test_coupled_rkl_training import build_case, stack_unrolled
from test_fused_configs import AR, CPL, CPL_R, DS, HS, NBS, OUTSIDE, SWEEP, _blocks, expected_fused, make_model
from test_maf_training import check_golden
from test_reverse_kld_training import layer_spec, sampling_unrolled
from test_spline_backward_configs import KINK_TOL, KNOT_TOL, PERTURB, check_grads, state_dict64

ROWS = 1061          # a ragged last 64-row tile
BIG_ROWS = 4133      # K = rows >= 2048 with few output tiles: launch_gemm_tc's split-K path
SPLIT_K_ROWS = 2048  # the split threshold itself


def _case(name, D, H, nb, layout, seed, kind=CPL, **kw):
    return dict(dict(name=name, kind=kind, D=D, H=H, nb=nb, tail=3.0, pm=False, sigma=0.05, lu_id=True,
                     layout=layout, K=8, bias_mult=1.0, seed=seed), **kw)


def _sampling_twin(i, c):
    """A forward-sweep entry as an admitted stack: coupling blocks (autoregressive entries alternate the two masks), a
    Permute layout as SLLS (two adjacent LU maps between the blocks)."""
    kind = c["kind"] if c["kind"] != AR else (CPL, CPL_R)[i % 2]
    layout = "SLLS" if c["layout"] == "SPSL" else c["layout"]
    name = c["name"] if (kind, layout) == (c["kind"], c["layout"]) else \
        f"{kind}_d{c['D']}_h{c['H']}_b{c['nb']}_{layout.lower()}"
    # large weights only up to D = 33: at D = 63 (coupled_r_d63_h64_b1) the LU gradients of the sampling pass reach
    # 3e8 and fp32 autograd of the restatement itself misses the fp64 ones by 73 % (relative Frobenius)
    sigma = 0.05 if c["sigma"] >= 0.5 and c["D"] > 33 else c["sigma"]
    return dict(c, kind=kind, layout=layout, name=name, sigma=sigma)


ADDED = [
    # H = 320: no fused kernel, so no whole-stack plan
    [c for c in OUTSIDE if c["name"] == "coupled_h320"][0],
    # past the fused kernel's 64 features: layer by layer, 32 .. 392 identity features
    _case("wide_coupled_d65_h320_b4", 65, 320, 4, "SS", 42, tail=1.0),
    _case("wide_coupled_r_d128_h96_b0", 128, 96, 0, "SS", 44, kind=CPL_R, sigma=0.0),
    _case("wide_coupled_d490_h128_b1", 490, 128, 1, "SS", 45),
    _case("wide_coupled_d784_h256_b0", 784, 256, 0, "SS", 46, tail=5.0),
    # one block alone; two adjacent LU maps (no plan), and LU maps alone
    _case("lone_coupled_d5_h64_b1", 5, 64, 1, "S", 54, kind=CPL_R),
    _case("lls_coupled_d17_h128_b1", 17, 128, 1, "LLS", 51, lu_id=False),
    _case("lu_d33", 33, 64, 0, "L", 52, lu_id=False, sigma=0.1),
    _case("lu_lu_d64", 64, 64, 0, "LL", 53, lu_id=False, sigma=0.1),
]
CASES = [dict(c, base=i % 3 == 1) for i, c in
         enumerate([_sampling_twin(i, c) for i, c in enumerate(SWEEP) if c["layout"] != "mixed" and c["D"] >= 2] + ADDED)]
BY_NAME = {c["name"]: c for c in CASES}
EDGE_CFGS = ["coupled_d63_h128_b2", "coupled_r_d2_h192_b3", "lls_coupled_d17_h128_b1"]   # rows 0, 1 and 2 048


def _pattern(cfg):
    return _blocks(cfg)[1]


def _hs(cfg):
    return [H for _, H, _ in _blocks(cfg)[0]] or [0]


def row_counts(cfg):
    return (ROWS, BIG_ROWS) if "L" in _pattern(cfg) or max(_hs(cfg)) >= 256 else (ROWS,)


def expected_units(cfg, use_tc):
    """Units of the whole-stack sampling plan (nfb_api.cu, the fwd_units rule of nfb_flow_finalize): every coupled block
    fused and every LU map directly in front of one or closing the list; else 0 (layer by layer)."""
    pattern = _pattern(cfg)
    fused = expected_fused(cfg)
    ok = use_tc and "S" in pattern and "LL" not in pattern and \
        all(i in fused for i, c in enumerate(pattern) if c == "S")
    return pattern.count("S") if ok else 0


def samp_model(cfg):
    """make_model's stack; with cfg["base"], a trainable DiagGaussian base moved off (0, 1)."""
    model, spec = make_model(cfg)
    if cfg.get("base"):
        q0 = nf.distributions.DiagGaussian(cfg["D"], trainable=True)
        g = torch.Generator().manual_seed(cfg["seed"] + 3)
        with torch.no_grad():
            q0.loc.copy_(0.3 * torch.randn(q0.loc.shape, generator=g))
            q0.log_scale.copy_(0.2 * torch.randn(q0.log_scale.shape, generator=g))
        model = nf.NormalizingFlow(q0, list(model.flows))
    return model, spec


def draws(cfg, rows, seed):
    """Base-like draws; about 2 % of the entries moved beyond the tail bound (both signs)."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((rows, cfg["D"]))
    out = rng.random(z.shape) < 0.02
    z[out] = np.sign(z[out] + 1e-3) * (cfg["tail"] + rng.uniform(0.05, 1.0, out.sum()))
    return z.astype(np.float32)


def cotangents(rows, D, seed):
    """g_x [rows, D] and g_l [rows]: per-row both signs and two decades of magnitude."""
    rng = np.random.default_rng(seed)
    mag = lambda: np.sign(rng.standard_normal(rows)) * 10.0 ** rng.uniform(-1, 1, rows) / max(rows, 1)
    return rng.standard_normal((rows, D)) * mag()[:, None], mag()


def near_discontinuity(spec, sd, z, base=False):
    """[rows] bool: rows within round-off of a point where the sampling gradient jumps, along the fp64 sampling pass:
    a knot of a block's inverse spline (the per-row height knots, computed at x_id), of the unconditional table's
    heights, the tail bounds (the outer knots), or a conditioner ReLU kink at x_id."""
    sd = O._cast(sd, np.float64)
    z = np.asarray(z, np.float64)
    if base:
        z = sd["q0.loc"].reshape(-1) + np.exp(sd["q0.log_scale"].reshape(-1)) * z
    flag = np.zeros(z.shape[0], bool)
    for i, L in enumerate(spec["flows"]):
        p = f"flows.{i}."
        x, _ = O.LAYERS[L["type"]](z, sd, p, L, "forward")
        if L["type"] == "CoupledRationalQuadraticSpline":
            tb = float(L["tail_bound"])
            near = lambda v, knots: (np.abs(v[..., None] - knots) < KNOT_TOL * 2 * tb).reshape(len(v), -1).any(1)
            q = p + "prqct."
            idf, trf = sd[q + "identity_features"].astype(np.int64), sd[q + "transform_features"].astype(np.int64)
            net = q + "transform_net."
            flag |= near(z[:, idf], O._knots(sd[q + "unconditional_transform.unnormalized_heights"], -tb, tb,
                                             O.MIN_BIN_HEIGHT)[0])
            inp = x[:, idf]
            params, acts, n, W = G._net_fwd(inp, sd, net, False)
            sq = lambda a, q: (a * a) @ (W(q) ** 2).T + sd[q + "bias"] ** 2
            s_h = sq(inp, net + "initial_layer.")
            for j in range(n):
                h, a0, t, a1 = acts[j]
                lin = f"{net}blocks.{j}.linear_layers."
                flag |= (np.abs(h) < KINK_TOL * np.sqrt(s_h)).any(1)
                flag |= (np.abs(t) < KINK_TOL * np.sqrt(sq(a0, lin + "0."))).any(1)
                s_h = s_h + sq(a1, lin + "1.")
            K = L.get("num_bins", 8)
            pr = params.reshape(len(z), len(trf), -1)
            sc = np.sqrt(sd[net + "initial_layer.weight"].shape[0])
            flag |= near(z[:, trf], O._knots(pr[..., K:2 * K] / sc, -tb, tb, O.MIN_BIN_HEIGHT)[0])
        z = x
    return flag


def oracle_grads(spec, sd, z, g_x, g_l, base):
    """{state_dict name: gradient, "z": gradient} of sum(g_x * x) + sum(g_l * l): l is the stack's log-det, or with a
    trainable base the sample's log q = log q0 - log_det (sample()'s second output)."""
    if base:
        _, _, g, gz = G.sampling_grads(spec, sd, z, g_x, -g_l, trainable_base=True, g_lq0=g_l)
    else:
        _, _, g, gz = G.sampling_grads(spec, sd, z, g_x, g_l)
    return dict(g, z=gz)


def perturbed_spread(spec, sd, z, g_x, g_l, base):
    """fp64 gradients with every weight and input moved by PERTURB (relative, random), minus the exact ones."""
    rng = np.random.default_rng(0)
    move = lambda v: v * (1 + PERTURB * rng.standard_normal(v.shape))
    sdp = {k: move(v) if v.dtype.kind == "f" else v for k, v in sd.items()}
    a = oracle_grads(spec, sdp, move(np.asarray(z, np.float64)), g_x, g_l, base)
    b = oracle_grads(spec, sd, np.asarray(z, np.float64), g_x, g_l, base)
    return {k: a[k] - b[k] for k in b}


# Bars of this backward (check_grads' BULK_TOL, FRO_MULT, FRO_FLOOR, FRO_CAP, ENTRY_TOL), calibrated on an H100 80GB
# HBM3 (700 W limit) with the rows near a discontinuity left out; see DESIGN.md 3.14 for the measured table.
BARS = (5e-3, 40.0, 3e-3, 1e-2, 3e-2)
# measured: native relative Frobenius 1e-5 .. 1.9e-3 (large weights: up to 0.9, inside the perturbed fp64 spread),
# native / interim 0.5 .. 760 (the largest where the interim error is below 1e-5), worst entry 1.3e-2 of scale
# (wide_coupled_d65_h320_b4); with large weights 96.8 % of one LU tensor lie within 2e-3 of its scale (coupled_d33_h64_b0)


# ---------------------------------------------------------------------------------------------------------------------
# the restatement (torch autograd, any device): the interim reference's fp32 error, and the oracle's fp64 pin
# ---------------------------------------------------------------------------------------------------------------------
def lu_sampling_restated(layer, y):
    """LULinearPermute.forward (sampling direction) on y's device."""
    lin = layer.linear
    n = lin.features
    dt, dev = y.dtype, y.device
    il, iu = torch.tril_indices(n, n, -1, device=dev), torch.triu_indices(n, n, 1, device=dev)
    lower = torch.eye(n, dtype=dt, device=dev).index_put((il[0], il[1]), lin.lower_entries)
    diag = torch.nn.functional.softplus(lin.unconstrained_upper_diag) + lin.eps
    upper = torch.diag(diag).index_put((iu[0], iu[1]), lin.upper_entries)
    t = torch.linalg.solve(lower @ upper, (y - lin.bias).T).T
    return t[:, torch.argsort(layer.permutation._permutation)], -torch.log(diag).sum().expand(y.shape[0])


def restated_grads(model, z, g_x, g_l, base):
    """Gradients of the same loss by autograd of the restated sampling pass, in z's dtype on z's device."""
    params = dict(model.named_parameters())
    for p in params.values():
        p.grad = None
    zz = z.clone().requires_grad_(True)
    with torch.enable_grad():
        if base:
            x, lq = R.replay_forward(model.q0, zz)(zz.shape[0])
        else:
            x, lq = zz, torch.zeros(zz.shape[0], dtype=zz.dtype, device=zz.device)
        for f in model.flows:
            x, ld = sampling_unrolled(layer_spec(f), x, None) if hasattr(f, "prqct") else lu_sampling_restated(f, x)
            lq = lq - ld if base else lq + ld
        ((x * g_x).sum() + (lq * g_l).sum()).backward()
    out = {k: p.grad.double().cpu().numpy() if p.grad is not None else np.zeros(tuple(p.shape))
           for k, p in params.items() if p.requires_grad}
    out["z"] = zz.grad.double().cpu().numpy()
    return out


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the design covers what it claims; the oracle equals torch fp64 autograd and the goldens; the bars reject slips
# ---------------------------------------------------------------------------------------------------------------------
def test_admitted_configurations_cover_the_sweep():
    sweep = [c for c in CASES if c["name"] in {_sampling_twin(i, s)["name"] for i, s in enumerate(SWEEP)}]
    assert all(c["kind"] in (CPL, CPL_R) and c["K"] == 8 and "P" not in _pattern(c) for c in CASES)
    axes = {"D": [d for d in DS if d >= 2], "H": HS, "nb": NBS}
    for a, b in itertools.combinations(axes, 2):
        have = {(c[a], c[b]) for c in sweep}
        want = set(itertools.product(axes[a], axes[b]))
        assert want <= have, (a, b, sorted(want - have))
    assert {c["tail"] for c in sweep} == {0.5, 1.0, 3.0, 8.0}
    assert {c["sigma"] for c in sweep} == {0.0, 1e-3, 0.05, 0.5}
    assert {c["sigma"] for c in CASES if c["name"] in RKL_CFGS} >= {0.5, 0.05}
    assert {c["lu_id"] for c in sweep} == {False, True} and any(c["bias_mult"] != 1 for c in sweep)
    assert {c["layout"] for c in CASES} >= {"SL", "SLx2", "LS", "SSL", "S", "SS", "SLLS", "LLS", "L", "LL"}
    wide = [c for c in CASES if c["D"] > 64]
    assert {c["D"] for c in wide} == {65, 128, 490, 784} and all(expected_units(c, True) == 0 for c in wide)
    n_id = lambda c: max(c["D"] // 2, (c["D"] + 1) // 2)
    assert max(n_id(c) for c in wide) == 392
    assert any(max(_hs(c)) == 320 and c["D"] <= 64 for c in CASES)
    assert any(expected_units(c, True) > 1 for c in CASES) and any(_pattern(c).endswith("L") and expected_units(c, True)
                                                                     for c in CASES)
    base = [c for c in CASES if c["base"]]
    assert 0.3 <= len(base) / len(CASES) <= 0.37
    assert sum(BIG_ROWS in row_counts(c) for c in CASES) >= len(CASES) // 2


PIN_CFGS = ["coupled_d63_h128_b2", "coupled_r_d3_h64_b2", "lls_coupled_d17_h128_b1", "lu_lu_d64",
            "wide_coupled_r_d128_h96_b0"]


@pytest.mark.parametrize("name", PIN_CFGS)
@pytest.mark.parametrize("base", [False, True], ids=["stack", "base"])
def test_oracle_matches_torch_fp64_autograd(name, base):
    """sampling_grads, with draws beyond the tail bound and per-row cotangents, against torch autograd of the
    restated sampling pass (stack_unrolled, and the reparameterised base draw) in fp64 on the CPU."""
    cfg = dict(BY_NAME[name], base=base)
    model, spec = samp_model(cfg)
    model = model.double()
    z = draws(cfg, 97, cfg["seed"] + 2).astype(np.float64)
    assert np.any(np.abs(z) > cfg["tail"])
    g_x, g_l = cotangents(97, cfg["D"], cfg["seed"] + 4)
    ref = oracle_grads(spec, state_dict64(model), z, g_x, g_l, base)
    zt = torch.from_numpy(z).requires_grad_(True)
    with torch.enable_grad():
        x0, lq = R.replay_forward(model.q0, zt)(97) if base else (zt, 0)
        x, ld = stack_unrolled(list(model.flows), x0)
        l = lq - ld if base else ld
        ((x * torch.from_numpy(g_x)).sum() + (l * torch.from_numpy(g_l)).sum()).backward()
    got = {k: p.grad.numpy() for k, p in model.named_parameters() if p.grad is not None}
    got["z"] = zt.grad.numpy()
    assert set(got) == set(ref), set(got) ^ set(ref)
    for k in got:
        np.testing.assert_allclose(ref[k], got[k], rtol=1e-9, atol=1e-9 * np.abs(got[k]).max(), err_msg=k)


@pytest.mark.parametrize("name", ["w", "y"])
def test_oracle_matches_reference_goldens(name):
    """reverse_kld of cases w and y (coupled + LU stacks with a trainable base, tests/golden/make_coupled_rkl_grads.py):
    the oracle's gradients plus the target's term equal the reference's autograd.  (x and z re-evaluate log q by the
    density pass.)"""
    model, eps, gd = build_case(name)
    model = model.double()
    spec = {"flows": [{"type": type(f).__name__, "num_bins": 8, "tail_bound": float(f.tail_bound)}
                      if hasattr(f, "prqct") else {"type": "LULinearPermute"} for f in model.flows]}
    sd = state_dict64(model)
    e = eps.double().numpy()
    n = e.shape[0]
    x, _, _, _ = G.sampling_grads(spec, sd, e, np.zeros_like(e), np.zeros(n), trainable_base=True)
    xt = torch.from_numpy(x).requires_grad_(True)
    with torch.enable_grad():
        model.p.log_prob(xt).sum().backward()
    g_x = -xt.grad.numpy() / n      # loss = mean(log q0 - log_det) - mean(log p(x))
    _, _, grads, _ = G.sampling_grads(spec, sd, e, g_x, np.full(n, -1.0 / n), trainable_base=True,
                                      g_lq0=np.full(n, 1.0 / n))
    names = [k for k, _ in model.named_parameters()]
    assert set(names) <= set(grads), set(names) - set(grads)
    for k in names:
        check_golden(torch.from_numpy(np.asarray(grads[k])), gd, k, 1e-9)


# the native error per configuration (relative Frobenius, H100, rows near a discontinuity left out): the noise on the
# correct gradients in the slip test
NATIVE_FRO = {"coupled_d63_h128_b2": 1.2e-5, "coupled_d3_h128_b3_slls": 2.0e-4}
MUTANT_CFGS = list(NATIVE_FRO)


def _lu_slip(slip, drop_rows):
    """lu_sampling_bwd with one slip."""
    def bwd(z, x, sd, p, L, g_out, g_ld, grads):
        perm = sd[p + "permutation._permutation"].astype(np.int64)
        lower, upper, diag = O.lu_matrices(sd, p, z.dtype)
        n = len(perm)
        t = x[:, perm]
        g_t = g_out[:, np.argsort(perm)] if slip == "perm" else g_out[:, perm]
        w = lower @ upper
        g_y = np.linalg.solve(w if slip == "W^-1" else w.T, g_t.T).T
        keep = slice(drop_rows, None) if slip == "split-K" else slice(None)
        d_w = -(g_y[keep].T @ t[keep])
        grads[p + "linear.bias"] = grads.get(p + "linear.bias", 0) - g_y.sum(0)
        g_lower, g_upper = d_w @ upper.T, lower.T @ d_w
        grads[p + "linear.lower_entries"] = grads.get(p + "linear.lower_entries", 0) + g_lower[np.tril_indices(n, -1)]
        grads[p + "linear.upper_entries"] = grads.get(p + "linear.upper_entries", 0) + g_upper[np.triu_indices(n, 1)]
        ud = sd[p + "linear.unconstrained_upper_diag"].astype(z.dtype)
        ld_term = {"no log-det": 0.0, "log-det sign": 1.0}.get(slip, -1.0) * g_ld.sum() / diag
        g_diag = np.diag(g_upper) + ld_term
        grads[p + "linear.unconstrained_upper_diag"] = grads.get(p + "linear.unconstrained_upper_diag", 0) + \
            g_diag * O.sigmoid(ud)
        return g_y
    return bwd


def _mutants(spec, sd, z0, rows):
    """(what, monkeypatch function) per sampling-specific slip of the native backward."""
    out = [(s, lambda mp, s=s: mp.setitem(G._SAMPLING_BWD, "LULinearPermute", _lu_slip(s, 512)))
           for s in ("W^-1", "perm", "no log-det", "log-det sign", "split-K")]
    orig = G.coupled_rqs_sampling_bwd

    def forward_adjoint(mp):   # the forward spline's adjoint on the transform columns (the first call per block)
        inv, calls = G.rqs_inv_bwd, []

        def f(x, uw, uh, ud, gx, g_ld, tb):
            calls.append(1)
            if len(calls) % 2:
                gy, a, b, c = G.rqs_bwd(x, uw, uh, ud, gx, g_ld, tb)
                return gy, a, b, c
            return inv(x, uw, uh, ud, gx, g_ld, tb)
        mp.setattr(G, "rqs_inv_bwd", f)
    out.append(("forward adjoint", forward_adjoint))

    def at_z(mp):              # the conditioner recomputed at z_id instead of x_id
        net_fwd, held = G._net_fwd, {}

        def bwd(z, x, sd_, p, L, g_out, g_ld, grads):
            held["z"] = z[:, sd_[p + "prqct.identity_features"].astype(np.int64)]
            return orig(z, x, sd_, p, L, g_out, g_ld, grads)
        mp.setattr(G, "_net_fwd", lambda x, sd_, p, masked: net_fwd(held["z"], sd_, p, masked))
        mp.setitem(G._SAMPLING_BWD, "CoupledRationalQuadraticSpline", bwd)
    out.append(("conditioner at z_id", at_z))

    def data_after(mp):        # the conditioner's data gradient added after the identity columns' inverse adjoint
        net_bwd, held = G._net_bwd, {}

        def nb(*a):
            held["g"] = net_bwd(*a)
            return np.zeros_like(held["g"])

        def bwd(z, x, sd_, p, L, g_out, g_ld, grads):
            r = orig(z, x, sd_, p, L, g_out, g_ld, grads)
            r[:, sd_[p + "prqct.identity_features"].astype(np.int64)] += held["g"]
            return r
        mp.setattr(G, "_net_bwd", nb)
        mp.setitem(G._SAMPLING_BWD, "CoupledRationalQuadraticSpline", bwd)
    out.append(("data gradient after", data_after))

    # a block behind an LU map recomputed from the LU's input instead of its output
    zs = [np.asarray(z0, np.float64)]
    for i, L in enumerate(spec["flows"]):
        zs.append(O.LAYERS[L["type"]](zs[-1], O._cast(sd, np.float64), f"flows.{i}.", L, "forward")[0])

    def lu_input(mp):
        def bwd(z, x, sd_, p, L, g_out, g_ld, grads):
            i = int(p.split(".")[1])
            if i and spec["flows"][i - 1]["type"] == "LULinearPermute":
                z = zs[i - 1]
                x = O.coupled_rqs(z, sd_, p, L, "forward")[0]
            return orig(z, x, sd_, p, L, g_out, g_ld, grads)
        mp.setitem(G._SAMPLING_BWD, "CoupledRationalQuadraticSpline", bwd)
    out.append(("block input before its LU", lu_input))
    return out


@pytest.mark.parametrize("name", MUTANT_CFGS)
def test_bars_reject_slips(name):
    """The fp64 oracle with each slip, plus noise at the native path's measured level (the fp32 oracle's own error,
    scaled per tensor to NATIVE_FRO), stands in for a native backward with that slip: check_grads must reject it at the
    sweep's split-K row count and accept the same noise on the correct gradients.  The fp32 oracle plays the interim
    path."""
    cfg = dict(BY_NAME[name], base=False)
    assert "SL" in _pattern(cfg) and cfg["nb"] >= 1 and cfg["sigma"] >= 0.05
    model, spec = samp_model(cfg)
    sd = state_dict64(model)
    rows = BIG_ROWS
    z = draws(cfg, rows, cfg["seed"] + 2)
    g_x, g_l = cotangents(rows, cfg["D"], cfg["seed"] + 4)
    g_l = np.where(near_discontinuity(spec, sd, z), 0.0, g_l)
    g_x = g_x * (g_l != 0)[:, None]
    ref = oracle_grads(spec, sd, z.astype(np.float64), g_x, g_l, False)
    with np.errstate(all="ignore"):
        g32 = oracle_grads(spec, O._cast(sd, np.float32), z, g_x.astype(np.float32), g_l.astype(np.float32), False)
    noise = {}
    for k in ref:
        d = np.asarray(g32[k], np.float64) - ref[k]
        nd = np.linalg.norm(d)
        noise[k] = d * (NATIVE_FRO[name] * np.linalg.norm(ref[k]) / nd) if nd > 0 else d
    check_grads({k: ref[k] + noise[k] for k in ref}, ref, g32, f"{name} correct", bars=BARS)
    mutants = _mutants(spec, sd, z, rows)
    assert len(mutants) == 9
    for what, patch in mutants:
        mp = pytest.MonkeyPatch()
        try:
            patch(mp)
            bad = oracle_grads(spec, sd, z.astype(np.float64), g_x, g_l, False)
        finally:
            mp.undo()
        assert any(not np.allclose(bad[k], ref[k], rtol=1e-12, atol=0) for k in ref), what
        with pytest.raises(AssertionError):
            check_grads({k: bad[k] + noise[k] for k in ref}, ref, g32, f"{name} {what}", bars=BARS)


def test_forward_and_log_det_refuses_a_stack_without_sampling_backward():
    """Under grad, an all-native stack whose sampling direction has no native backward raises before any launch: its
    transform would return values with no autograd node (the parameters' gradients silently missing)."""
    Cq, LU = nf.flows.CoupledRationalQuadraticSpline, nf.flows.LULinearPermute
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    for flows in ([nf.flows.AutoregressiveRationalQuadraticSpline(4, 1, 16), LU(4)],
                  [Cq(4, 1, 16), nf.flows.Permute(4), Cq(4, 1, 16), LU(4)], [Cq(4, 1, 16, num_bins=10), LU(4)]):
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(4), flows)
        assert model._stack() is not None and not model._stack_sampling_backward()
        with torch.enable_grad(), pytest.raises(NotImplementedError, match=msg):
            model.forward_and_log_det(torch.zeros(3, 4))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def paths(monkeypatch):
    """Records every StackSamplingFn backward (the one native sampling backward); restores the tensor-core switch."""
    taken = []
    orig = StackSamplingFn.backward

    def rec(ctx, *g):
        taken.append(True)
        return orig(ctx, *g)
    monkeypatch.setattr(StackSamplingFn, "backward", staticmethod(rec))
    yield taken
    NativeFlow.use_tensor_cores = True


def gpu_grads(model, z, g_x, g_l, base):
    """{parameter name: gradient, "z": gradient} of sum(g_x * x) + sum(g_l * l) on the native path: l = log_det of
    forward_and_log_det(z), or with a trainable base log q of sample() on the replayed draws z."""
    model.zero_grad(set_to_none=True)
    zz = torch.from_numpy(np.ascontiguousarray(z, np.float32)).cuda().requires_grad_(True)
    with torch.enable_grad():
        if base:
            model.q0.forward = R.replay_forward(model.q0, zz)
            x, l = model.sample(zz.shape[0])
        else:
            x, l = model.forward_and_log_det(zz)
        assert x.requires_grad and l.requires_grad and x.grad_fn is not None
        ((x * torch.from_numpy(g_x).float().cuda()).sum() + (l * torch.from_numpy(g_l).float().cuda()).sum()).backward()
    if base:
        del model.q0.forward
    out = {k: p.grad.double().cpu().numpy() for k, p in model.named_parameters() if p.grad is not None}
    out["z"] = zz.grad.double().cpu().numpy()
    return out, x.detach(), l.detach()


def _interim(model, z, g_x, g_l, base):
    dev = torch.device("cuda")
    return restated_grads(model, torch.from_numpy(np.ascontiguousarray(z, np.float32)).to(dev),
                          torch.from_numpy(g_x).float().to(dev), torch.from_numpy(g_l).float().to(dev), base)


def _inputs(cfg, spec, sd, rows):
    z = draws(cfg, rows, cfg["seed"] + 2)
    g_x, g_l = cotangents(rows, cfg["D"], cfg["seed"] + 4)
    keep = ~near_discontinuity(spec, sd, z, cfg["base"]) if rows else np.ones(0, bool)
    # (past 64 features a row has thousands of knots: at D = 784, 64 % of the rows are clear of all of them)
    assert rows == 0 or keep.mean() >= (0.9 if cfg["D"] <= 64 else 0.6), f"{cfg['name']}: {keep.mean():.3f} kept"
    return z, g_x * keep[:, None], g_l * keep


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_sampling_backward_matches_oracle(name, paths):
    cfg = BY_NAME[name]
    model, spec = samp_model(cfg)
    sd = state_dict64(model)
    model = model.cuda()
    rows_list = row_counts(cfg) + ((0, 1, SPLIT_K_ROWS) if name in EDGE_CFGS else ())
    for rows in rows_list:
        z, g_x, g_l = _inputs(cfg, spec, sd, rows)
        ref = oracle_grads(spec, sd, z.astype(np.float64), g_x, g_l, cfg["base"]) if rows else None
        interim = _interim(model, z, g_x, g_l, cfg["base"]) if rows > 1 else None
        spread = perturbed_spread(spec, sd, z, g_x, g_l, cfg["base"]) if cfg["sigma"] >= 0.5 and rows > 1 else None
        for use_tc in (True, False):
            NativeFlow.use_tensor_cores = use_tc
            paths.clear()
            got, _, _ = gpu_grads(model, z, g_x, g_l, cfg["base"])
            units = model._stack().sampling_units()
            assert paths == [True], f"{name}: backward {paths}"
            assert units == expected_units(cfg, use_tc), f"{name} tc={use_tc}: {units} plan units"
            path = f"plan x{units}" if units else "layer by layer"
            if rows == 0:
                assert got["z"].shape == (0, cfg["D"]) and all(not np.any(v) for v in got.values()), name
                assert set(got) == {k for k, p in model.named_parameters()} | {"z"}
                continue
            if rows == 1:   # one row: no interim spread to scale by; every entry within 1e-3 of its tensor's scale
                for k, r in ref.items():
                    assert np.abs(got[k] - r).max() <= 1e-3 * np.abs(r).max(), (name, k)
                continue
            ratio, fro, entry, frac = check_grads(got, ref, interim, f"{name} rows {rows} {path}", spread, bars=BARS)
            split = " split-K dW" if rows >= SPLIT_K_ROWS and "L" in _pattern(cfg) else ""
            print(f"[spline-samp-bwd] {name} rows={rows} {path}{split}: worst native/interim Frobenius {ratio:.1f}, "
                  f"rel. Frobenius {fro:.2e}, entry/scale {entry:.2e}, bulk {frac:.4f}")
            if cfg["sigma"] == 0.0 and "S" in _pattern(cfg):   # zero final layers: nothing reaches the hidden layers
                for k in got:
                    if "transform_net" in k and ("initial_layer" in k or ".blocks." in k):
                        assert not np.any(got[k]) and not np.any(ref[k]), f"{name} {k}"


@pytest.mark.gpu
def test_exact_zeros(paths):
    """Identity and transform columns beyond the tails at the first block: that table row and those 23 conditioner
    outputs get exactly zero gradient; all-zero cotangents give exactly zero gradients."""
    cfg = dict(BY_NAME["coupled_d63_h128_b2"], base=False)
    model, spec = samp_model(cfg)
    sd = state_dict64(model)
    q = model.flows[0].prqct
    idf, trf = q.identity_features.tolist(), q.transform_features.tolist()
    z, g_x, g_l = _inputs(cfg, spec, sd, ROWS)
    for c in (idf[0], idf[-1], trf[0], trf[-1]):
        z[:, c] = np.sign(z[:, c] + 0.5) * (cfg["tail"] + 0.25 + np.abs(z[:, c]))
    model = model.cuda()
    for use_tc in (True, False):
        NativeFlow.use_tensor_cores = use_tc
        got, _, _ = gpu_grads(model, z, g_x, g_l, False)
        p = "flows.0.prqct."
        for t in (0, len(trf) - 1):
            for k in ("transform_net.final_layer.weight", "transform_net.final_layer.bias"):
                assert not np.any(got[p + k][23 * t:23 * t + 23]), (k, t)
        for j in (0, len(idf) - 1):
            for n in ("widths", "heights", "derivatives"):
                assert not np.any(got[f"{p}unconditional_transform.unnormalized_{n}"][j]), (n, j)
        assert np.any(got[p + "transform_net.final_layer.weight"][23:46])
        zero, _, _ = gpu_grads(model, z, np.zeros_like(g_x), np.zeros_like(g_l), False)
        assert all(not np.any(v) for v in zero.values())
    assert paths == [True] * 4


@pytest.mark.gpu
def test_frozen_subsets(paths):
    """Frozen LU maps, then also one conditioner, then every parameter with z still requiring grad: the remaining
    gradients equal the full run's (to 1e-6 of each tensor's scale: the atomics reorder sums), frozen tensors get none."""
    cfg = dict(BY_NAME["coupled_d63_h128_b2"], base=False)
    model, spec = samp_model(cfg)
    model = model.cuda()
    z = draws(cfg, ROWS, 11)
    g_x, g_l = cotangents(ROWS, cfg["D"], 12)
    full, _, _ = gpu_grads(model, z, g_x, g_l, False)
    pattern = _pattern(cfg)
    params = dict(model.named_parameters())
    lu = [k for k in params if pattern[int(k.split(".")[1])] == "L"]
    cond = [k for k in params if k.startswith("flows.0.prqct.transform_net.")]
    assert lu and cond
    for frozen in (lu, lu + cond, list(params)):
        for k, p in params.items():
            p.requires_grad_(k not in frozen)
        got, _, _ = gpu_grads(model, z, g_x, g_l, False)
        assert set(got) == set(full) - set(frozen), sorted(set(got) ^ (set(full) - set(frozen)))
        for k in got:
            assert np.abs(got[k] - full[k]).max() <= 1e-6 * np.abs(full[k]).max(), (k, len(frozen))
    assert paths == [True] * 4


@pytest.mark.gpu
def test_shared_layer_gets_the_sum(paths):
    """One LULinearPermute module at two places of the stack: its parameters' gradients are the sum of both uses."""
    cfg = dict(BY_NAME["coupled_d63_h128_b2"], base=False)
    model, spec = samp_model(cfg)
    flows = list(model.flows)
    assert _pattern(cfg) == "SLSL"
    flows[3] = flows[1]
    model = nf.NormalizingFlow(model.q0, flows)
    sd = state_dict64(model)
    assert "flows.3.linear.bias" in sd
    z, g_x, g_l = _inputs(cfg, spec, sd, ROWS)
    ref = oracle_grads(spec, sd, z.astype(np.float64), g_x, g_l, False)
    for k in [k for k in ref if k.startswith("flows.3.")]:
        ref["flows.1." + k[len("flows.3."):]] = ref["flows.1." + k[len("flows.3."):]] + ref.pop(k)
    model = model.cuda()
    interim = _interim(model, z, g_x, g_l, False)
    for use_tc in (True, False):
        NativeFlow.use_tensor_cores = use_tc
        got, _, _ = gpu_grads(model, z, g_x, g_l, False)
        check_grads(got, ref, interim, f"shared LU tc={use_tc}", bars=BARS)
    assert paths == [True] * 2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["coupled_d63_h128_b2", "coupled_r_d3_h256_b1", "wide_coupled_d490_h128_b1"])
def test_values_identical_with_and_without_grad(name):
    cfg = dict(BY_NAME[name], base=False)
    model = samp_model(cfg)[0].cuda()
    z = torch.from_numpy(draws(cfg, ROWS, 13)).cuda()
    for use_tc in (True, False):
        NativeFlow.use_tensor_cores = use_tc
        with torch.no_grad():
            a, la = model.forward_and_log_det(z)
        with torch.enable_grad():
            b, lb = model.forward_and_log_det(z.clone().requires_grad_(True))
        assert b.grad_fn is not None and torch.equal(a, b.detach())
        # the log-det may differ in its last bits between two calls on these stacks (seen on coupled_d63_h128_b2 and
        # wide_coupled_d490_h128_b1, not traced)
        assert torch.allclose(la, lb.detach(), rtol=1e-6, atol=1e-6)
    NativeFlow.use_tensor_cores = True


class GaussTarget(torch.nn.Module):
    """A correlated Gaussian target: log p(x) = -1/2 sum ((x_j - 0.4 x_{j-1}) / s_j)^2."""

    def __init__(self, D):
        super().__init__()
        self.s = torch.linspace(0.7, 1.5, D, dtype=torch.float64)

    def log_prob(self, x):
        r = x.clone()
        r[:, 1:] = x[:, 1:] - 0.4 * x[:, :-1]
        return -0.5 * torch.sum((r / self.s.to(x)) ** 2, 1)


RKL_CFGS = ["coupled_d33_h64_b0", "coupled_d63_h128_b2", "coupled_r_d2_h192_b3", "lls_coupled_d17_h128_b1"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", RKL_CFGS)
def test_reverse_kld_end_to_end(name, paths):
    """reverse_kld on the replayed draws, trainable base: every .grad against the oracle's plus the target's and the
    base's terms (loss = mean(log q0 - log_det) - mean(log p(x)))."""
    cfg = dict(BY_NAME[name], base=True)
    model, spec = samp_model(cfg)
    model.p = GaussTarget(cfg["D"])
    sd = state_dict64(model)
    n = ROWS
    eps = draws(cfg, n, cfg["seed"] + 7)
    keep = ~near_discontinuity(spec, sd, eps, True)
    eps = eps[keep]
    n = len(eps)
    x, _, _, _ = G.sampling_grads(spec, sd, eps.astype(np.float64), np.zeros(eps.shape), np.zeros(n),
                                  trainable_base=True)
    xt = torch.from_numpy(x).requires_grad_(True)
    with torch.enable_grad():
        model.p.log_prob(xt).sum().backward()
    ref = oracle_grads(spec, sd, eps.astype(np.float64), -xt.grad.numpy() / n, np.full(n, 1.0 / n), True)
    ref.pop("z")
    interim_model = samp_model(cfg)[0].cuda()
    interim = _interim(interim_model, eps, -xt.grad.numpy() / n, np.full(n, 1.0 / n), True)
    interim.pop("z")
    model = model.cuda()
    model.p.s = model.p.s.cuda()
    model.q0.forward = R.replay_forward(model.q0, torch.from_numpy(eps).cuda())
    with torch.enable_grad():
        loss = model.reverse_kld(n)
        loss.backward()
    del model.q0.forward
    assert paths == [True]
    got = {k: p.grad.double().cpu().numpy() for k, p in model.named_parameters()}
    spread = perturbed_spread(spec, sd, eps, -xt.grad.numpy() / n, np.full(n, 1.0 / n), True) \
        if cfg["sigma"] >= 0.5 else None
    if spread is not None:
        spread.pop("z")
    check_grads(got, ref, interim, f"{name} reverse_kld", spread, bars=BARS)


def _not_admitted():
    ar = [c for c in SWEEP if c["kind"] == AR and c["D"] >= 2][:2]
    spsl = [c for c in SWEEP if c["layout"] == "SPSL" and c["kind"] != AR][:1]
    k10 = [c for c in OUTSIDE if c["name"] == "coupled_k10"]
    return [dict(c, base=False) for c in ar + spsl + k10] + [dict(name="coupled_context", D=6, seed=61, base=False)]


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", _not_admitted(), ids=lambda c: c["name"])
def test_stacks_without_sampling_backward_raise(cfg):
    """forward_and_log_det, sample and reverse_kld under grad on stacks outside coupled_lu_sampling_backward: each
    raises the documented error; none returns a result detached from the parameters."""
    if cfg["name"] == "coupled_context":
        flows = [nf.flows.CoupledRationalQuadraticSpline(cfg["D"], 1, 64, num_context_channels=3),
                 nf.flows.LULinearPermute(cfg["D"])]
        model = nf.NormalizingFlow(nf.distributions.DiagGaussian(cfg["D"]), flows)
    else:
        model = samp_model(cfg)[0]
    model.p = GaussTarget(cfg["D"])
    model = model.cuda()
    model.p.s = model.p.s.cuda()
    msg = "gradients through the sampling direction are not on the CUDA path yet"
    z = torch.from_numpy(draws(dict(cfg, tail=3.0), 64, 1)).cuda()
    calls = {"forward_and_log_det": lambda: model.forward_and_log_det(z.clone().requires_grad_(True)),
             "sample": lambda: model.sample(64), "reverse_kld": lambda: model.reverse_kld(64)}
    for what, call in calls.items():
        with torch.enable_grad():
            try:
                out = call()
            except NotImplementedError as e:
                assert msg in str(e), (what, str(e))
                print(f"[spline-samp-bwd] {cfg['name']} {what}: raises")
                continue
        out = out if isinstance(out, tuple) else (out,)
        assert False, f"{cfg['name']} {what} returned {[o.grad_fn for o in out]} instead of raising"
