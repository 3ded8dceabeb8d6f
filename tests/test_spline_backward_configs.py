"""The native density backward of spline stacks (nfb_flow_log_prob_backward, csrc/nfb_api.cu) across the configuration
space of tests/test_fused_configs.py, against the fp64 gradient oracle (oracle/nf_oracle_grad.py log_prob_grads), with
per-row loss weights of both signs (a wrong row of g_logq shows; forward_kld's uniform weights hide it).  Added here:
spline-only stacks past the fused kernel's 64 features (layer-by-layer recompute on gemm_tc, coupling blocks with up
to 392 identity features), [S, Permute, S, LU] stacks at 33 and 64 features (a one-Permute affine group on the wide
path inside a spline stack) and a trainable DiagGaussian base.  Every GPU case asserts which backward ran (native, or
the interim torch path for num_bins != 8) and is judged against the oracle with bars scaled by the interim path's own
fp32 error on the same rows; rows within round-off of a knot, tail bound or ReLU kink are left out of the loss
(near_discontinuity).  On the CPU: the oracle extensions against torch's fp64 autograd, and the bars reject
gradients with specific slips."""
import numpy as np
import pytest
import torch

import normflows as nf
import normflows._autograd as A
from normflows._autograd import DensityFn
from oracle import nf_oracle as O
from oracle import nf_oracle_grad as G
from test_fused_configs import AR, CPL, CPL_R, MUTANT_CFGS, OUTSIDE, SWEEP, _blocks, check_log_prob, inputs, make_model

ROWS = 1061          # a ragged last 64-row tile
BIG_ROWS = 4133      # weight gradients with K = rows >= 2048 (launch_gemm_tc's split-K path), on the H >= 256 nets


def _wide(name, kind, D, H, nb, layout, seed, **kw):
    return dict(dict(name=name, kind=kind, D=D, H=H, nb=nb, tail=3.0, pm=seed % 2 == 0, sigma=0.05, lu_id=True,
                     layout=layout, K=8, bias_mult=1.0, seed=seed), **kw)


# spline blocks and Permute past the fused kernel's D <= 64 (LULinearPermute stops at 64 features)
WIDE = [
    _wide("wide_ar_d65_h96_b0", AR, 65, 96, 0, "SS", 41),
    _wide("wide_coupled_d65_h320_b4", CPL, 65, 320, 4, "SS", 42, tail=1.0),
    _wide("wide_ar_d128_h320_b4", AR, 128, 320, 4, "SPS", 43, sigma=1e-3),
    _wide("wide_coupled_r_d128_h96_b0", CPL_R, 128, 96, 0, "SPS", 44, sigma=0.0),
    # 245 identity features per block: the first count whose table gradient passes the LU-sized scratch
    _wide("wide_coupled_d490_h128_b1", CPL, 490, 128, 1, "SS", 45),
    _wide("wide_coupled_d784_h256_b0", CPL, 784, 256, 0, "SS", 46, tail=5.0),
]
# a Permute inside a spline stack wider than the affine stack kernel's 16 features
SPSL = [
    _wide("spsl_coupled_d33_h128_b1", CPL, 33, 128, 1, "SPSL", 47, lu_id=False),
    _wide("spsl_ar_d64_h256_b2", AR, 64, 256, 2, "SPSL", 48, tail=1.0),
]
# every third configuration gets a trainable base
CASES = [dict(c, base=i % 3 == 1) for i, c in enumerate(SWEEP + WIDE + SPSL + OUTSIDE)]
BY_NAME = {c["name"]: c for c in CASES}


def _hs(cfg):
    return [H for _, H, _ in _blocks(cfg)[0]]


def row_counts(cfg):
    return (ROWS, BIG_ROWS) if max(_hs(cfg)) >= 256 else (ROWS,)


def bwd_model(cfg):
    """make_model's stack and spec; with cfg["base"], a trainable DiagGaussian base moved off (0, 1)."""
    model, spec = make_model(cfg)
    if cfg.get("base"):
        q0 = nf.distributions.DiagGaussian(cfg["D"], trainable=True)
        g = torch.Generator().manual_seed(cfg["seed"] + 3)
        with torch.no_grad():
            q0.loc.copy_(0.3 * torch.randn(q0.loc.shape, generator=g))
            q0.log_scale.copy_(0.2 * torch.randn(q0.log_scale.shape, generator=g))
        model = nf.NormalizingFlow(q0, list(model.flows))
    return model, spec


def row_weights(rows, seed):
    """Both signs, magnitudes over two decades."""
    rng = np.random.default_rng(seed)
    return rng.standard_normal(rows) * 10.0 ** rng.uniform(-1, 1, rows) / max(rows, 1)


def state_dict64(model):
    return {k: v.detach().cpu().numpy().astype(np.float64) if v.dtype.is_floating_point else v.detach().cpu().numpy()
            for k, v in model.state_dict().items()}


def oracle_grads(spec, sd, x, w, base):
    lp, g, gx = G.log_prob_grads(spec, sd, x, w, trainable_base=base)
    return dict(g, x=gx)


# The gradient of log q is discontinuous where a spline input crosses a knot or a tail bound (the log-det's derivative
# jumps) and where a ReLU's pre-activation crosses zero.  A row whose fp64 values lie closer to such a point than the
# kernels' round-off may be evaluated on the other side, and its whole contribution moves: one element 3.3e-7 from a
# knot of wide_coupled_d784_h256_b0 moves that block's gradients by 7e-3 (relative Frobenius) in the fp64 oracle itself.
# Such rows get weight 0 in both the kernel's and the oracle's loss; every other row is judged at the round-off level.
KNOT_TOL = 2e-5      # x 2 tail: distance of a spline input to a knot or tail bound
KINK_TOL = 1e-5      # x the root sum of squares of the terms that make the pre-activation


def near_discontinuity(spec, sd, x):
    """[rows] bool: rows within KNOT_TOL / KINK_TOL of a discontinuity of the gradient, in the fp64 density pass (a ReLU
    input's round-off grows with the root sum of squares of the terms it adds up)."""
    sd = O._cast(sd, np.float64)
    z = np.asarray(x, np.float64)
    flag = np.zeros(z.shape[0], bool)
    flows = spec["flows"]
    for i in range(len(flows) - 1, -1, -1):
        L, p = flows[i], f"flows.{i}."
        if L["type"] in ("AutoregressiveRationalQuadraticSpline", "CoupledRationalQuadraticSpline"):
            tb = float(L["tail_bound"])
            near = lambda v, knots: (np.abs(v[..., None] - knots) < KNOT_TOL * 2 * tb).reshape(len(v), -1).any(1)
            if L["type"] == "AutoregressiveRationalQuadraticSpline":
                net, inp, xs, masked = p + "mprqat.autoregressive_net.", z, z, True
            else:
                q = p + "prqct."
                idf, trf = sd[q + "identity_features"].astype(np.int64), sd[q + "transform_features"].astype(np.int64)
                net, inp, xs, masked = q + "transform_net.", z[:, idf], z[:, trf], False
                flag |= near(z[:, idf], O._knots(sd[q + "unconditional_transform.unnormalized_widths"], -tb, tb,
                                                 O.MIN_BIN_WIDTH)[0])
            params, acts, n, W = G._net_fwd(inp, sd, net, masked)
            sq = lambda a, q: (a * a) @ (W(q) ** 2).T + sd[q + "bias"] ** 2   # sum of squared terms
            s_h = sq(inp, net + "initial_layer.")
            for j in range(n):
                h, a0, t, a1 = acts[j]
                lin = f"{net}blocks.{j}.linear_layers."
                flag |= (np.abs(h) < KINK_TOL * np.sqrt(s_h)).any(1)
                flag |= (np.abs(t) < KINK_TOL * np.sqrt(sq(a0, lin + "0."))).any(1)
                s_h = s_h + sq(a1, lin + "1.")
            pr = params.reshape(len(z), xs.shape[1], -1)
            sc = 1.0 if masked else np.sqrt(sd[net + "initial_layer.weight"].shape[0])
            flag |= near(xs, O._knots(pr[..., :L.get("num_bins", 8)] / sc, -tb, tb, O.MIN_BIN_WIDTH)[0])
        z, _ = O.LAYERS[L["type"]](z, sd, p, L, "inverse")
    return flag


def loss_weights(spec, sd, x, seed):
    """row_weights with the rows near a discontinuity set to 0."""
    return np.where(near_discontinuity(spec, sd, x), 0.0, row_weights(len(x), seed))


# ---------------------------------------------------------------------------------------------------------------------
# the bars (also applied, on the CPU, to mutated gradients: they must reject those)
# ---------------------------------------------------------------------------------------------------------------------
# Bars, calibrated on an H100 80GB HBM3 (700 W limit) with the rows near a discontinuity left out (near_discontinuity):
# the native path's GEMMs are split-bf16 (~2^-17 per product, nfb_gemm_tc.cu), the interim torch path's fp32.
BULK_FRAC, BULK_TOL = 0.97, 2e-3     # >= 97 % of the entries within 2e-3 of the tensor's scale ...
BULK_MIN = 34                        # ... on tensors of at least 34 entries (below, 97 % means every entry)
FRO_MULT, FRO_FLOOR, FRO_CAP = 40.0, 5e-4, 1e-2   # relative Frobenius: <= FRO_MULT x the interim path's, floored
ENTRY_TOL = 1e-2                     # worst single entry / scale
# measured: native relative Frobenius 5e-6 .. 2.6e-4 (large weights: up to 3.4e-2), native / interim 3 .. 90 with two
# outliers of 260 and 340 where the interim error is 4e-8 and 1e-7; worst entry 2.6e-3 of scale (large weights: 4.4e-2)
PERTURB = 2.0 ** -17                 # the split-bf16 product's relative error


def perturbed_spread(spec, sd, x, w, base):
    """An fp64 evaluation at the kernels' precision: every weight and input moved by PERTURB (relative, random), minus
    the exact gradients.  With large weights the gradients are this sensitive; an fp32 run (the interim path) can
    happen to land closer."""
    rng = np.random.default_rng(0)
    move = lambda v: v * (1 + PERTURB * rng.standard_normal(v.shape))
    sdp = {k: move(v) if v.dtype.kind == "f" else v for k, v in sd.items()}
    a = oracle_grads(spec, sdp, move(np.asarray(x, np.float64)), w, base)
    b = oracle_grads(spec, sd, np.asarray(x, np.float64), w, base)
    return {k: a[k] - b[k] for k in b}


def check_grads(got, ref, interim, what, spread=None, bars=None):
    """Per tensor (every parameter gradient and "x"), scale = max|ref|: the bulk of the entries within BULK_TOL * scale
    (tensors of BULK_MIN entries or more), the relative Frobenius error within FRO_MULT x the interim path's (never
    below FRO_FLOOR nor above FRO_CAP), the worst entry within ENTRY_TOL * scale.  A reference that is exactly zero
    must be matched exactly.  With large weights an evaluation at the kernels' precision itself can miss by more
    (`spread`: perturbed_spread): there each entry may also miss by 10 x the larger of the interim path's and that
    spread's error on it, and the Frobenius and entry bars are at least 10 x theirs, as test_fused_configs.check_layer
    does for the forward.  Returns the worst native / interim Frobenius ratio, relative
    Frobenius error, entry / scale and bulk fraction over the tensors.  bars: (BULK_TOL, FRO_MULT, FRO_FLOOR, FRO_CAP,
    ENTRY_TOL) of another backward (default: this file's)."""
    bulk_tol, fro_mult, fro_floor, fro_cap, entry_tol = bars or (BULK_TOL, FRO_MULT, FRO_FLOOR, FRO_CAP, ENTRY_TOL)
    assert set(got) == set(ref), f"{what}: gradients for {sorted(set(got) ^ set(ref))}"
    worst = [0.0, 0.0, 0.0, 1.0]
    for k, r in ref.items():
        r = np.asarray(r, np.float64)
        d = np.asarray(got[k], np.float64) - r
        assert d.shape == r.shape and np.all(np.isfinite(d)), f"{what} {k}: shape {d.shape} vs {r.shape} or non-finite"
        scale = float(np.abs(r).max()) if r.size else 0.0
        if scale == 0.0:
            assert not np.any(d), f"{what} {k}: {np.count_nonzero(d)} non-zero entries where the gradient is exactly 0"
            continue
        di = np.asarray(interim[k], np.float64) - r
        nr = np.linalg.norm(r)
        fro, fro_i = np.linalg.norm(d) / nr, np.linalg.norm(di) / nr
        e, e_i = np.abs(d).max() / scale, np.abs(di).max() / scale
        tol = bulk_tol * scale
        fro_bar, e_bar = min(fro_cap, max(fro_floor, fro_mult * fro_i)), entry_tol
        if spread is not None:
            ds = np.maximum(np.abs(di), np.abs(spread[k]))
            tol = np.maximum(tol, 10 * ds)
            fro_bar, e_bar = max(fro_bar, 10 * np.linalg.norm(ds) / nr), max(e_bar, 10 * ds.max() / scale)
        frac = float(np.mean(np.abs(d) <= tol))
        assert (frac >= BULK_FRAC or r.size < BULK_MIN) and fro <= fro_bar and e <= e_bar, \
            f"{what} {k}: {frac:.4f} within {bulk_tol:g} x scale, rel. Frobenius {fro:.3e} (bar {fro_bar:.3e}, " \
            f"interim {fro_i:.3e}), worst entry {e:.3e} x scale (bar {e_bar:.3e}), scale {scale:.3e}"
        worst = [max(worst[0], fro / max(fro_i, 1e-300)), max(worst[1], fro), max(worst[2], e), min(worst[3], frac)]
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the design covers what it claims; the oracle extensions equal torch's fp64 autograd; the bars reject slips
# ---------------------------------------------------------------------------------------------------------------------
def test_additions_cover_what_they_claim():
    wide = [c for c in CASES if c["name"].startswith("wide_")]
    assert {(c["D"], c["H"], c["nb"]) for c in wide if c["D"] in (65, 128)} >= \
        {(65, 96, 0), (65, 320, 4), (128, 320, 4), (128, 96, 0)}
    assert all(set(_blocks(c)[1]) <= {"S", "P"} and c["D"] > 64 for c in wide)
    assert any("P" in _blocks(c)[1] for c in wide)
    assert {c["kind"] for c in wide} == {AR, CPL, CPL_R}
    # the coupling widths: 245 identity features (first past the old scratch) and the D = 784 stack at H = 256
    n_id = lambda c: max(c["D"] // 2, (c["D"] + 1) // 2) if c["kind"] != AR else 0
    assert any(c["kind"] != AR and c["D"] == 490 and min(c["D"] // 2, (c["D"] + 1) // 2) == 245 for c in wide)
    assert any(c["D"] == 784 and c["H"] == 256 and n_id(c) == 392 for c in wide)
    assert {c["D"] for c in SPSL} == {33, 64} and all(c["layout"] == "SPSL" for c in SPSL)
    assert {c["sigma"] for c in wide} >= {0.0, 1e-3, 0.05}
    base = [c for c in CASES if c["base"]]
    assert 0.3 <= len(base) / len(CASES) <= 0.37
    assert {c["kind"] for c in base} >= {AR, CPL, CPL_R} and any(c["name"].startswith("wide_") for c in base)
    assert any(c["K"] != 8 for c in CASES) and any(c["sigma"] == 0.0 for c in CASES)
    assert any(max(_hs(c)) >= 256 for c in wide) and any(max(_hs(c)) < 256 for c in wide)
    # the oracle pins reach both kinds, a Permute and a wide stack
    assert {BY_NAME[n]["kind"] for n in PIN_CFGS} >= {AR, CPL} and any(BY_NAME[n]["D"] > 64 for n in PIN_CFGS)
    assert any("P" in _blocks(BY_NAME[n])[1] for n in PIN_CFGS)


PIN_CFGS = ["coupled_d3_h128_b3", "ar_d7_h256_b2", "wide_coupled_r_d128_h96_b0", "spsl_coupled_d33_h128_b1"]


@pytest.mark.parametrize("name", PIN_CFGS)
def test_oracle_extensions_match_torch_fp64_autograd(name):
    """log_prob_grads with random per-row weights, the Permute adjoint and the trainable base's gradients against
    torch autograd of normflows._autograd.log_prob on the same model in fp64 on the CPU."""
    cfg = dict(BY_NAME[name], base=True)
    model, spec = bwd_model(cfg)
    model = model.double()
    x = inputs(cfg["D"], 97, cfg["seed"] + 2).astype(np.float64)
    w = row_weights(97, cfg["seed"] + 4)
    _, gref, gx = G.log_prob_grads(spec, state_dict64(model), x, w, trainable_base=True)
    xt = torch.from_numpy(x).requires_grad_(True)
    with torch.enable_grad():
        (torch.from_numpy(w) * A.log_prob(model, xt)).sum().backward()
    got = {k: p.grad.numpy() for k, p in model.named_parameters()}
    assert set(got) == set(gref) and {"q0.loc", "q0.log_scale"} <= set(got)
    for k in got:
        np.testing.assert_allclose(gref[k], got[k], rtol=1e-9, atol=1e-9 * np.abs(got[k]).max(), err_msg=k)
    np.testing.assert_allclose(gx, xt.grad.numpy(), rtol=1e-9, atol=1e-9 * np.abs(gx).max())


# the noise on the correct gradients in the mutant test: the fp32 oracle's own error, scaled per tensor to the native
# path's relative Frobenius error measured on that configuration (H100, rows near a discontinuity left out)
NATIVE_FRO = {"ar_d7_h256_b2": 9.8e-5, "coupled_d63_h128_b2": 1.3e-5, "coupled_d3_h128_b3": 6.8e-5}


def _mutants(cfg):
    """(what, context manager factory) per slip; each factory monkeypatches the oracle to make that slip."""
    blocks, pattern = _blocks(cfg)
    kind, H, nb = blocks[0]
    coupled = kind != AR
    net = "flows.0.prqct.transform_net." if coupled else "flows.0.mprqat.autoregressive_net."
    out = []

    def patch(fn):
        def ctx():
            mp = pytest.MonkeyPatch()
            fn(mp)
            return mp
        return ctx

    # 1. g_logq replaced by its mean: the caller passes the mean weight (see test_bars_reject_slips)
    out.append(("mean g_logq", None))
    if nb:
        def relu(mp):   # 2. the last residual block's inner ReLU mask dropped in dgrad (only in the first layer's net)
            orig_bwd = G._net_bwd

            def net_bwd(g_out, acts, n, W, sd, p, masked, grads):
                if p == net:
                    h, a0, t, a1 = acts[n - 1]
                    acts = dict(acts)
                    acts[n - 1] = (h, a0, np.abs(t) + 1, a1)    # t > 0 everywhere: the mask is all ones
                return orig_bwd(g_out, acts, n, W, sd, p, masked, grads)
            mp.setattr(G, "_net_bwd", net_bwd)
        out.append(("ReLU mask", patch(relu)))
    if coupled:
        def sqrt_h(mp):  # 3. the coupled widths / heights' 1/sqrt(H) missing from their gradient
            orig_bwd = G._net_bwd

            def net_bwd(g_out, acts, n, W, sd, p, masked, grads):
                if p == net:
                    g = g_out.reshape(g_out.shape[0], -1, 23).copy()
                    g[..., :16] *= np.sqrt(H)
                    g_out = g.reshape(g_out.shape)
                return orig_bwd(g_out, acts, n, W, sd, p, masked, grads)
            mp.setattr(G, "_net_bwd", net_bwd)
        out.append(("1/sqrt(H)", patch(sqrt_h)))

        def table(mp):   # 4. one identity feature's unconditional-table gradient dropped
            orig = G._BWD["CoupledRationalQuadraticSpline"]

            def bwd(z, sd, p, L, g_out, g_ld, grads):
                r = orig(z, sd, p, L, g_out, g_ld, grads)
                if p == "flows.0.":
                    for n in ("widths", "heights", "derivatives"):
                        grads[f"{p}prqct.unconditional_transform.unnormalized_{n}"][0] = 0
                return r
            mp.setitem(G._BWD, "CoupledRationalQuadraticSpline", bwd)
        out.append(("table row", patch(table)))

        def scatter(mp):  # 8. the identity columns' data gradient scattered to the transform columns
            orig = G._BWD["CoupledRationalQuadraticSpline"]
            orig_bwd = G._net_bwd
            held = {}

            def net_bwd(g_out, acts, n, W, sd, p, masked, grads):
                g = orig_bwd(g_out, acts, n, W, sd, p, masked, grads)
                held[p] = g
                return np.zeros_like(g)

            def bwd(z, sd, p, L, g_out, g_ld, grads):
                r = orig(z, sd, p, L, g_out, g_ld, grads)
                trf = sd[p + "prqct.transform_features"].astype(np.int64)
                gi = held.pop(p + "prqct.transform_net.")
                np.add.at(r, (slice(None), trf[np.arange(gi.shape[1]) % len(trf)]), gi)
                return r
            mp.setattr(G, "_net_bwd", net_bwd)
            mp.setitem(G._BWD, "CoupledRationalQuadraticSpline", bwd)
        out.append(("data scatter", patch(scatter)))
    else:
        def mulm(mp):    # 6. the MADE mask not applied to the final layer's weight gradient
            orig_bwd = G._net_bwd

            def net_bwd(g_out, acts, n, W, sd, p, masked, grads):
                if p == net:
                    sd = dict(sd)
                    sd[p + "final_layer.mask"] = np.ones_like(sd[p + "final_layer.mask"])
                return orig_bwd(g_out, acts, n, W, sd, p, masked, grads)
            mp.setattr(G, "_net_bwd", net_bwd)
        out.append(("MADE mask", patch(mulm)))
    if "L" in pattern:
        def logdet(mp):  # 5. the LU log-det term g_ld.sum() / diag dropped
            orig = G._BWD["LULinearPermute"]
            mp.setitem(G._BWD, "LULinearPermute", lambda z, sd, p, L, g, gl, gr: orig(z, sd, p, L, g, gl * 0, gr))
        out.append(("LU log-det", patch(logdet)))
    # 7. the last 64 rows' contribution to one weight gradient lost (the caller swaps in that tensor)
    out.append(("split-K partial", net + "final_layer.weight"))
    return out


@pytest.mark.parametrize("name", MUTANT_CFGS)
def test_bars_reject_slips(name):
    """The fp64 oracle with each slip, plus noise at the native path's level (the fp32 oracle's own error on the same
    rows, scaled to the native path's measured error), stands in for a native backward with that slip; check_grads must reject it at the sweep's row count, and
    accept the same noise on the correct gradients.  The fp32 oracle plays the interim path."""
    cfg = BY_NAME[name]
    model, spec = bwd_model(cfg)
    sd = state_dict64(model)
    x = inputs(cfg["D"], ROWS, cfg["seed"] + 2)
    w = loss_weights(spec, sd, x, cfg["seed"] + 4)
    ref = oracle_grads(spec, sd, x.astype(np.float64), w, cfg["base"])
    with np.errstate(all="ignore"):
        g32 = oracle_grads(spec, {k: v.astype(np.float32) if v.dtype.kind == "f" else v for k, v in sd.items()},
                           x, w.astype(np.float32), cfg["base"])
    noise = {}
    for k in ref:
        d = np.asarray(g32[k], np.float64) - ref[k]
        nd = np.linalg.norm(d)
        noise[k] = d * (NATIVE_FRO[name] * np.linalg.norm(ref[k]) / nd) if nd > 0 else d
    check_grads({k: ref[k] + noise[k] for k in ref}, ref, g32, f"{name} correct")
    mutants = _mutants(cfg)
    assert len(mutants) >= 5
    for what, how in mutants:
        if how is None:
            bad = oracle_grads(spec, sd, x.astype(np.float64), np.full(ROWS, w.mean()), cfg["base"])
        elif isinstance(how, str):
            w_cut = w.copy()
            w_cut[-64:] = 0
            bad = dict(ref)
            bad[how] = oracle_grads(spec, sd, x.astype(np.float64), w_cut, cfg["base"])[how]
        else:
            mp = how()
            try:
                bad = oracle_grads(spec, sd, x.astype(np.float64), w, cfg["base"])
            finally:
                mp.undo()
        assert any(not np.array_equal(bad[k], ref[k]) for k in ref), what
        with pytest.raises(AssertionError):
            check_grads({k: bad[k] + noise[k] for k in ref}, ref, g32, f"{name} {what}")


def test_mutant_configs_have_the_slips():
    kinds = set()
    for n in MUTANT_CFGS:
        c = BY_NAME[n]
        blocks, pattern = _blocks(c)
        assert any(c["name"] == d["name"] for d in SWEEP) and blocks[0][2] >= 1 and "L" in pattern and c["sigma"] >= 0.05
        kinds.add(blocks[0][0] != AR)
    assert kinds == {False, True}


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def paths(monkeypatch):
    """Records, per DensityFn backward that tried the native path, whether it ran (True) or fell back (False)."""
    taken = []
    orig = A.native_backward

    def rec(*a, **k):
        r = orig(*a, **k)
        taken.append(r is not None)
        return r
    monkeypatch.setattr(A, "native_backward", rec)
    yield taken
    DensityFn.use_native_backward = True


def gpu_grads(model, x, w, native):
    """{parameter name: gradient, "x": gradient} of sum(w * model.log_prob(x)), in float64 on the host."""
    DensityFn.use_native_backward = native
    model.zero_grad(set_to_none=True)
    xx = torch.from_numpy(x).cuda().requires_grad_(True)
    with torch.enable_grad():
        (torch.from_numpy(w).float().cuda() * model.log_prob(xx)).sum().backward()
    out = {k: p.grad.double().cpu().numpy() for k, p in model.named_parameters() if p.grad is not None}
    out["x"] = xx.grad.double().cpu().numpy()
    return out


def _hidden_names(model, i):
    net = dict(model.named_parameters())
    return [k for k in net if k.startswith(f"flows.{i}.") and ("initial_layer" in k or ".blocks." in k)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_backward_matches_oracle(name, paths):
    cfg = BY_NAME[name]
    model, spec = bwd_model(cfg)    # a fresh handle for every configuration
    sd = state_dict64(model)
    model = model.cuda()
    native = cfg["K"] == 8
    blocks, pattern = _blocks(cfg)
    for rows in row_counts(cfg):
        x = inputs(cfg["D"], rows, cfg["seed"] + 2)
        w = loss_weights(spec, sd, x, cfg["seed"] + 4)
        if rows == ROWS and name.startswith("spsl_"):   # nothing else checks the forward of these against the oracle
            check_log_prob(model.log_prob(torch.from_numpy(x).cuda()).cpu().numpy(),
                           O.log_prob(spec, sd, x.astype(np.float64)), name)
        ref = oracle_grads(spec, sd, x.astype(np.float64), w, cfg["base"])
        paths.clear()
        got = gpu_grads(model, x, w, True)
        assert paths == [native], f"{name}: backward paths {paths}, want {'native' if native else 'interim'}"
        interim = gpu_grads(model, x, w, False)
        spread = perturbed_spread(spec, sd, x, w, cfg["base"]) if cfg["sigma"] >= 0.5 else None
        ratio, fro, entry, frac = check_grads(got, ref, interim, f"{name} rows {rows}", spread)
        print(f"[spline-bwd] {name} rows={rows} {'native' if native else 'interim'}: worst native/interim Frobenius "
              f"{ratio:.1f}, rel. Frobenius {fro:.2e}, entry/scale {entry:.2e}, bulk {frac:.4f}")
        if cfg["sigma"] == 0.0:   # zero final layers: nothing reaches the hidden layers
            for i, c in enumerate(pattern):
                if c == "S":
                    for k in _hidden_names(model, i):
                        assert not np.any(got[k]) and not np.any(ref[k]), f"{name} {k}"
    # no rows: zero gradients, no error
    paths.clear()
    got = gpu_grads(model, inputs(cfg["D"], 0, 1), np.zeros(0), True)
    assert paths == [native] and got["x"].shape == (0, cfg["D"])
    assert all(not np.any(v) for v in got.values())


@pytest.mark.gpu
def test_columns_outside_the_tails(paths):
    """Whole columns outside +-tail at the first block the density pass runs: a transformed column's 23 spline
    parameters, and an identity column's table row, get exactly zero gradient."""
    cfg = dict(BY_NAME["wide_coupled_d65_h320_b4"], base=False)
    model, spec = bwd_model(cfg)
    sd = state_dict64(model)
    last = len(model.flows) - 1
    q = model.flows[last].prqct
    idf, trf = q.identity_features.tolist(), q.transform_features.tolist()
    x = inputs(cfg["D"], ROWS, 9)
    for c in (idf[0], idf[-1], trf[0], trf[-1]):
        x[:, c] = np.sign(x[:, c] + 0.5) * (cfg["tail"] + 0.25 + np.abs(x[:, c]))
    w = loss_weights(spec, sd, x, 10)
    ref = oracle_grads(spec, sd, x.astype(np.float64), w, False)
    model = model.cuda()
    got = gpu_grads(model, x, w, True)
    assert paths == [True]
    check_grads(got, ref, gpu_grads(model, x, w, False), "outside tails")
    p = f"flows.{last}.prqct."
    for t in (0, len(trf) - 1):
        for k in ("transform_net.final_layer.weight", "transform_net.final_layer.bias"):
            assert not np.any(got[p + k][23 * t:23 * t + 23]) and not np.any(ref[p + k][23 * t:23 * t + 23]), (k, t)
    for j in (0, len(idf) - 1):
        for n in ("widths", "heights", "derivatives"):
            k = f"{p}unconditional_transform.unnormalized_{n}"
            assert not np.any(got[k][j]) and not np.any(ref[k][j]), (k, j)
    # the other rows of those tensors are live
    assert np.any(got[p + "transform_net.final_layer.weight"][23:46])


@pytest.mark.gpu
def test_frozen_subsets(paths):
    """Frozen LU maps, then also one conditioner, then every parameter with x still requiring grad: the remaining
    gradients equal the full run's (to 1e-6 of each tensor's scale: the atomics reorder sums), frozen tensors get none."""
    cfg = BY_NAME["coupled_d63_h128_b2"]
    model, spec = bwd_model(cfg)
    model = model.cuda()
    x = inputs(cfg["D"], ROWS, 11)
    w = row_weights(ROWS, 12)
    full = gpu_grads(model, x, w, True)
    pattern = _blocks(cfg)[1]
    lu = [k for k, _ in model.named_parameters() if pattern[int(k.split(".")[1])] == "L"]
    cond = [k for k, _ in model.named_parameters() if k.startswith("flows.0.prqct.transform_net.")]
    params = dict(model.named_parameters())
    assert lu and cond
    for frozen in (lu, lu + cond, list(params)):
        for k, p in params.items():
            p.requires_grad_(k not in frozen)
        got = gpu_grads(model, x, w, True)
        assert set(got) == set(full) - set(frozen), sorted(set(got) ^ (set(full) - set(frozen)))
        for k in got:
            tol = 1e-6 * np.abs(full[k]).max()
            assert np.abs(got[k] - full[k]).max() <= tol, (k, len(frozen))
    assert paths == [True] * 4


@pytest.mark.gpu
def test_training_step_past_the_fused_limit(paths):
    """One Adam step on a 65-feature coupling stack: the next log_prob uses the updated weights (the packed operands
    follow the update), against the oracle on the new state."""
    cfg = BY_NAME["wide_coupled_d65_h320_b4"]
    model, spec = bwd_model(cfg)
    model = model.cuda()
    x = torch.from_numpy(inputs(cfg["D"], ROWS, 13)).cuda()
    w = torch.from_numpy(row_weights(ROWS, 14)).float().cuda()
    lp0 = model.log_prob(x).cpu().numpy()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    with torch.enable_grad():
        (w * model.log_prob(x)).sum().backward()
    opt.step()
    assert paths == [True]
    lp1 = model.log_prob(x).cpu().numpy()
    ref = O.log_prob(spec, state_dict64(model), x.cpu().numpy().astype(np.float64))
    assert np.abs(lp1 - lp0).max() > 1e-2
    check_log_prob(lp1, ref, "after one Adam step")
