"""The fused spline kernel (csrc/nfb_fused_rqs.cu) across the configuration space `build_fused` accepts, against the fp64
numpy oracle: conditioner kind and depth, hidden width, D (ragged float4s, odd and unequal coupling splits), tail bound,
MADE mask order, weight scale (constructor init with its all-zero final layer up to large weights), LU init and stack
layout.  The same configurations run on the plain-fp32 kernels.  Then inputs at the edges of the kernel's fp16 operand
planning, execution paths that must agree bit for bit, the LU fold taken / rejected / disabled, and (CPU only) a check
that the tolerances used here reject a subtly wrong conditioner."""
import itertools
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import normflows as nf
from conftest import PKG, ROOT
from normflows.flows.base import NativeFlow
from oracle import nf_oracle as O
from test_fused_plan_host import needs

AR, CPL, CPL_R = "ar", "coupled", "coupled_r"
KINDS = (AR, CPL, CPL_R)
DS = (1, 2, 3, 7, 33, 63, 64)
HS = (64, 128, 192, 256)
NBS = (0, 1, 2, 3)
TAILS = (0.5, 1.0, 3.0, 8.0)
SIGMAS = (0.05, 0.0, 1e-3)
LAYOUTS = ("SL", "SLx2", "LS", "SSL", "SPSL", "S", "SS")
ROWS = 1024          # density rows (oracle, fp64)
SAMPLE_ROWS = 512    # sampling rows (oracle, fp64 and fp32)


# ---------------------------------------------------------------------------------------------------------------------
# configurations
# ---------------------------------------------------------------------------------------------------------------------
def _sweep():
    """Covering design over (kind, D, H, num_blocks): D x H is the full product, num_blocks = (i_D + i_H) mod 4 covers
    D x nb and H x nb, kind = (i_D + 2 i_H) mod 3 (autoregressive at D = 1) covers kind x every other axis.  The
    remaining axes cycle with the row index; large weights (sigma 0.5) go to the shallow H = 64 nets (their derivative
    parameters reach 1e2 .. 1e3: the inverse spline's root in bins that are flat at one end and steep at the other,
    nfb_spline.cuh rqs_inverse_root).  LULinearPermute
    needs D >= 2 (D = 1: spline blocks alone) and the native Permute D <= 16 ([S, Permute, S, LU] only there)."""
    out = []
    for k, (di, hi) in enumerate(itertools.product(range(len(DS)), range(len(HS)))):
        D, H = DS[di], HS[hi]
        kind = AR if D == 1 else KINDS[(di + 2 * hi) % 3]
        nb = NBS[(di + hi) % 4]
        sigma = 0.5 if (H == 64 and nb <= 1) else SIGMAS[k % 3]
        layout = LAYOUTS[k % 5]
        if D == 1:
            layout = ("S", "SS")[k % 2]
        elif layout == "SPSL" and D > 16:
            layout = "SSL"
        out.append(dict(name=f"{kind}_d{D}_h{H}_b{nb}", kind=kind, D=D, H=H, nb=nb, tail=TAILS[k % 4],
                        pm=bool((k // 2) % 2), sigma=sigma, lu_id=k % 3 != 2, layout=layout, K=8,
                        bias_mult=10.0 if k == 9 else 1.0, seed=100 + k))
    # one persistent launch over blocks of different kind, width and depth
    out.append(dict(name="mixed_d16", kind="mixed", D=16, H=None, nb=None, tail=3.0, pm=True, sigma=0.05, lu_id=False,
                    layout="mixed", K=8, bias_mult=1.0, seed=7,
                    blocks=[(AR, 128, 1), (CPL, 256, 2), (AR, 64, 0), (CPL_R, 192, 3)]))
    return out


SWEEP = _sweep()
# just outside the fused kernel's reach: must run (on the fp32 kernels) and say so
OUTSIDE = [
    dict(name="ar_k7", kind=AR, D=5, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=True, layout="SL", K=7,
         bias_mult=1.0, seed=1),
    dict(name="coupled_k10", kind=CPL, D=6, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=True, layout="SL",
         K=10, bias_mult=1.0, seed=2),
    dict(name="ar_h96", kind=AR, D=7, H=96, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=True, layout="SL", K=8,
         bias_mult=1.0, seed=3),
    dict(name="coupled_h320", kind=CPL, D=8, H=320, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=True, layout="SL",
         K=8, bias_mult=1.0, seed=4),
    dict(name="ar_b4", kind=AR, D=5, H=128, nb=4, tail=3.0, pm=False, sigma=0.05, lu_id=True, layout="SL", K=8,
         bias_mult=1.0, seed=5),
]
BY_NAME = {c["name"]: c for c in SWEEP + OUTSIDE}


def _blocks(cfg):
    """[(kind, H, nb)] of the spline blocks and the layer layout as a string of S / L / P."""
    lay = cfg["layout"]
    if lay == "mixed":
        return cfg["blocks"], "SL" * len(cfg["blocks"])
    pattern = {"SL": "SL", "SLx2": "SLSL", "LS": "LS", "SSL": "SSL", "SPSL": "SPSL", "SPS": "SPS", "S": "S",
               "SS": "SS", "SLLS": "SLLS", "LLS": "LLS", "L": "L", "LL": "LL"}[lay]
    n = pattern.count("S")
    kinds = [cfg["kind"]] * n
    if cfg["kind"] in (CPL, CPL_R):   # consecutive coupling blocks alternate their masks, the first one as configured
        kinds = [(CPL, CPL_R)[(i + (cfg["kind"] == CPL_R)) % 2] for i in range(n)]
    return [(k, cfg["H"], cfg["nb"]) for k in kinds], pattern


def make_model(cfg):
    """(model on the CPU, oracle spec).  Constructors under torch.manual_seed(seed), every parameter moved by
    sigma * randn (seed + 1), conditioner biases optionally scaled (tests/helpers.py nsf_model does the same)."""
    D, K, tail = cfg["D"], cfg["K"], cfg["tail"]
    blocks, pattern = _blocks(cfg)
    torch.manual_seed(cfg["seed"])
    flows, spec, bi = [], [], 0
    for c in pattern:
        if c == "S":
            kind, H, nb = blocks[bi]
            bi += 1
            if kind == AR:
                flows.append(nf.flows.AutoregressiveRationalQuadraticSpline(D, nb, H, num_bins=K, tail_bound=tail,
                                                                            permute_mask=cfg["pm"]))
                spec.append({"type": "AutoregressiveRationalQuadraticSpline", "num_bins": K, "tail_bound": tail})
            else:
                flows.append(nf.flows.CoupledRationalQuadraticSpline(D, nb, H, num_bins=K, tail_bound=tail,
                                                                     reverse_mask=kind == CPL_R))
                spec.append({"type": "CoupledRationalQuadraticSpline", "num_bins": K, "tail_bound": tail})
        elif c == "L":
            flows.append(nf.flows.LULinearPermute(D, identity_init=cfg["lu_id"]))
            spec.append({"type": "LULinearPermute", "num_channels": D})
        else:
            flows.append(nf.flows.Permute(D, mode="shuffle"))
            spec.append({"type": "Permute", "num_channels": D, "mode": "shuffle"})
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D, trainable=False), flows)
    g = torch.Generator().manual_seed(cfg["seed"] + 1)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(cfg["sigma"] * torch.randn(p.shape, generator=g, dtype=p.dtype))
        if cfg["bias_mult"] != 1.0:
            for name, p in model.named_parameters():
                if name.endswith(".bias") and ("autoregressive_net" in name or "transform_net" in name):
                    p.mul_(cfg["bias_mult"])
    return model, {"kind": "NormalizingFlow", "q0": {"shape": [D]}, "flows": spec}


def state_dict(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


def expected_fused(cfg):
    """Layers that must run on the fused kernel, by the rule in nfb_api.cu build_fused: K = 8, H % 64 = 0, H <= 256,
    n_hidden = 1 + 2 num_blocks <= 7, D <= 64 (so T <= 64); an LU right after a fused block joins it as a pair."""
    blocks, pattern = _blocks(cfg)
    ok = [cfg["K"] == 8 and H % 64 == 0 and H <= 256 and 1 + 2 * nb <= 7 and cfg["D"] <= 64 for _, H, nb in blocks]
    out, bi, prev_fused_spline = [], 0, False
    for i, c in enumerate(pattern):
        if c == "S":
            f = ok[bi]
            bi += 1
            if f:
                out.append(i)
            prev_fused_spline = f
        else:
            if c == "L" and prev_fused_spline:
                out.append(i)
            prev_fused_spline = False
    return out


def inputs(D, rows, seed):
    return (torch.randn(rows, D, generator=torch.Generator().manual_seed(seed)) * 1.5).numpy()


_ORACLE = {}


def oracle(cfg):
    """fp64 oracle of the density pass (with its per-layer trace) and of the sampling pass from the oracle's own z,
    plus the sampling pass in fp32 (the reference's own round-off on the same rows).  Cached per configuration."""
    name = cfg["name"]
    if name not in _ORACLE:
        model, spec = make_model(cfg)
        sd = state_dict(model)
        x = inputs(cfg["D"], ROWS, cfg["seed"] + 2)
        x64 = x.astype(np.float64)
        z, ld, trace = O.inverse_and_log_det(spec, sd, x64, per_layer=True)
        lp = ld + O.diag_gaussian_log_prob(z, O._cast(sd, np.float64), "q0.")
        # the reference's own fp32 error of each layer, from the same (fp32-rounded) input
        spread, zin, sd32 = {}, x64, O._cast(sd, np.float32)
        with np.errstate(all="ignore"):
            for i, zr, ldr in trace:
                z32, ld32 = O.LAYERS[spec["flows"][i]["type"]](zin.astype(np.float32), sd32, f"flows.{i}.",
                                                                spec["flows"][i], "inverse")
                spread[i] = (np.nanmax(np.abs(z32 - zr)), np.nanmax(np.abs(ld32 - ldr)))
                zin = zr
        zs = z[:SAMPLE_ROWS].astype(np.float32)
        xs64, lds64 = O.forward_and_log_det(spec, sd, zs.astype(np.float64))
        xs32, lds32 = O.forward_and_log_det(spec, sd, zs)
        _ORACLE[name] = dict(spec=spec, sd=sd, x=x, z=z, ld=ld, lp=lp, trace=trace, spread=spread, zs=zs, xs64=xs64, lds64=lds64,
                             xs32=xs32, lds32=lds32)
    return _ORACLE[name]


# ---------------------------------------------------------------------------------------------------------------------
# assertions (also applied, on the CPU, to mutated conditioners: they must reject those)
# ---------------------------------------------------------------------------------------------------------------------
def check_log_prob(lp, ref, what=""):
    """rtol 1e-4 with atol 1e-3 on every row (BASELINE.json's north-star bar)."""
    lp, ref = np.asarray(lp, np.float64), np.asarray(ref, np.float64)
    assert np.all(np.isfinite(lp)), f"{what}: non-finite log_prob"
    err = np.abs(lp - ref) - 1e-4 * np.abs(ref)
    i = int(np.argmax(err))
    assert err[i] <= 1e-3, f"{what}: log_prob row {i}: {lp[i]!r} vs {ref[i]!r}"
    return float(np.max(np.abs(lp - ref)))


def check_layer(z, ld, z_ref, ld_ref, what="", spread=(0.0, 0.0)):
    """z: atol 2e-4 on >= 99.5 % of the elements, 2e-3 on all; log-det: atol 2e-3.  Where the layer is so
    ill-conditioned (large weights) that the reference's own fp32 run of it misses by more, the maxima are judged
    against 10 x that spread instead, as for the sampling direction."""
    ez = np.abs(np.asarray(z, np.float64) - z_ref)
    assert np.all(np.isfinite(ez)), f"{what}: non-finite z"
    assert np.mean(ez < 2e-4) >= 0.995 and ez.max() < max(2e-3, 10 * spread[0]), \
        f"{what}: z err max {ez.max():.3e}, {np.mean(ez >= 2e-4):.4f} above 2e-4 (fp32 spread {spread[0]:.3e})"
    el = np.abs(np.asarray(ld, np.float64) - ld_ref)
    assert np.all(np.isfinite(el)) and el.max() < max(2e-3, 10 * spread[1]), \
        f"{what}: log-det err max {el.max():.3e} (fp32 spread {spread[1]:.3e})"


def check_sampling(x, ld, o, what=""):
    """Judged against the reference's own fp32 spread on the same rows (test_gpu_parity.py does the same), on the rows
    where that fp32 run is finite."""
    ok = np.all(np.isfinite(o["xs32"]), axis=1) & np.isfinite(o["lds32"])
    assert np.mean(ok) >= 0.95, f"{what}: the reference's fp32 run is not finite on {np.sum(~ok)} rows"
    o = {k: o[k][ok] for k in ("xs32", "xs64", "lds32", "lds64")}
    x, ld = np.asarray(x)[ok], np.asarray(ld)[ok]
    ex = np.abs(np.asarray(x, np.float64) - o["xs64"]).max(axis=1)
    rows = np.abs(o["xs32"] - o["xs64"]).max(axis=1)
    spread = rows.max()
    # (large weights can make the inverse chaotic: then the reference's own fp32 median sets the median bar)
    assert np.all(np.isfinite(ex)), f"{what}: non-finite sample"
    assert np.median(ex) < max(2e-4, 10 * np.median(rows)) and ex.max() <= max(10 * spread, 2e-3), \
        f"{what}: x err median {np.median(ex):.3e} max {ex.max():.3e} (fp32 spread {spread:.3e})"
    el = np.abs(np.asarray(ld, np.float64) - o["lds64"])
    spread_l = np.abs(o["lds32"] - o["lds64"]).max()
    assert np.median(el) < max(2e-3, 10 * np.median(np.abs(o["lds32"] - o["lds64"]))) and el.max() <= max(10 * spread_l, 2e-2), \
        f"{what}: log-det err median {np.median(el):.3e} max {el.max():.3e} (fp32 spread {spread_l:.3e})"


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the design covers what it claims; the assertions reject wrong conditioners
# ---------------------------------------------------------------------------------------------------------------------
def test_sweep_is_a_covering_design():
    rows = [c for c in SWEEP if c["layout"] != "mixed"]
    axes = {"kind": KINDS, "D": DS, "H": HS, "nb": NBS}
    for a, b in itertools.combinations(axes, 2):
        have = {(c[a], c[b]) for c in rows}
        want = {(u, v) for u in axes[a] for v in axes[b]
                if not ((a == "kind" and u != AR and b == "D" and v == 1))}
        assert want <= have, (a, b, sorted(want - have))
    assert {c["tail"] for c in rows} == set(TAILS)
    assert {c["pm"] for c in rows if c["kind"] == AR} == {False, True}
    assert {c["sigma"] for c in rows} == {0.0, 1e-3, 0.05, 0.5}
    assert {c["lu_id"] for c in rows} == {False, True}
    assert {c["layout"] for c in rows} == set(LAYOUTS)
    assert sum(c["bias_mult"] != 1.0 for c in rows) == 1
    assert 25 <= len(SWEEP) <= 35
    for c in OUTSIDE:
        assert expected_fused(c) == [], c["name"]


def _mutants(cfg, sd):
    """(what, mutated state_dict) for each slip of the packer the fused kernel could make, on the first spline block
    (flows.0) and the first LU map."""
    out = []
    D = cfg["D"]
    blocks, _ = _blocks(cfg)
    kind, H, nb = blocks[0]
    if kind == AR:
        net = "flows.0.mprqat.autoregressive_net."
        m_init = sd[net + "initial_layer.mask"]
        m_hid = sd[net + "blocks.0.linear_layers.0.mask"] if nb else None
        perm = np.argsort(m_init.sum(1), kind="stable")
    else:
        net = "flows.0.prqct.transform_net."
        m_init = m_hid = None
        perm = np.arange(H)
    if nb:
        # a dropped record: the last non-zero [64 x 64] block (degree-sorted order) of a hidden-to-hidden GEMM
        need = needs(H, None if m_hid is None else (m_init, m_hid, None))
        jb, kb = [(j, k) for j in range(H // 64) for k in range(H // 64) if need[j][k]][-1]
        s = dict(sd)
        w = s[net + "blocks.0.linear_layers.1.weight"].copy()
        w[np.ix_(perm[64 * jb:64 * jb + 64], perm[64 * kb:64 * kb + 64])] = 0
        s[net + "blocks.0.linear_layers.1.weight"] = w
        out.append(("hidden block", s))
        # the cum bias pre-sum: one hidden unit's second residual bias left out (the most visible one)
        s = dict(sd)
        b = s[net + "blocks.0.linear_layers.1.bias"].copy()
        wf = np.abs(s[net + "final_layer.weight"] * s.get(net + "final_layer.mask", 1.0)).max(axis=0)
        j = int(np.argmax(np.abs(b) * wf))
        b[j] = 0
        s[net + "blocks.0.linear_layers.1.bias"] = b
        out.append(("residual bias", s))
    # a wrong slab shift: the last non-zero K = 16 slab (sorted hidden order) of the first final-layer chunk zeroed
    s = dict(sd)
    wf = (s[net + "final_layer.weight"] * s.get(net + "final_layer.mask", 1.0))[:2 * 23][:, perm]
    live = np.flatnonzero(np.abs(wf).max(axis=0) > 0)
    k0 = 16 * (int(live[-1]) // 16)
    w = s[net + "final_layer.weight"].copy()
    rows = np.arange(min(2, w.shape[0] // 23) * 23)
    w[np.ix_(rows, perm[k0:k0 + 16])] = 0
    s[net + "final_layer.weight"] = w
    out.append(("final slab", s))
    # the fold's bias shift: the bias of the first LU map left out
    s = dict(sd)
    s[f"flows.{_blocks(cfg)[1].index('L')}.linear.bias"] = np.zeros(D, np.float32)
    out.append(("LU bias", s))
    return out


MUTANT_CFGS = ["ar_d7_h256_b2", "coupled_d63_h128_b2", "coupled_d3_h128_b3"]


@pytest.mark.parametrize("name", MUTANT_CFGS)
def test_tolerances_reject_a_wrong_conditioner(name):
    """The oracle's output for a mutated state_dict stands in for a kernel with that slip; the density assertions of
    the GPU sweep must fail on it at the sample sizes the sweep uses."""
    cfg = BY_NAME[name]
    blocks, pattern = _blocks(cfg)
    assert pattern[0] == "S" and cfg["sigma"] > 0
    o = oracle(cfg)
    mut = _mutants(cfg, o["sd"])
    assert len(mut) == (4 if blocks[0][2] else 2)
    for what, sd in mut:
        z, ld, trace = O.inverse_and_log_det(o["spec"], sd, o["x"].astype(np.float64), per_layer=True)
        lp = ld + O.diag_gaussian_log_prob(z, O._cast(sd, np.float64), "q0.")
        with pytest.raises(AssertionError):
            check_log_prob(lp, o["lp"], what)
        # ... and layer by layer (the mutated block's own output, from the correct input)
        zin = [t[1] for t in o["trace"] if t[0] == 1][0]
        zl, ldl = O.LAYERS[o["spec"]["flows"][0]["type"]](zin, O._cast(sd, np.float64), "flows.0.",
                                                          o["spec"]["flows"][0], "inverse")
        zr, ldr = [(t[1], t[2]) for t in o["trace"] if t[0] == 0][0]
        if what != "LU bias":
            with pytest.raises(AssertionError):
                check_layer(zl, ldl, zr, ldr, what, o["spread"][0])


def test_mutant_configs_are_in_the_sweep():
    for n in MUTANT_CFGS:
        c = BY_NAME[n]
        assert c in SWEEP and c["nb"] >= 1 and c["sigma"] >= 0.05
    assert {BY_NAME[n]["kind"] for n in MUTANT_CFGS} >= {AR, CPL} and any(BY_NAME[n]["bias_mult"] != 1 for n in MUTANT_CFGS)


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def tc():
    yield
    NativeFlow.use_tensor_cores = True


def _np(t):
    return t.detach().cpu().numpy()


def _run_config(cfg, use_tc):
    NativeFlow.use_tensor_cores = use_tc
    o = oracle(cfg)
    model, _ = make_model(cfg)
    model = model.cuda()
    x = torch.from_numpy(o["x"]).cuda()
    lp = _np(model.log_prob(x))
    h = model._stack()
    want = expected_fused(cfg) if use_tc else []
    assert h.fused_layers() == want, f"fused layers {h.fused_layers()} != {want}"
    worst = check_log_prob(lp, o["lp"], cfg["name"])
    # layer by layer (single-layer launches of the same packed stack) from the oracle's inputs
    n = len(model.flows)
    zin = o["x"].astype(np.float64)
    for i, zr, ldr in o["trace"]:
        zi, ldi = h.layer_apply(i, 0, torch.from_numpy(zin.astype(np.float32)).cuda())
        check_layer(_np(zi), _np(ldi), zr, ldr, f"{cfg['name']} layer {i}/{n}", o["spread"][i])
        zin = zr
    xs, lds = model.forward_and_log_det(torch.from_numpy(o["zs"]).cuda())
    check_sampling(_np(xs), _np(lds), o, cfg["name"] + " sampling")
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("use_tc", [True, False], ids=["fused", "fp32"])
@pytest.mark.parametrize("name", [c["name"] for c in SWEEP])
def test_config_matches_oracle(name, use_tc, tc):
    worst = _run_config(BY_NAME[name], use_tc)
    print(f"[fused-configs] {name} {'fused' if use_tc else 'fp32'}: fused={expected_fused(BY_NAME[name]) if use_tc else []}"
          f" worst |dlog_prob| = {worst:.3e}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c["name"] for c in OUTSIDE])
def test_outside_eligibility_runs_unfused(name, tc):
    worst = _run_config(BY_NAME[name], True)
    print(f"[fused-configs] {name}: fused=[] worst |dlog_prob| = {worst:.3e}")


# ---- input edges -----------------------------------------------------------------------------------------------------
EDGE_CFGS = [
    dict(name="edge_ar", kind=AR, D=7, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=False, layout="SL", K=8,
         bias_mult=1.0, seed=11),
    dict(name="edge_coupled", kind=CPL, D=7, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=False, layout="SL",
         K=8, bias_mult=1.0, seed=12),
]


PRECISE_ROW_MAX = 1e6   # rows up to this magnitude keep the density tolerances on every element


def quantisation_bound(spec, sd, row):
    """What the fused kernel may lose on a row with a large element (DESIGN.md 3.1): every operand of the LU stage and
    of the first conditioner GEMM is quantised to q = 2^(e - 38), e = floor(log2 max|x_row|) + 1 (fp16 hi/lo pairs
    reach 2^-24 below a 2^14 scale).  Bound: twice the sum over the row's elements of the fp64 reference's response to
    moving that element by q (zero for the large element itself, which keeps 22 bits)."""
    e = int(np.floor(np.log2(np.abs(row).max()))) + 1
    q = 2.0 ** (e - 38)
    x0 = row.astype(np.float64)[None]
    z0, l0 = O.inverse_and_log_det(spec, sd, x0)
    dz, dl = np.zeros(len(row)), 0.0
    for j in range(len(row)):
        if abs(row[j]) > PRECISE_ROW_MAX:
            continue
        x1 = x0.copy()
        x1[0, j] += q
        z1, l1 = O.inverse_and_log_det(spec, sd, x1)
        dz += np.abs(z1[0] - z0[0])
        dl += abs(float(l1[0] - l0[0]))
    return 2 * dz, 2 * dl


def edge_values(tail):
    t = np.float32(tail)
    up, dn = np.nextafter(t, np.float32(np.inf)), np.nextafter(t, np.float32(0))
    return [0.0, 1e-40, -1e-40, 1e-30, t, -t, up, -up, dn, -dn, 1e6, 2.0 ** 39, 2.0 ** 40, 2.0 ** 41, -2.0 ** 41,
            1e13, -1e13, 3e38, -3e38]


def edge_batch(D, tail, seed):
    """1 024 normal rows; rows 64 + 3 k carry edge value k in column k mod D (row 61: all zeros), so that every 64-row
    tile with edge rows also has normal rows."""
    x = inputs(D, ROWS, seed)
    base = x.copy()
    rows = [61]
    x[61] = 0
    for k, v in enumerate(edge_values(tail)):
        r = 64 + 3 * k
        x[r, k % D] = np.float32(v)
        rows.append(r)
    return base, x, rows


@pytest.mark.gpu
@pytest.mark.parametrize("with_lu", [False, True], ids=["alone", "with_lu"])
@pytest.mark.parametrize("cfg", EDGE_CFGS, ids=[c["name"] for c in EDGE_CFGS])
def test_input_edges(cfg, with_lu):
    cfg = dict(cfg, layout="SL")
    model, spec = make_model(cfg)
    if not with_lu:
        model = nf.NormalizingFlow(model.q0, [model.flows[0]])
        spec = dict(spec, flows=spec["flows"][:1])
    sd = state_dict(model)
    base, x, rows = edge_batch(cfg["D"], cfg["tail"], cfg["seed"])
    with np.errstate(all="ignore"):
        z64, ld64 = O.inverse_and_log_det(spec, sd, x.astype(np.float64))
        z32, ld32 = O.inverse_and_log_det(spec, sd, x)
    model = model.cuda()
    assert model._stack() is not None
    z, ld = model.inverse_and_log_det(torch.from_numpy(x).cuda())
    assert model._stack().fused_layers() == list(range(len(model.flows)))
    z, ld = _np(z).astype(np.float64), _np(ld).astype(np.float64)
    with np.errstate(all="ignore"):
        for r in rows:
            if not (np.all(np.isfinite(z32[r])) and np.isfinite(ld32[r])):
                continue
            assert np.all(np.isfinite(z[r])) and np.isfinite(ld[r]), f"row {r} ({x[r]}): kernel {z[r]} {ld[r]}"
            tol_z = np.maximum(2e-3 + 1e-5 * np.abs(z64[r]), 10 * np.abs(z32[r] - z64[r]))
            tol_l = max(2e-3 + 1e-5 * abs(ld64[r]), 10 * abs(ld32[r] - ld64[r]))
            if np.abs(x[r]).max() > PRECISE_ROW_MAX:
                qz, ql = quantisation_bound(spec, sd, x[r])
                tol_z, tol_l = tol_z + qz, tol_l + ql
            assert np.all(np.abs(z[r] - z64[r]) <= tol_z), f"row {r} ({x[r]}): z {z[r]} vs {z64[r]}"
            assert abs(ld[r] - ld64[r]) <= tol_l, f"row {r} ({x[r]}): log-det {ld[r]} vs {ld64[r]}"
    # the normal rows of the same tiles are untouched by their neighbours
    zb, ldb = model.inverse_and_log_det(torch.from_numpy(base).cuda())
    keep = np.setdiff1d(np.arange(ROWS), rows)
    assert np.array_equal(_np(zb)[keep], z[keep].astype(np.float32))
    assert np.array_equal(_np(ldb)[keep], ld[keep].astype(np.float32))


# ---- paths that must agree bit for bit -------------------------------------------------------------------------------
BIT_CFGS = ["ar_d7_h256_b2", "coupled_d63_h128_b2", "mixed_d16"]
# the diagonal wave order needs a whole-stack launch of more than one unit (nfb_api.cu launch_fused_stack)
WAVE_CFGS = ["ar_d1_h256_b3", "coupled_d63_h128_b2", "mixed_d16"]


def _same(a, b, what):
    a, b = _np(a), _np(b)
    assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True), \
        f"{what}: {np.sum(a != b)} elements differ, max {np.nanmax(np.abs(a.astype(np.float64) - b)):.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_CFGS)
def test_stack_launch_equals_group_launches(name, monkeypatch):
    cfg = BY_NAME[name]
    x = torch.from_numpy(inputs(cfg["D"], 5000, 3)).cuda()
    model = make_model(cfg)[0].cuda()
    z, ld = model.inverse_and_log_det(x)
    assert model._stack().launch_count() <= 3, "whole-stack launch not taken"   # fill, memset, kernel
    monkeypatch.setenv("NFB_NO_STACK", "1")
    other = make_model(cfg)[0].cuda()
    z2, ld2 = other.inverse_and_log_det(x)
    groups = _blocks(cfg)[1].count("S")   # every block is paired with its LU: one launch per pair, after the fill
    assert other._stack().launch_count() == 1 + groups, "NFB_NO_STACK did not split the launch"
    _same(z, z2, "z")
    _same(ld, ld2, "log-det")


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_CFGS)
def test_ticket_equals_static_units(name, monkeypatch):
    cfg = BY_NAME[name]
    x = torch.from_numpy(inputs(cfg["D"], 20000, 4)).cuda()
    model = make_model(cfg)[0].cuda()
    z, ld = model.inverse_and_log_det(x)
    xs, lds = model.forward_and_log_det(z)
    monkeypatch.setenv("NFB_STATIC_UNITS", "1")
    z2, ld2 = model.inverse_and_log_det(x)
    xs2, lds2 = model.forward_and_log_det(z)
    for a, b, w in ((z, z2, "z"), (ld, ld2, "log-det"), (xs, xs2, "sample"), (lds, lds2, "sample log-det")):
        _same(a, b, w)


@pytest.mark.gpu
@pytest.mark.parametrize("name", WAVE_CFGS)
def test_wave_order_equals_layer_order(name, monkeypatch):
    cfg = BY_NAME[name]
    pattern = _blocks(cfg)[1]
    # preconditions of the wave order: every layer fused, >= 2 units in the launch, >= 8192 rows (64 tiles)
    assert expected_fused(cfg) == list(range(len(pattern))) and pattern.count("S") >= 2
    xh = torch.from_numpy(inputs(cfg["D"], 8192 + 640 + 5, 5)).contiguous()
    model = make_model(cfg)[0].cuda()
    h = model._stack()
    dev = torch.device("cuda", torch.cuda.current_device())
    lp_dev = model.log_prob(xh.cuda())
    lp = h.log_prob_host(xh, dev)
    monkeypatch.setenv("NFB_NO_WAVE_ORDER", "1")
    lp2 = h.log_prob_host(xh, dev)
    _same(lp, lp2, "host log_prob, wave vs layer order")
    _same(lp, lp_dev.cpu(), "host vs device log_prob")


@pytest.mark.gpu
@pytest.mark.parametrize("name", BIT_CFGS)
def test_row_result_independent_of_batch(name):
    cfg = BY_NAME[name]
    model = make_model(cfg)[0].cuda()
    xb = torch.from_numpy(inputs(cfg["D"], 65536 + 77, 6)).cuda()
    lp = model.log_prob(xb)
    xs, lds = model.forward_and_log_det(xb)
    for n in (1, 127, 128, 129):
        for r0 in (0, 65536 + 77 - n, 1000):
            sl = slice(r0, r0 + n)
            _same(model.log_prob(xb[sl].contiguous()), lp[sl], f"log_prob rows {r0}+{n}")
            a, b = model.forward_and_log_det(xb[sl].contiguous())
            _same(a, xs[sl], f"sample rows {r0}+{n}")
            _same(b, lds[sl], f"sample log-det rows {r0}+{n}")


# ---- the LU fold: taken, rejected by the scale plan, disabled --------------------------------------------------------
FOLD_CFGS = {
    # the default: an autoregressive block with its LU folded into the first conditioner GEMM
    "taken": dict(name="fold_taken", kind=AR, D=12, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=True,
                  layout="SL", K=8, bias_mult=1.0, seed=21),
    # a coupled block with tail 16 (conditioner inputs bounded by 16) after an LU map of diagonal 1e-3: the folded
    # matrix is ~10 binades below the first GEMM's, its fp16 scale would have to drop > 12 binades -> not folded
    "rejected": dict(name="fold_rejected", kind=CPL, D=12, H=128, nb=1, tail=16.0, pm=False, sigma=0.0,
                     lu_id=True, layout="SL", K=8, bias_mult=1.0, seed=22, lu_diag=-30.0),
}

_CHILD = r"""
import sys, json, numpy as np, torch
sys.path[:0] = json.loads(sys.argv[1])
from test_fused_configs import FOLD_CFGS, fold_model, inputs, ROWS
cfg = FOLD_CFGS[sys.argv[2]]
model = fold_model(cfg)[0].cuda()
torch.set_grad_enabled(False)
lp = model.log_prob(torch.from_numpy(inputs(cfg["D"], ROWS, 9)).cuda())
assert model._stack().fused_layers() == [0, 1]
np.save(sys.argv[3], lp.cpu().numpy())
"""


def fold_model(cfg):
    model, spec = make_model(cfg)
    if "lu_diag" in cfg:
        with torch.no_grad():
            model.flows[1].linear.unconstrained_upper_diag.fill_(cfg["lu_diag"])
    return model, spec


@pytest.mark.gpu
@pytest.mark.parametrize("state", ["taken", "rejected", "disabled"])
def test_lu_fold_states(state, tmp_path):
    cfg = FOLD_CFGS["taken" if state == "disabled" else state]
    env = dict(os.environ, NFB_DEBUG_PACK="1")
    if state == "disabled":
        env["NFB_NO_FOLD"] = "1"
    out = str(tmp_path / "lp.npy")
    r = subprocess.run([sys.executable, "-c", _CHILD, json.dumps([os.path.join(ROOT, "tests"), ROOT, PKG]),
                        state if state != "disabled" else "taken", out],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [ln for ln in r.stderr.splitlines() if ln.startswith("[nfb pack] fold:")]
    assert lines, r.stderr[-2000:]
    m = re.search(r"U=(\S+) pair_ok=(\d) pw_fold=(-?\d+)", lines[-1])
    u, pair_ok, pw_fold = m.group(1), int(m.group(2)), int(m.group(3))
    assert pair_ok == 1
    if state == "disabled":
        assert u in ("(nil)", "0", "0x0"), lines[-1]
    else:
        assert u not in ("(nil)", "0", "0x0"), lines[-1]
        assert (pw_fold > -100) == (state == "taken"), lines[-1]
    model, spec = fold_model(cfg)
    sd = state_dict(model)
    x = inputs(cfg["D"], ROWS, 9).astype(np.float64)
    z, ld = O.inverse_and_log_det(spec, sd, x)
    ref = ld + O.diag_gaussian_log_prob(z, O._cast(sd, np.float64), "q0.")
    check_log_prob(np.load(out), ref, f"fold {state}")


@pytest.mark.gpu
@pytest.mark.parametrize("use_tc", [True, False], ids=["fused", "fp32"])
def test_one_feature_with_lu(use_tc, tc):
    """D = 1 with an LULinearPermute (whose strictly triangular parameters are empty tensors) after each block."""
    cfg = dict(name="ar_d1_lu", kind=AR, D=1, H=128, nb=1, tail=3.0, pm=False, sigma=0.05, lu_id=False, layout="SLx2",
               K=8, bias_mult=1.0, seed=31)
    _run_config(cfg, use_tc)
