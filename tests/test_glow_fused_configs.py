"""The fused Glow conditioner (csrc/nfb_glow_fused.cu glow_cond_kernel), the tap-form affine coupling, the tap sum and the
ActNorm + Invertible1x1Conv folds (csrc/nfb_glow.cu), and the one-call GlowBlock (nfb_glow_block) across their
configuration space against the fp64 numpy oracle.  The conditioner sweep is a covering design over hidden width, input
channels (GEMM 1 K-chunks), output channels (GEMM 3 slices), image geometry (1x1 images, odd non-square images, tiles
that cross image rows and images, more tiles than SMs), channel slice, LeakyReLU slope and weight scale.  Then the
coupling's options and both staging paths, its shared-memory limit, paths that must agree bit for bit, the folds up to
their channel limits and (CPU only) a check that the tolerances used here reject a subtly wrong conditioner or coupling."""
import itertools

import numpy as np
import pytest
import torch

import normflows as nf
from oracle import nf_oracle as O

HS = (64, 128, 192, 256)
CINS = (1, 7, 8, 15, 22, 28)     # 9 cin = 9, 63, 72, 135, 198, 252: 1, 1, 2, 3, 4, 4 K-chunks of GEMM 1
COUTS = (1, 7, 8, 14, 43, 56)    # 9 cout = 9, 63, 72, 126, 387, 504: 1, 1, 2, 2, 7, 8 output slices of GEMM 3
GEOMS = {                        # (B, H, W)
    "1x1": (37, 1, 1),           # every tap but the centre lies in the padding; 37 pixels: one partial tile
    "3x5": (9, 3, 5),            # odd, non-square, HW = 15 does not divide 64: tiles end mid-row
    "4x4": (27, 4, 4),           # four images per tile, 432 pixels: a ragged last tile
    "16x16": (3, 16, 16),
    "7x9_many": (540, 7, 9),     # odd, non-square; 34 020 pixels = 532 tiles: every CTA runs the tile loop >= 4 times
}
MANY = "7x9_many"
MANY_IMAGES = (0, 270, 539)      # the images of a many-tile row that are compared with the oracle
LEAKS = (0.0, 0.01, 0.2)
SCALES = ("init", "large", "zero")   # constructor init; every parameter x 3; init_zeros (last convolution all zero)
U32 = 2.0 ** -24                 # unit roundoff of fp32

# Error model of the fused conditioner (csrc/nfb_glow_fused.cu header).  Per product, split bf16 (8 significant bits):
# a w - (a_hi w_hi + a_lo w_hi + a_hi w_lo) is a_lo w_lo plus the rounding residues of a_lo and w_lo, <= 3 * 2^-16 |a w|.
# Per output, at most 12 kcs <= 48 truncating K = 16 accumulate steps, each <= 2^-23 of the running sum <= sum |a w|
# (0.375 * 2^-16), and the compensating gain moves it by <= 48 * 2.4e-8 (0.08 * 2^-16): <= 3.5 * 2^-16 of the absolute
# sum per GEMM.  LeakyReLU is 1-Lipschitz, so each GEMM's input error reaches the output through |W|: three chained
# GEMMs stay within 10.5 * 2^-16 of the same network run on |x|, |W|, |b| with identity activations.
KAPPA = 12 * 2.0 ** -16
# That worst case is a sum of |.| over K products (K = 9 cin, hid, hid) and looser than a slip such as a dropped LeakyReLU
# slope of 0.01 on the deepest configuration.  The second bound is statistical: the rounded pieces of a split product are
# each < 2^-16 |a w| and spread evenly, so one product's error has an rms below SIGMA_P = 2^-16 |a w|; the K errors of a
# sum are independent, so its rms is SIGMA_P sqrt(sum (a w)^2) = SIGMA_P Q, and Q^2 of the chain is the oracle run on
# squares (conditioner_scales).  Z_Q = 8 standard deviations (a Gaussian tail of < 1e-9 over a million elements), plus
# 16 u |net| for the rounded bias adds and the random part of the accumulate truncation left by the gain.
SIGMA_P = 2.0 ** -16
Z_Q = 8.0
FLOOR = 1e-30                    # a zero absolute network (init_zeros) must give an exact zero


# ---------------------------------------------------------------------------------------------------------------------
# configurations
# ---------------------------------------------------------------------------------------------------------------------
def _sweep():
    """cin x geometry is the full product (30 rows); hidden = HS[(2 i + 3 j) % 4] and cout = COUTS[(i + j + 3) % 6]
    (i, j: cin and geometry index) cover hidden x cin and hidden x cout pairwise.  The channel slice alternates, the
    slope cycles with the row and the weight scale with every third row, so slope x scale is covered too."""
    out = []
    for k, (i, j) in enumerate(itertools.product(range(len(CINS)), range(len(GEOMS)))):
        cin, geom = CINS[i], list(GEOMS)[j]
        hid, cout = HS[(2 * i + 3 * j) % 4], COUTS[(i + j + 3) % 6]
        c0, ctot = (0, cin) if k % 2 == 0 else (2, cin + 5)
        out.append(dict(name=f"h{hid}_cin{cin}_cout{cout}_{geom}" + ("_slice" if c0 else ""), hid=hid, cin=cin,
                        cout=cout, geom=geom, c0=c0, ctot=ctot, leaky=LEAKS[k % 3], scale=SCALES[(k // 3) % 3],
                        seed=300 + k))
    return out


SWEEP = _sweep()
BY_NAME = {c["name"]: c for c in SWEEP}
DEEPEST = [c["name"] for c in SWEEP if (c["hid"], c["cin"], c["cout"]) == (256, 28, 56)][0]


def make_case(cfg, batch=None):
    """(ConvNet2d on the CPU, its weights as fp32 numpy arrays, input x [B, ctot, H, W]).  The net's constructor runs
    under torch.manual_seed(seed)."""
    B, H, W = GEOMS[cfg["geom"]]
    B = B if batch is None else batch
    torch.manual_seed(cfg["seed"])
    net = nf.nets.ConvNet2d((cfg["cin"], cfg["hid"], cfg["hid"], cfg["cout"]), (3, 1, 3), cfg["leaky"],
                            init_zeros=cfg["scale"] == "zero")
    if cfg["scale"] == "large":
        with torch.no_grad():
            for p in net.parameters():
                p.mul_(3.0)
    c1, c2, c3 = net.conv_layers()
    w = {k: v.detach().numpy().copy() for k, v in (("w1", c1.weight), ("b1", c1.bias), ("w2", c2.weight),
                                                   ("b2", c2.bias), ("w3", c3.weight), ("b3", c3.bias))}
    x = (torch.randn(B, cfg["ctot"], H, W, generator=torch.Generator().manual_seed(cfg["seed"] + 1)) * 1.5).numpy()
    return net, w, x


def tap_weights(w3):
    """[cout, hid, 3, 3] -> [9 cout, hid], row (3 kh + kw) cout + n = W3[n, :, kh, kw] (the layout nfb_glow_conditioner
    takes)."""
    return np.ascontiguousarray(w3.transpose(2, 3, 0, 1).reshape(-1, w3.shape[1]))


# ---------------------------------------------------------------------------------------------------------------------
# fp64 references
# ---------------------------------------------------------------------------------------------------------------------
def taps(h, w3):
    """Tap form of the last 3x3 convolution: Y[b, t cout + n] = sum_c W3[n, c, kh, kw] h[b, c], t = 3 kh + kw."""
    cout, hid = w3.shape[:2]
    y = np.einsum("bchw,nct->btnhw", h, w3.reshape(cout, hid, 9), optimize=True)
    return y.reshape(h.shape[0], 9 * cout, *h.shape[2:])


def tap_sum(y, bias):
    """out[b, n, y, x] = bias[n] + sum_t Y[b, t cout + n, y + kh - 1, x + kw - 1] (zero outside the image)."""
    B, n9, H, W = y.shape
    cout = n9 // 9
    yp = np.pad(y.reshape(B, 9, cout, H, W).astype(np.float64), ((0, 0), (0, 0), (0, 0), (1, 1), (1, 1)))
    out = np.zeros((B, cout, H, W))
    if bias is not None:
        out += np.asarray(bias, np.float64)[None, :, None, None]
    for kh in range(3):
        for kw in range(3):
            out += yp[:, 3 * kh + kw, :, kh:kh + H, kw:kw + W]
    return out


def _conv3x3_wrapped(x, c0, cin, w1, b1):
    """The first convolution with im2col's column check dropped: a tap left or right of the image reads the flat
    [B, ctot, H, W] array at row * W + column, i.e. the neighbouring row's first / last pixel (outside the array: 0)."""
    B, ctot, H, W = x.shape
    flat = x.reshape(-1)
    r0, q0 = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    base = (np.arange(B)[:, None] * ctot + c0 + np.arange(cin)[None, :]) * (H * W)
    out = np.zeros((B, w1.shape[0], H, W)) + b1[None, :, None, None]
    for kh in range(3):
        for kw in range(3):
            r, q = r0 + kh - 1, q0 + kw - 1
            idx = base[:, :, None, None] + (r * W + q)[None, None]
            ok = ((r >= 0) & (r < H))[None, None] & (idx >= 0) & (idx < flat.size)
            col = np.where(ok, flat[np.clip(idx, 0, flat.size - 1)], 0.0)
            out += np.einsum("bchw,nc->bnhw", col, w1[:, :, kh, kw], optimize=True)
    return out


def conditioner_oracle(x, c0, cin, w, leaky, absolute=False, wrap=False):
    """(Y, h2) of the conditioner in fp64: h1 = act(conv3x3(x[:, c0:c0+cin]) + b1), h2 = act(conv1x1(h1) + b2),
    Y = taps(h2, W3).  absolute: the same network on |x|, |W|, |b| with identity activations (the error model's scale).
    wrap: the first convolution as _conv3x3_wrapped (a mutant)."""
    f = np.abs if absolute else (lambda a: a)
    w = {k: f(v.astype(np.float64)) for k, v in w.items()}
    act = (lambda a: a) if absolute else (lambda a: O.leaky_relu(a, leaky))
    x = f(np.asarray(x, np.float64))
    h1 = _conv3x3_wrapped(x, c0, cin, w["w1"], w["b1"]) if wrap else O.conv2d(x[:, c0:c0 + cin], w["w1"], w["b1"])
    h2 = act(O.conv2d(act(h1), w["w2"], w["b2"]))
    return taps(h2, w["w3"]), h2


def conditioner_scales(x, c0, cin, w, leaky):
    """(|net|, Q) of the error model: the absolute network, and Q with Q1^2 = conv(x^2, W1^2),
    Q2^2 = conv(Q1^2 + h1^2, W2^2), Q^2 = taps(Q2^2 + h2^2, W3^2) (an input's error and the layer's own products)."""
    w64 = {k: v.astype(np.float64) for k, v in w.items()}
    x = np.asarray(x, np.float64)[:, c0:c0 + cin]
    h1 = O.leaky_relu(O.conv2d(x, w64["w1"], w64["b1"]), leaky)
    h2 = O.leaky_relu(O.conv2d(h1, w64["w2"], w64["b2"]), leaky)
    q1 = O.conv2d(x ** 2, w64["w1"] ** 2)
    q2 = O.conv2d(q1 + h1 ** 2, w64["w2"] ** 2)
    q3 = taps(q2 + h2 ** 2, w64["w3"] ** 2)
    return conditioner_oracle(x, 0, cin, w, leaky, absolute=True)[0], np.sqrt(q3)


def check_taps(y, ref, scales, what=""):
    """|y - ref| <= KAPPA |net| + FLOOR and <= Z_Q SIGMA_P Q + 16 u |net| + FLOOR element by element; returns the worst
    ratio of error to each bound."""
    y = np.asarray(y, np.float64)
    net, q = scales
    assert y.shape == ref.shape and np.all(np.isfinite(y)), f"{what}: shape {y.shape} / non-finite y_taps"
    err = np.abs(y - ref)
    worst = []
    for name, bound in (("kappa |net|", KAPPA * net + FLOOR), ("Z sigma Q", Z_Q * SIGMA_P * q + 16 * U32 * net + FLOOR)):
        ratio = err / bound
        i = np.unravel_index(np.argmax(ratio), ratio.shape)
        assert ratio[i] <= 1.0, \
            f"{what}: y_taps{list(i)} = {y[i]!r} vs {ref[i]!r} (|net| {net[i]:.3e}, Q {q[i]:.3e}): {ratio[i]:.3g} x {name}"
        worst.append(float(ratio[i]))
    return worst


# ---- the tap-form coupling ------------------------------------------------------------------------------------------
SMAPS = {"exp": 0, "sigmoid": 1, "sigmoid_inv": 2}
MODES = [(True, "exp"), (True, "sigmoid"), (True, "sigmoid_inv"), (False, "exp")]   # (scale, scale_map)
SPLITS = ("channel", "channel_inv")
COUPLING_SHAPES = [(3, 7, 4, 4), (5, 7, 3, 5), (4, 5, 5, 3)]   # (B, C, H, W)


def coupling_dims(C, scale, split):
    """(offset of the transformed chunk, its channels n2, conditioner outputs cout) as the coupling kernels take them."""
    h = (C + 1) // 2
    o2, n2 = (h, C - h) if split == "channel" else (0, h)
    return o2, n2, (2 if scale else 1) * n2


def staging_path(C, H, W, scale, split):
    """coupling_taps_kernel stages a sample's taps with float4 loads when 9 cout HW % 4 == 0 (the tensors here are
    allocated 16-byte aligned), element by element otherwise."""
    return "float4" if 9 * coupling_dims(C, scale, split)[2] * H * W % 4 == 0 else "scalar"


def coupling_case(B, C, H, W, scale, split, seed):
    """z [B, C, H, W], taps Y [B, 9 cout, H, W], bias [cout], log-det constant, previous log-det [B]."""
    rng = np.random.default_rng(seed)
    cout = coupling_dims(C, scale, split)[2]
    return (rng.normal(size=(B, C, H, W)).astype(np.float32), (0.2 * rng.normal(size=(B, 9 * cout, H, W))).astype(np.float32),
            (0.3 * rng.normal(size=cout)).astype(np.float32), np.float32(rng.normal() * 3),
            rng.normal(size=B).astype(np.float32))


def coupling_oracle(z, Y, bias, ldc, ld0, scale, smap, split, direction, accumulate, param=None):
    """fp64 (z', log-det) of the coupling whose parameters are the tap sum of Y plus bias (O.affine_coupling_apply),
    and the error bounds of an fp32 kernel: (out, ld, tol_out, tol_ld)."""
    z64 = z.astype(np.float64)
    param = tap_sum(Y, bias) if param is None else param
    pabs = tap_sum(np.abs(Y), None if bias is None else np.abs(bias))
    spec = dict(scale=scale, scale_map=smap, split_mode=split)
    out, ld = O.affine_coupling_apply(z64, param, spec, "forward" if direction else "inverse")
    o2, n2, _ = coupling_dims(z.shape[1], scale, split)
    B, HW = z.shape[0], z.shape[2] * z.shape[3]
    dp = 12 * U32 * pabs                                   # fp32 sum of bias and <= 9 taps
    zt = np.abs(z64[:, o2:o2 + n2])
    tol = 16 * U32 * np.abs(out)
    if not scale:
        tol[:, o2:o2 + n2] += dp + 4 * U32 * zt
        lterm, dl = np.zeros((B, 1)), np.zeros(B)
    else:
        shift, sc, dsh, dsc = param[:, 0::2], param[:, 1::2], dp[:, 0::2], dp[:, 1::2]
        # the factor on z (or z - shift) and d log(factor) / d sc <= 1 in magnitude for all three maps
        fac = np.exp(np.abs(sc)) if smap == "exp" else 1.0 / O.sigmoid(sc + 2)
        tol[:, o2:o2 + n2] += fac * (dsh + (zt + np.abs(shift)) * (dsc + 16 * U32) + 16 * U32 * np.abs(shift))
        lterm = (np.abs(sc) if smap == "exp" else np.abs(np.log(O.sigmoid(sc + 2)))).reshape(B, -1)
        dl = dsc.reshape(B, -1).sum(axis=1)
    if ldc is not None:
        ld = ld + np.float64(ldc)
    if accumulate:
        ld = ld + ld0.astype(np.float64)
    depth = n2 * HW / 256 + 24                             # per-thread sums, warp tree, 8 partials, + constant
    mag = lterm.sum(axis=1) + (0 if ldc is None else abs(float(ldc))) + (np.abs(ld0) if accumulate else 0)
    return out, ld, tol + FLOOR, dl + depth * U32 * mag + 4 * U32 * lterm.sum(axis=1) + FLOOR


def check_coupling(z, ld, ref, what=""):
    out, ld_ref, tol, tol_ld = ref
    z, ld = np.asarray(z, np.float64), np.asarray(ld, np.float64)
    assert np.all(np.isfinite(z)) and np.all(np.isfinite(ld)), f"{what}: non-finite output"
    r = np.abs(z - out) / tol
    i = np.unravel_index(np.argmax(r), r.shape)
    assert r[i] <= 1.0, f"{what}: z{list(i)} = {z[i]!r} vs {out[i]!r}: {r[i]:.3g} x bound"
    rl = np.abs(ld - ld_ref) / tol_ld
    j = int(np.argmax(rl))
    assert rl[j] <= 1.0, f"{what}: log-det[{j}] = {ld[j]!r} vs {ld_ref[j]!r}: {rl[j]:.3g} x bound"
    return max(float(r[i]), float(rl[j]))


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the designs cover what they claim; the assertions reject wrong kernels
# ---------------------------------------------------------------------------------------------------------------------
def test_sweep_is_a_covering_design():
    axes = {"hid": HS, "cin": CINS, "cout": COUTS, "geom": tuple(GEOMS)}
    for a, b in (("hid", "cin"), ("hid", "cout"), ("cin", "geom")):
        have = {(c[a], c[b]) for c in SWEEP}
        want = set(itertools.product(axes[a], axes[b]))
        assert want <= have, (a, b, sorted(want - have))
    assert {c["cout"] for c in SWEEP} == set(COUTS) and {c["hid"] for c in SWEEP} == set(HS)
    assert {c["leaky"] for c in SWEEP} == set(LEAKS)
    assert {(c["leaky"], c["scale"]) for c in SWEEP} == set(itertools.product(LEAKS, SCALES))
    assert {c["c0"] > 0 and c["ctot"] > c["c0"] + c["cin"] for c in SWEEP} == {False, True}
    assert all(c["c0"] == 0 and c["ctot"] == c["cin"] for c in SWEEP if c["c0"] == 0)
    assert 25 <= len(SWEEP) <= 35 and len(BY_NAME) == len(SWEEP)
    # the shapes are what the kernel's loops are sized by
    assert sorted({(9 * c + 63) // 64 for c in CINS}) == [1, 2, 3, 4] and 9 * max(CINS) == 252
    assert sorted({(9 * c + 63) // 64 for c in COUTS}) == [1, 2, 7, 8] and 9 * max(COUTS) == 504
    assert {9 * c % 64 for c in COUTS} >= {63, 3}          # last slice one column short of full / three real columns
    B, H, W = GEOMS[MANY]
    assert B * H * W > 4 * 132 * 64 and 64 % (H * W) and B * H * W % 64
    assert GEOMS["4x4"][0] * 16 % 64 and GEOMS["1x1"][1:] == (1, 1)


def test_coupling_design_takes_both_staging_paths():
    for (scale, _), split in itertools.product(MODES, SPLITS):
        paths = {staging_path(C, H, W, scale, split) for _, C, H, W in COUPLING_SHAPES}
        assert paths == {"float4", "scalar"}, (scale, split, paths)
    # 9 cout HW odd: odd HW, scale=False, odd n2
    assert any(9 * coupling_dims(C, False, s)[2] * H * W % 2 for _, C, H, W in COUPLING_SHAPES for s in SPLITS)
    # odd C: unequal halves, so n2 differs between the two split modes
    assert any(coupling_dims(C, True, "channel")[1] != coupling_dims(C, True, "channel_inv")[1]
               for _, C, _, _ in COUPLING_SHAPES)


def _mutants(cfg, w, x):
    """(what, Y) for each slip of the fused conditioner, as the oracle's output on a mutated state."""
    c0, cin, leaky, hid, cout = cfg["c0"], cfg["cin"], cfg["leaky"], cfg["hid"], cfg["cout"]

    def run(w2=None, x2=None, **kw):
        kw.setdefault("leaky", leaky)
        return conditioner_oracle(x if x2 is None else x2, c0, cin, w if w2 is None else w2, **kw)[0]

    def with_(**upd):
        return dict(w, **upd)
    out = []
    if hid >= 128:   # the last [64 x 64] record of GEMM 2 never multiplied
        w2 = w["w2"].copy()
        w2[hid - 64:, hid - 64:] = 0
        out.append(("GEMM 2 record", run(with_(w2=w2))))
    w1 = w["w1"].copy()
    w1[:, cin - 1] = 0     # c < cin - 1
    out.append(("last input channel", run(with_(w1=w1))))
    w3 = w["w3"].copy()
    w3[cout - 1, :, 2, 2] = 0    # column 9 cout - 1 = tap 8, output cout - 1
    out.append(("last GEMM 3 column", run(with_(w3=w3))))
    w3 = w["w3"].copy()
    w3[:, :, 1, 0] = 0
    out.append(("one tap", run(with_(w3=w3))))
    out.append(("im2col column wrap", run(wrap=True)))
    if leaky > 0:
        out.append(("LeakyReLU slope", run(leaky=0.0)))
    # one hidden bias left out: the one that moves the output most
    h2 = conditioner_oracle(x, c0, cin, w, leaky)[1]
    j = int(np.argmax(np.abs(w["b2"]) * (h2 > 0).mean(axis=(0, 2, 3)) * np.abs(w["w3"]).sum(axis=(0, 2, 3))))
    b2 = w["b2"].copy()
    b2[j] = 0
    out.append(("hidden bias", run(with_(b2=b2))))
    return out


MUTANT_CFGS = [c["name"] for c in SWEEP if c["scale"] != "zero" and c["geom"] in ("16x16", "3x5") and c["hid"] >= 128
               and c["leaky"] == 0.01]


@pytest.mark.parametrize("name", MUTANT_CFGS)
def test_tolerances_reject_a_wrong_conditioner(name):
    """The oracle's output for a mutated state stands in for a kernel with that slip; the comparison of the GPU sweep
    must fail on it at the row's own sample size."""
    cfg = BY_NAME[name]
    _, w, x = make_case(cfg)
    ref = conditioner_oracle(x, cfg["c0"], cfg["cin"], w, cfg["leaky"])[0]
    scales = conditioner_scales(x, cfg["c0"], cfg["cin"], w, cfg["leaky"])
    check_taps(ref.astype(np.float32), ref, scales, name)     # the correct answer, rounded to fp32, passes
    mut = _mutants(cfg, w, x)
    assert len(mut) == 7
    for what, y in mut:
        with pytest.raises(AssertionError):
            check_taps(y, ref, scales, f"{name} / {what}")


def _coupling_mutants(z, Y, bias, scale, smap, split, direction):
    """(what, z', log-det) of a coupling kernel with the split modes swapped (it reads Y with the other mode's cout and
    per-sample stride and transforms the other chunk) or the sigmoid / sigmoid_inv division swapped."""
    out = []
    other = SPLITS[1 - SPLITS.index(split)]
    B, C, H, W = z.shape
    cout2 = coupling_dims(C, scale, other)[2]
    per = 9 * cout2 * H * W
    flat = np.concatenate([Y.reshape(-1), np.zeros(B * per)])[:B * per]
    b2 = np.concatenate([bias, np.zeros(cout2)])[:cout2]
    r = coupling_oracle(z, flat.reshape(B, 9 * cout2, H, W), b2, None, None, scale, smap, other, direction, 0)
    out.append(("split modes swapped", r[0], r[1]))
    if smap != "exp":
        r = coupling_oracle(z, Y, bias, None, None, scale, {"sigmoid": "sigmoid_inv", "sigmoid_inv": "sigmoid"}[smap],
                            split, direction, 0)
        out.append(("sigmoid division swapped", r[0], r[1]))
    return out


COUPLING_MUTANT_CASES = [(mode, split, d) for mode in MODES if mode[0] for split in SPLITS for d in (0, 1)]


@pytest.mark.parametrize("mode,split,direction", COUPLING_MUTANT_CASES)
def test_tolerances_reject_a_wrong_coupling(mode, split, direction):
    scale, smap = mode
    for k, (B, C, H, W) in enumerate(COUPLING_SHAPES):
        z, Y, bias, _, _ = coupling_case(B, C, H, W, scale, split, 40 + k)
        ref = coupling_oracle(z, Y, bias, None, None, scale, smap, split, direction, 0)
        check_coupling(ref[0].astype(np.float32), ref[1].astype(np.float32), ref, "fp32-rounded oracle")
        for what, zm, ldm in _coupling_mutants(z, Y, bias, scale, smap, split, direction):
            with pytest.raises(AssertionError):
                check_coupling(zm, ldm, ref, what)


def test_mutant_configs_are_in_the_sweep():
    assert len(MUTANT_CFGS) >= 2
    for n in MUTANT_CFGS:
        c = BY_NAME[n]
        assert c in SWEEP and c["hid"] >= 128 and c["leaky"] == 0.01 and c["scale"] != "zero" and c["geom"] != MANY
    assert {BY_NAME[n]["geom"] for n in MUTANT_CFGS} == {"16x16", "3x5"}
    # the coupling mutants run on the shapes and options the GPU coupling test uses
    assert {(m, s, d) for m, s, d in COUPLING_MUTANT_CASES} <= set(itertools.product(MODES, SPLITS, (0, 1)))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def _np(t):
    return t.detach().cpu().numpy()


def _lib():
    from normflows import _lib as L
    return L


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def run_conditioner(cfg, w, x, packed=True):
    """y_taps [B, 9 cout, H, W] of the fused kernel: packed = nfb_glow_conditioner_pack + _packed, else the
    unpacked nfb_glow_conditioner (packs on every call)."""
    L = _lib()
    lib, st = L.lib(), L.stream_ptr()
    B, _, H, W = x.shape
    cin, hid, cout = cfg["cin"], cfg["hid"], cfg["cout"]
    xd, w1, b1, w2, b2, w3t = (cuda(a) for a in (x, w["w1"], w["b1"], w["w2"], w["b2"], tap_weights(w["w3"])))
    y = _nan(B, 9 * cout, H, W)
    if packed:
        nbytes = lib.nfb_glow_conditioner_packed_bytes(cin, hid, cout)
        assert nbytes == ((hid // 64) * ((9 * cin + 63) // 64) + (hid // 64) ** 2 + (9 * cout + 63) // 64 * (hid // 64)) * 16384
        buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        L.check(lib.nfb_glow_conditioner_pack(L.ptr(w1), L.ptr(w2), L.ptr(w3t), cin, hid, cout, L.ptr(buf), st))
        L.check(lib.nfb_glow_conditioner_packed(L.ptr(xd), cfg["ctot"], cfg["c0"], cin, L.ptr(buf), L.ptr(b1), L.ptr(b2),
                                                L.ptr(y), B, H, W, hid, cout, float(cfg["leaky"]), st))
    else:
        L.check(lib.nfb_glow_conditioner(L.ptr(xd), cfg["ctot"], cfg["c0"], cin, L.ptr(w1), L.ptr(b1), L.ptr(w2),
                                         L.ptr(b2), L.ptr(w3t), L.ptr(y), B, H, W, hid, cout, float(cfg["leaky"]), st))
    return _np(y)


def _same(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and np.array_equal(a, b, equal_nan=True), \
        f"{what}: {np.sum(a != b)} elements differ, max {np.nanmax(np.abs(a.astype(np.float64) - b)):.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c["name"] for c in SWEEP])
def test_conditioner_matches_oracle(name):
    cfg = BY_NAME[name]
    _, w, x = make_case(cfg)
    y = run_conditioner(cfg, w, x)
    _same(run_conditioner(cfg, w, x, packed=False), y, "unpacked vs packed y_taps")
    if cfg["scale"] == "zero":
        assert np.all(y == 0), f"{np.sum(y != 0)} non-zero y_taps with an all-zero last convolution"
    imgs = list(MANY_IMAGES) if cfg["geom"] == MANY else slice(None)
    if cfg["geom"] == MANY:
        # one image alone (one or two tiles from offset 0) equals the same image inside the batch (another tile offset)
        for b in MANY_IMAGES:
            _same(run_conditioner(cfg, w, x[b:b + 1])[0], y[b], f"image {b} alone vs in the batch")
    ref, h2 = conditioner_oracle(x[imgs], cfg["c0"], cfg["cin"], w, cfg["leaky"])
    worst = check_taps(y[imgs], ref, conditioner_scales(x[imgs], cfg["c0"], cfg["cin"], w, cfg["leaky"]), name)
    print(f"[glow-configs] {name}: leaky {cfg['leaky']} {cfg['scale']}: worst |dY| / (kappa |net|) = {worst[0]:.3e}, "
          f"/ (Z sigma Q + 16 u |net|) = {worst[1]:.3e}")
    # the shifted tap sum of the reference taps against the oracle's direct 3x3 convolution
    L = _lib()
    B, _, H, W = ref.shape
    out, yd, b3 = _nan(B, cfg["cout"], H, W), cuda(ref), cuda(w["b3"])
    L.check(L.lib().nfb_tap_shift_add(L.ptr(yd), L.ptr(b3), L.ptr(out), B, cfg["cout"], H, W, 3, L.stream_ptr()))
    direct = O.conv2d(h2, w["w3"].astype(np.float64), w["b3"].astype(np.float64))
    bound = 12 * U32 * tap_sum(np.abs(ref), np.abs(w["b3"])) + FLOOR
    err = np.abs(_np(out) - direct)
    assert np.all(err <= bound), f"tap_shift_add: {np.max(err / bound):.3g} x bound"


NET_CFGS = [c["name"] for c in SWEEP if c["c0"] == 0 and c["geom"] != MANY and c["scale"] != "zero"][:4]


@pytest.mark.gpu
@pytest.mark.parametrize("name", NET_CFGS)
def test_convnet2d_forward_takes_the_fused_kernel(name):
    """ConvNet2d.forward end to end (fused conditioner + tap sum) against O.convnet2d."""
    cfg = BY_NAME[name]
    net, w, x = make_case(cfg)
    net = net.cuda()
    assert net.glow_shape(cfg["cin"]), "the Glow conditioner shape must take the fused kernel"
    got = _np(net(cuda(x)))
    sd = {"net." + k: v.detach().cpu().numpy().astype(np.float64) for k, v in net.net.state_dict().items()}
    ref = O.convnet2d(x.astype(np.float64), sd, "", leaky=cfg["leaky"])
    net_abs, q = conditioner_scales(x, 0, cfg["cin"], w, cfg["leaky"])
    check_taps(got, ref, (tap_sum(net_abs, np.abs(w["b3"])), np.sqrt(tap_sum(q ** 2, None))), name)


@pytest.mark.gpu
def test_conditioner_signed_bias():
    """No one-sided accumulate bias left (the gain of launch_glow_cond_pack, 12 kcs steps per GEMM) on the deepest
    configuration with unit-scale data: He-scaled weights keep every layer's output near unit scale.  Uncompensated,
    3 GEMMs x 48 steps x 2.4e-8 would take ~3.5e-6 of every output: the fitted relative gain must stay below half that;
    the mean error, as for the tensor-core convolution, below 3e-6.  Measured on an H100 80GB HBM3 (700 W limit): fitted
    gain +1.15e-6 with the gain, -2.31e-6 without it (NFB_ACC_COMP_STEP=0), mean error -7.6e-8."""
    cfg = dict(BY_NAME[DEEPEST], leaky=0.0, c0=0, ctot=28)
    hid, cin, cout = cfg["hid"], cfg["cin"], cfg["cout"]
    rng = np.random.default_rng(5)
    w = {"w1": rng.normal(0, np.sqrt(2 / (9 * cin)), (hid, cin, 3, 3)), "b1": rng.normal(0, 0.1, hid),
         "w2": rng.normal(0, np.sqrt(2 / hid), (hid, hid, 1, 1)), "b2": rng.normal(0, 0.1, hid),
         "w3": rng.normal(0, np.sqrt(1 / hid), (cout, hid, 3, 3)), "b3": np.zeros(cout)}
    w = {k: v.astype(np.float32) for k, v in w.items()}
    x = rng.normal(size=(8, cin, 16, 16)).astype(np.float32)
    y = run_conditioner(cfg, w, x).astype(np.float64)
    ref = conditioner_oracle(x, 0, cin, w, 0.0)[0]
    d = y - ref
    gain = float(np.sum(d * ref) / np.sum(ref * ref))
    print(f"[glow-configs] signed bias h256 cin28 cout56 8x16x16: mean(y - ref) = {d.mean():.3e}, "
          f"rms(ref) = {np.sqrt(np.mean(ref ** 2)):.3f}, fitted relative gain = {gain:.3e}")
    assert abs(d.mean()) < 3e-6
    assert abs(gain) < 1.75e-6


@pytest.mark.gpu
def test_conditioner_edge_calls():
    L = _lib()
    lib, st = L.lib(), L.stream_ptr()
    dummy = torch.zeros(4096, device="cuda")
    y = _nan(64)
    p = L.ptr(dummy)
    # an empty batch: nothing to do
    assert lib.nfb_glow_conditioner(p, 4, 0, 4, p, p, p, p, p, L.ptr(y), 0, 8, 8, 64, 8, 0.0, st) == 0
    assert lib.nfb_glow_conditioner_packed(p, 4, 0, 4, p, p, p, L.ptr(y), 0, 8, 8, 64, 8, 0.0, st) == 0
    for cin, hid, cout in [(29, 64, 8), (0, 64, 8), (4, 96, 8), (4, 320, 8), (4, 0, 8), (4, 64, 57), (4, 64, 0)]:
        assert lib.nfb_glow_conditioner_packed_bytes(cin, hid, cout) == -1, (cin, hid, cout)
        assert lib.nfb_glow_conditioner(p, cin, 0, cin, p, p, p, p, p, L.ptr(y), 1, 2, 2, hid, cout, 0.0, st) == 3
        assert lib.nfb_glow_conditioner_packed(p, cin, 0, cin, p, p, p, L.ptr(y), 1, 2, 2, hid, cout, 0.0, st) == 3
        assert lib.nfb_glow_conditioner_pack(p, p, p, cin, hid, cout, p, st) == 3
    torch.cuda.synchronize()
    assert torch.isnan(y).all(), "an unsupported call wrote its output"
    assert lib.nfb_glow_conditioner_packed_bytes(28, 256, 56) > 0 and lib.nfb_glow_conditioner_packed_bytes(1, 64, 1) > 0


# ---- the tap-form coupling ------------------------------------------------------------------------------------------
def _opt(a):
    """Device copy of an optional array (None stays None)."""
    return None if a is None else cuda(np.asarray(a))


def run_coupling_taps(z, Y, bias, ldc, ld0, scale, smap, split, direction, accumulate):
    """(z', log-det, return code) of nfb_affine_coupling_image_taps on copies of z and ld0."""
    L = _lib()
    B, C, H, W = z.shape
    zd, ld, yd, bd, cd = cuda(z), cuda(ld0), cuda(Y), _opt(bias), _opt(ldc)   # alive until the kernel has run
    rc = L.lib().nfb_affine_coupling_image_taps(L.ptr(zd), L.ptr(yd), L.ptr(bd), L.ptr(ld), L.ptr(cd), B, C, H, W,
                                                int(scale), SMAPS[smap], SPLITS.index(split), direction, accumulate,
                                                L.stream_ptr())
    return _np(zd), _np(ld), rc


@pytest.mark.gpu
@pytest.mark.parametrize("direction", [0, 1])
@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("mode", MODES, ids=["exp", "sigmoid", "sigmoid_inv", "noscale"])
def test_tap_coupling_matches_oracle(mode, split, direction):
    """nfb_affine_coupling_image_taps against the oracle coupling over accumulate x log-det constant x bias, on shapes
    that stage with float4 loads and shapes that stage element by element; and bit for bit against the shifted tap sum
    followed by nfb_affine_coupling_image (both add the bias, then the taps in (kh, kw) order)."""
    L = _lib()
    scale, smap = mode
    worst, paths = 0.0, set()
    for k, (B, C, H, W) in enumerate(COUPLING_SHAPES):
        z, Y, bias0, ldc0, ld0 = coupling_case(B, C, H, W, scale, split, 60 + k)
        cout = coupling_dims(C, scale, split)[2]
        paths.add(staging_path(C, H, W, scale, split))
        for accumulate, with_ldc, with_bias in itertools.product((0, 1), (False, True), (False, True)):
            bias, ldc = (bias0 if with_bias else None), (ldc0 if with_ldc else None)
            what = f"{B}x{C}x{H}x{W} acc={accumulate} ldc={with_ldc} bias={with_bias}"
            zt, ldt, rc = run_coupling_taps(z, Y, bias, ldc, ld0, scale, smap, split, direction, accumulate)
            assert rc == 0, L.lib().nfb_last_error()
            ref = coupling_oracle(z, Y, bias, ldc, ld0, scale, smap, split, direction, accumulate)
            worst = max(worst, check_coupling(zt, ldt, ref, what))
            # the same through the tap sum and the plain coupling kernel
            param, yd, bd, cd = _nan(B, cout, H, W), cuda(Y), _opt(bias), _opt(ldc)
            L.check(L.lib().nfb_tap_shift_add(L.ptr(yd), L.ptr(bd), L.ptr(param), B, cout, H, W, 3, L.stream_ptr()))
            zd, ld = cuda(z), cuda(ld0)
            L.check(L.lib().nfb_affine_coupling_image(L.ptr(zd), L.ptr(param), L.ptr(ld), L.ptr(cd), B, C, H * W,
                                                      int(scale), SMAPS[smap], SPLITS.index(split), direction,
                                                      accumulate, L.stream_ptr()))
            _same(zt, _np(zd), f"{what}: taps vs tap sum + coupling, z")
            _same(ldt, _np(ld), f"{what}: taps vs tap sum + coupling, log-det")
    assert paths == {"float4", "scalar"}
    print(f"[glow-configs] coupling {mode} {split} dir {direction}: worst error / bound = {worst:.3e}")


# (scale, (H, W) just inside, (H, W) just outside) for C = 7: 9 (1 + scale) 4 HW * 4 bytes against 200 KB
LIMIT_PAIRS = [(True, (9, 79), (8, 89)), (False, (18, 79), (1, 1423))]


@pytest.mark.gpu
@pytest.mark.parametrize("scale,inside,outside", LIMIT_PAIRS, ids=["scale", "noscale"])
def test_tap_coupling_shared_memory_limit(scale, inside, outside):
    L = _lib()
    C, h = 7, 4
    for (H, W), fits in ((inside, True), (outside, False)):
        assert (9 * (2 if scale else 1) * h * H * W * 4 <= 200 * 1024) == fits
        assert L.lib().nfb_affine_coupling_image_taps_supported(C, H, W, int(scale)) == int(fits)
        z, Y, bias, ldc, ld0 = coupling_case(2, C, H, W, scale, "channel_inv", 7)   # n2 = h: the full 200 KB
        smap = "sigmoid" if scale else "exp"
        zt, ldt, rc = run_coupling_taps(z, Y, bias, ldc, ld0, scale, smap, "channel_inv", 0, 0)
        if fits:
            assert rc == 0, L.lib().nfb_last_error()
            check_coupling(zt, ldt, coupling_oracle(z, Y, bias, ldc, ld0, scale, smap, "channel_inv", 0, 0), f"{H}x{W}")
        else:
            assert rc == 3 and b"shared memory" in L.lib().nfb_last_error()
            _same(zt, z, "z after a refused call")
            _same(ldt, ld0, "log-det after a refused call")


# ---- one-call GlowBlock ---------------------------------------------------------------------------------------------
BLOCK_CS = {2: (4, 6, 10), 7: (3, 5, 7), 24: (2, 9, 11), 48: (2, 8, 8)}   # channels: (B, H, W) inside the 200 KB limit
COMBOS = [(s, m, sp) for s, m in MODES for sp in SPLITS]


def _block_rows():
    """channels x hidden in full (16 rows); every (scale, scale map, split) combination twice, once per slope."""
    out = []
    for k, (C, hid) in enumerate(itertools.product(BLOCK_CS, HS)):
        scale, smap, split = COMBOS[(k + 2 * (k // 4)) % 8]
        out.append(dict(name=f"c{C}_h{hid}_{smap if scale else 'noscale'}_{split}", C=C, hid=hid, scale=scale,
                        smap=smap, split=split, leaky=(0.0, 0.2)[(k // 2) % 2], seed=500 + k))
    return out


BLOCK_ROWS = _block_rows()


def test_block_grid_covers_every_coupling_option():
    assert {(r["C"], r["hid"]) for r in BLOCK_ROWS} == set(itertools.product(BLOCK_CS, HS))
    assert {(r["scale"], r["smap"], r["split"]) for r in BLOCK_ROWS} == set(COMBOS)
    assert {(r["scale"], r["smap"], r["split"], r["leaky"]) for r in BLOCK_ROWS} == \
        set((*c, lk) for c in COMBOS for lk in (0.0, 0.2))
    for C, (B, H, W) in BLOCK_CS.items():
        assert 9 * 2 * ((C + 1) // 2) * H * W * 4 <= 200 * 1024 and 9 * ((C + 1) // 2) <= 256


@pytest.mark.gpu
@pytest.mark.parametrize("row", BLOCK_ROWS, ids=[r["name"] for r in BLOCK_ROWS])
def test_glow_block_one_call_matches_oracle(row, monkeypatch):
    C, hid = row["C"], row["hid"]
    B, H, W = BLOCK_CS[C]
    torch.manual_seed(row["seed"])
    blk = nf.flows.GlowBlock(C, hid, scale=row["scale"], scale_map=row["smap"], split_mode=row["split"],
                             leaky=row["leaky"])
    g = torch.Generator().manual_seed(row["seed"] + 1)
    last = blk._param_map().conv_layers()[-1]
    with torch.no_grad():
        last.weight.copy_(0.05 * torch.randn(last.weight.shape, generator=g))
        last.bias.copy_(0.1 * torch.randn(last.bias.shape, generator=g))
    blk = blk.cuda()
    taken = []
    one_call = nf.flows.GlowBlock._one_call

    def spy(self, *a):
        r = one_call(self, *a)
        taken.append(r)
        return r
    monkeypatch.setattr(nf.flows.GlowBlock, "_one_call", spy)
    z = (1.5 * torch.randn(B, C, H, W, generator=g)).numpy()
    zi, ldi = blk.inverse(cuda(z))          # initialises ActNorm from this batch first
    xs, lds = blk.forward(cuda(z))
    assert taken == [True, True], "nfb_glow_block was not taken"
    sd = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in blk.state_dict().items()}
    assert sd["flows.2.data_dep_init_done"] == 1.0
    spec = dict(scale=row["scale"], scale_map=row["smap"], split_mode=row["split"], leaky=row["leaky"])
    for direction, (got, ld) in (("inverse", (zi, ldi)), ("forward", (xs, lds))):
        zo, ldo = O.glow_block(z.astype(np.float64), sd, "", spec, direction)
        np.testing.assert_allclose(_np(got), zo, rtol=1e-4, atol=2e-4, err_msg=direction)
        np.testing.assert_allclose(_np(ld), ldo, rtol=1e-4, atol=5e-3, err_msg=direction + " log-det")
    zr, ldr = blk.forward(zi)
    np.testing.assert_allclose(_np(zr), z, rtol=1e-4, atol=5e-4, err_msg="forward(inverse(z))")
    assert np.abs(_np(ldr + ldi)).max() < 5e-3
    # the step-by-step path (fold, fused conditioner, tap sum, coupling): the same sums in the same order
    monkeypatch.setattr(nf.flows.GlowBlock, "_one_call", lambda self, *a: False)
    zi2, ldi2 = blk.inverse(cuda(z))
    xs2, lds2 = blk.forward(cuda(z))
    for a, b, what in ((zi, zi2, "inverse z"), (ldi, ldi2, "inverse log-det"), (xs, xs2, "forward x"),
                       (lds, lds2, "forward log-det")):
        _same(_np(a), _np(b), f"one call vs step by step: {what}")


@pytest.mark.gpu
def test_glow_block_sampling_beyond_the_forward_fold_raises():
    """The sampling fold inverts W on one block, C <= 64: a 96-channel LU GlowBlock says so instead of answering."""
    torch.manual_seed(3)
    blk = nf.flows.GlowBlock(96, 64).cuda()
    z = torch.randn(2, 96, 4, 4, device="cuda")
    zi, ld = blk.inverse(z)
    assert torch.isfinite(zi).all() and torch.isfinite(ld).all()
    with pytest.raises(NotImplementedError, match="> 64"):
        blk.forward(z)


# ---- the ActNorm + Invertible1x1Conv folds --------------------------------------------------------------------------
FOLD_CS = (2, 3, 12, 48, 64, 128)


def fold_inputs(C, kind, seed):
    torch.manual_seed(seed)
    conv = nf.flows.Invertible1x1Conv(C, use_lu=True)
    f = {k: getattr(conv, k).detach().numpy().astype(np.float32) for k in ("P", "L", "U", "sign_S", "log_S")}
    rng = np.random.default_rng(seed)
    if kind == "ill":
        f["log_S"] = rng.uniform(-3, 3, C).astype(np.float32)
    f["s"] = rng.normal(0, 0.5, C).astype(np.float32)
    f["t"] = rng.normal(0, 1.0, C).astype(np.float32)
    return f


def _lu64(f):
    C = len(f["s"])
    lo = np.tril(f["L"].astype(np.float64), -1) + np.eye(C)
    up = np.triu(f["U"].astype(np.float64), 1) + np.diag(f["sign_S"].astype(np.float64) * np.exp(f["log_S"].astype(np.float64)))
    return f["P"].astype(np.float64), lo, up


def run_fold(f, C, hw, direction):
    L = _lib()
    fn = L.lib().nfb_glow_fold_actnorm_conv1x1 if direction == 0 else L.lib().nfb_glow_fold_conv1x1_actnorm_forward
    ins = [cuda(f[k]) for k in ("P", "L", "U", "sign_S", "log_S", "s", "t")]
    w, b, ld = _nan(C, C), _nan(C), _nan(1)
    rc = fn(*[L.ptr(t) for t in ins], C, hw, L.ptr(w), L.ptr(b), L.ptr(ld), L.stream_ptr())
    return _np(w), _np(b), float(_np(ld)[0]), rc


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["constructor", "ill"])
@pytest.mark.parametrize("C", FOLD_CS)
def test_folds_match_numpy(C, kind):
    hw = 12
    f = fold_inputs(C, kind, 70 + C)
    P, lo, up = _lu64(f)
    s, t, log_S = (f[k].astype(np.float64) for k in ("s", "t", "log_S"))
    # density: w = P L U diag(exp(-s)), b = -w t, log-det HW (sum log_S - sum s); fp32 sums of C products
    w, b, ld, rc = run_fold(f, C, hw, 0)
    assert rc == 0, _lib().lib().nfb_last_error()
    w_ref = (P @ lo @ up) * np.exp(-s)[None, :]
    w_abs = (np.abs(P) @ np.abs(lo) @ np.abs(up)) * np.exp(-s)[None, :]
    assert np.all(np.abs(w - w_ref) <= (C + 8) * U32 * w_abs + FLOOR), np.max(np.abs(w - w_ref) / (w_abs + FLOOR))
    b_ref = -(w_ref @ t)
    assert np.all(np.abs(b - b_ref) <= (2 * C + 10) * U32 * (w_abs @ np.abs(t)) + FLOOR)
    ld_ref = hw * (log_S.sum() - s.sum())
    assert abs(ld - ld_ref) <= (C + 4) * U32 * hw * (np.abs(log_S).sum() + np.abs(s).sum())
    if C > 64:
        return
    # sampling: w = diag(exp(s)) U^-1 L^-1 P^T in fp64, rounded once to fp32; b = t
    w, b, ld, rc = run_fold(f, C, hw, 1)
    assert rc == 0, _lib().lib().nfb_last_error()
    w_ref = np.exp(s)[:, None] * (np.linalg.inv(up) @ np.linalg.inv(lo) @ P.T)
    assert np.all(np.abs(w - w_ref) <= 2 * U32 * np.abs(w_ref) + 1e-10 * np.abs(w_ref).max())
    _same(b, f["t"], "sampling fold bias")
    assert abs(ld - hw * (s.sum() - log_S.sum())) <= 2 * U32 * hw * (np.abs(log_S).sum() + np.abs(s).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("direction,C,limit", [(1, 65, b"> 64"), (0, 129, b"> 128")], ids=["sampling", "density"])
def test_folds_refuse_beyond_their_limit(direction, C, limit):
    f = fold_inputs(C, "constructor", 1)
    w, b, ld, rc = run_fold(f, C, 4, direction)
    assert rc == 3 and limit in _lib().lib().nfb_last_error()
    assert np.isnan(w).all() and np.isnan(b).all() and np.isnan(ld)
