"""Training pass of the image path: `MultiscaleFlow.forward_kld(x, y).backward()` (examples/glow.ipynb cell 4).

GPU tests check the new CUDA primitives (convolution weight / data gradient, coupling adjoint) against torch in fp64 on
the CPU, whole Glow models against an independent fp64 torch restatement of the density pass, the identity of the
values with and without gradients, and a short training run against the fp64 numpy oracle.  The CPU test checks that
the library exports the new entry points."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import normflows as nf
from normflows import _lib as L

NEW_SYMBOLS = ("nfb_conv2d_wgrad", "nfb_conv2d_dgrad", "nfb_affine_coupling_image_backward",
               "nfb_gaussian_table_log_prob_backward", "nfb_logit_transform_backward")


def test_new_symbols_exported():
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    handle = ctypes.CDLL(L.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(handle, name), name
        assert name in L.SYMBOLS, name


# ---- primitives ----------------------------------------------------------------------------------------------------
WGRAD_CASES = [  # (k, cin, cout, H, W, B)
    (1, 6, 6, 4, 4, 3), (3, 6, 64, 4, 4, 5), (3, 12, 256, 16, 16, 4), (1, 256, 256, 8, 8, 3),
    (3, 256, 24, 16, 16, 2), (3, 7, 33, 5, 7, 3), (5, 6, 10, 6, 6, 2), (3, 24, 200, 9, 11, 2), (1, 48, 48, 16, 16, 70),
]


@pytest.mark.gpu
@pytest.mark.parametrize("k,cin,cout,H,W,B", WGRAD_CASES)
def test_conv_wgrad_matches_torch(k, cin, cout, H, W, B):
    g = torch.Generator().manual_seed(k * 1000 + cin + cout)
    ctot, c0 = cin + 3, 2
    x = torch.randn(B, ctot, H, W, generator=g, dtype=torch.float64)
    gy = torch.randn(B, cout, H, W, generator=g, dtype=torch.float64)
    xs = x[:, c0:c0 + cin]
    ref_w = torch.nn.grad.conv2d_weight(xs, (cout, cin, k, k), gy, padding=k // 2)
    bound = 1e-4 * torch.nn.grad.conv2d_weight(xs.abs(), (cout, cin, k, k), gy.abs(), padding=k // 2) + 1e-6
    ref_b = gy.sum((0, 2, 3))
    xd, gyd = x.float().cuda(), gy.float().cuda()
    gw = torch.empty(cout, cin, k, k, device="cuda")
    gb = torch.empty(cout, device="cuda")
    for acc in (0, 1):
        L.check(L.lib().nfb_conv2d_wgrad(L.ptr(xd), ctot, c0, L.ptr(gyd), L.ptr(gw), L.ptr(gb), B, cin, H, W, cout, k,
                                         acc, L.stream_ptr()))
        m = 1 + acc
        err = (gw.double().cpu() - m * ref_w).abs()
        assert (err <= m * bound).all(), f"wgrad acc={acc}: max err {err.max():.3e}"
        assert torch.allclose(gb.double().cpu(), m * ref_b, rtol=1e-5, atol=1e-4)


@pytest.mark.gpu
def test_conv_wgrad_longest_pixel_splits():
    """C3's pixel count at its 16x16 level with batch 1024 (B*H*W = 262 144 = 4 096 chunks of 64).  With cin*k*k = 576
    there are 5 A tiles x 1 B tile x 128 splits = 640 units >= two per SM, so the launcher keeps the longest split, 32
    chunks = 2 048 pixels (384 truncating K=16 steps) per accumulator: the error bound of the short cases must hold."""
    k, cin, cout, H, W, B = 3, 64, 24, 16, 16, 1024
    g = torch.Generator().manual_seed(99)
    x = torch.randn(B, cin, H, W, generator=g, dtype=torch.float64)
    gy = torch.randn(B, cout, H, W, generator=g, dtype=torch.float64)
    ref = torch.nn.grad.conv2d_weight(x, (cout, cin, k, k), gy, padding=1)
    bound = 1e-4 * torch.nn.grad.conv2d_weight(x.abs(), (cout, cin, k, k), gy.abs(), padding=1) + 1e-6
    xd, gyd = x.float().cuda(), gy.float().cuda()
    gw = torch.empty(cout, cin, k, k, device="cuda")
    L.check(L.lib().nfb_conv2d_wgrad(L.ptr(xd), cin, 0, L.ptr(gyd), L.ptr(gw), None, B, cin, H, W, cout, k, 0,
                                     L.stream_ptr()))
    err = (gw.double().cpu() - ref).abs()
    print(f"\n[wgrad, 262144 pixels] max err / bound {float((err / bound).max()):.3f}, "
          f"max rel err {float((err / ref.abs().clamp_min(1e-3 * float(ref.abs().max()))).max()):.2e}")
    assert (err <= bound).all(), f"max err {err.max():.3e}"


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["diag", "glow", "glow_cc"])
def test_image_base_gradients_match_torch(kind):
    """DiagGaussian (image shape) and GlowBase with / without classes: g_z and every parameter gradient of log_prob
    against torch autograd in fp64 (GlowBase: tables shared by the pixels of a channel, differentiable _channel_params)."""
    shape, ncls, B = (4, 3, 5), 5, 7
    g = torch.Generator().manual_seed(3)
    q = nf.distributions.DiagGaussian(shape) if kind == "diag" else \
        nf.distributions.GlowBase(shape, num_classes=ncls if kind == "glow_cc" else None)
    with torch.no_grad():
        for p in q.parameters():
            p.copy_(0.2 * torch.randn(p.shape, generator=g))
    z = torch.randn(B, *shape, generator=g, dtype=torch.float64)
    y = torch.randint(ncls, (B,), generator=g)
    w = torch.randn(B, generator=g, dtype=torch.float64)
    ref = _double_params(q)
    with torch.enable_grad():
        zr = z.clone().requires_grad_(True)
        if kind == "diag":
            lq = -0.5 * q.d * np.log(2 * np.pi) - (ref["log_scale"] + 0.5 * ((zr - ref["loc"]) /
                                                   torch.exp(ref["log_scale"])) ** 2).sum((1, 2, 3))
        else:
            loc = ref["loc"] * torch.exp(ref["loc_logs"] * 3.0)
            ls = ref["log_scale"] * torch.exp(ref["log_scale_logs"] * 3.0)
            if kind == "glow_cc":
                loc = loc + ref["loc_cc"][y][:, :, None, None]
                ls = ls + ref["log_scale_cc"][y][:, :, None, None]
            ls = ls.expand(B, *shape)
            lq = -0.5 * q.d * np.log(2 * np.pi) - (ls + 0.5 * ((zr - loc) / torch.exp(ls)) ** 2).sum((1, 2, 3))
        (lq * w).sum().backward()
        qc = q.cuda()
        zc = z.float().cuda().requires_grad_(True)
        out = qc.log_prob(zc) if kind == "diag" else qc.log_prob(zc, y.cuda() if kind == "glow_cc" else None)
        (out * w.float().cuda()).sum().backward()
    np.testing.assert_allclose(out.detach().cpu().double(), lq.detach(), rtol=1e-5)
    _check_grad("z", zc.grad, zr.grad)
    for n, p in qc.named_parameters():
        _check_grad(n, p.grad, ref[n].grad)


def _double_params(module):
    return {n: p.detach().double().clone().requires_grad_(True) for n, p in module.named_parameters()}


DGRAD_CASES = [  # (k, cin, cout, H, W, B, slope, accumulate)
    (3, 12, 64, 8, 8, 3, None, 0), (3, 64, 24, 8, 8, 3, 0.0, 0), (1, 256, 256, 4, 4, 2, 0.1, 1),
    (3, 256, 24, 16, 16, 2, 0.0, 1), (1, 48, 48, 5, 7, 4, None, 0), (3, 32, 32, 8, 8, 2, 0.1, 0),
    (3, 6, 32, 4, 4, 3, None, 1),
]


@pytest.mark.gpu
@pytest.mark.parametrize("k,cin,cout,H,W,B,slope,acc", DGRAD_CASES)
def test_conv_dgrad_matches_torch(k, cin, cout, H, W, B, slope, acc):
    g = torch.Generator().manual_seed(7 * k + cin + 3 * cout)
    w = torch.randn(cout, cin, k, k, generator=g, dtype=torch.float64) / (cin * k * k) ** 0.5
    gy = torch.randn(B, cout, H, W, generator=g, dtype=torch.float64)
    prior = torch.randn(B, cin, H, W, generator=g, dtype=torch.float64)
    act = F.leaky_relu(torch.randn(B, cin, H, W, generator=g, dtype=torch.float64), slope or 0.0)
    ref = torch.nn.grad.conv2d_input((B, cin, H, W), w, gy, padding=k // 2)
    bound = 1e-4 * torch.nn.grad.conv2d_input((B, cin, H, W), w.abs(), gy.abs(), padding=k // 2) + 1e-6
    if slope is not None:
        d = torch.where(act > 0, 1.0, slope).double()
        ref, bound = ref * d, bound * d.abs()
    if acc:
        ref = ref + prior
    gx = prior.float().cuda() if acc else torch.empty(B, cin, H, W, device="cuda")
    mask = act.float().cuda() if slope is not None else None
    gyd, wd = gy.float().cuda(), w.float().cuda()   # kept alive until the kernel has run
    L.check(L.lib().nfb_conv2d_dgrad(L.ptr(gyd), L.ptr(wd), L.ptr(gx), B, cin, H, W, cout, k, L.ptr(mask),
                                     float(slope or 0.0), acc, L.stream_ptr()))
    err = (gx.double().cpu() - ref).abs()
    assert (err <= bound + 1e-6 * ref.abs()).all(), f"dgrad: max err {err.max():.3e}"


def _coupling_ref(z, param, scale, smap, mode):
    C = z.shape[1]
    h = (C + 1) // 2
    a, c = z[:, :h], z[:, h:]
    z1, z2 = (a, c) if mode == "channel" else (c, a)
    if not scale:
        z2, ld = z2 - param, 0 * param.sum((1, 2, 3))
    else:
        shift, sc = param[:, 0::2], param[:, 1::2]
        if smap == "exp":
            z2, ld = (z2 - shift) * torch.exp(-sc), -sc.sum((1, 2, 3))
        else:
            sg = torch.sigmoid(sc + 2)
            if smap == "sigmoid":
                z2, ld = (z2 - shift) * sg, torch.log(sg).sum((1, 2, 3))
            else:
                z2, ld = (z2 - shift) / sg, -torch.log(sg).sum((1, 2, 3))
    return torch.cat([z1, z2] if mode == "channel" else [z2, z1], 1), ld


@pytest.mark.gpu
@pytest.mark.parametrize("scale,smap", [(True, "exp"), (True, "sigmoid"), (True, "sigmoid_inv"), (False, "sigmoid")])
@pytest.mark.parametrize("mode", ["channel", "channel_inv"])
def test_coupling_adjoint_matches_torch(scale, smap, mode):
    from normflows.flows.glow import _MAPS
    g = torch.Generator().manual_seed(5)
    B, C, H, W = 3, 7, 5, 4
    h = (C + 1) // 2
    n2 = C - h if mode == "channel" else h
    o2 = h if mode == "channel" else 0
    z = torch.randn(B, C, H, W, generator=g, dtype=torch.float64).requires_grad_(True)
    param = (0.5 * torch.randn(B, (2 if scale else 1) * n2, H, W, generator=g, dtype=torch.float64)).requires_grad_(True)
    g_out = torch.randn(B, C, H, W, generator=g, dtype=torch.float64)
    g_ld = torch.randn(B, generator=g, dtype=torch.float64)
    with torch.enable_grad():
        out, ld = _coupling_ref(z, param, scale, smap, mode)
        rz, rp = torch.autograd.grad([out, ld], [z, param], [g_out, g_ld])
    gz = torch.zeros(B, C, H, W, device="cuda")
    gp = torch.empty(param.shape, device="cuda")
    dev = [t.detach().float().cuda() for t in (z, param, g_out, g_ld)]   # kept alive until the kernel has run
    L.check(L.lib().nfb_affine_coupling_image_backward(
        *[L.ptr(t) for t in dev], L.ptr(gz), L.ptr(gp), B, C, H * W, int(scale), _MAPS[smap],
        0 if mode == "channel" else 1, L.stream_ptr()))
    np.testing.assert_allclose(gz.cpu().double()[:, o2:o2 + n2], rz[:, o2:o2 + n2], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(gp.cpu().double(), rp, rtol=1e-5, atol=1e-5)


# ---- whole models --------------------------------------------------------------------------------------------------
def build_glow(L_=2, K=2, hidden=32, shape=(3, 8, 8), ncls=10, use_lu=True, net_actnorm=False, transform=None,
               seed=13):
    torch.manual_seed(seed)
    q0, merges, flows = [], [], []
    for i in range(L_):
        flows.append([nf.flows.GlowBlock(shape[0] * 2 ** (L_ + 1 - i), hidden, split_mode="channel", scale=True,
                                         use_lu=use_lu, net_actnorm=net_actnorm) for _ in range(K)]
                     + [nf.flows.Squeeze()])
        if i > 0:
            merges.append(nf.flows.ImageMerge())
            ls = (shape[0] * 2 ** (L_ - i), shape[1] // 2 ** (L_ - i), shape[2] // 2 ** (L_ - i))
        else:
            ls = (shape[0] * 2 ** (L_ + 1), shape[1] // 2 ** L_, shape[2] // 2 ** L_)
        q0.append(nf.distributions.ClassCondDiagGaussian(ls, ncls))
    return nf.MultiscaleFlow(q0, flows, merges, transform=transform)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# gradient goldens (tests/golden/make_glow_grads.py) -> (golden holding the model and inputs, build_glow arguments)
GRAD_CASES = {
    "glow_small": ("glow_small", dict(hidden=32, shape=(3, 8, 8))),           # generic conditioner path
    "glow_width": (None, dict(hidden=64, shape=(3, 16, 16))),                 # Glow-shaped: fused kernel, tap form
    "glow_options": ("options", dict(hidden=16, shape=(3, 8, 8), use_lu=False, net_actnorm=True, logit=True)),
}


def _grad_golden(case):
    """(our model with the golden's weights on the CPU, x, y, gradient golden); digests of weights and inputs checked."""
    import json
    from helpers import check_digests, load_npz_parts, sha256
    g = load_npz_parts(os.path.join(GOLDEN, f"grads_{case}.npz"))
    src, kw = GRAD_CASES[case]
    f = dict(np.load(os.path.join(GOLDEN, src + ".npz"))) if src else g
    sd = {k[4:]: np.asarray(v) for k, v in f.items() if k.startswith("sd__")}
    check_digests(sd, json.loads(str(g["sd_sha256"])), f"grads_{case}")
    x, y = np.asarray(f["x"], dtype=np.float32), np.asarray(f["y"])
    assert sha256(x) == str(g["x_sha256"]) and sha256(y) == str(g["y_sha256"])
    kw = dict(kw)
    model = build_glow(transform=nf.transforms.Logit(0.05) if kw.pop("logit", False) else None, **kw)
    model.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()}, strict=True)
    return model, torch.from_numpy(x), torch.from_numpy(y), g


def test_glow_gradient_goldens_rebuild():
    """CPU: every gradient golden names the weights and inputs it was minted for, and they rebuild bit for bit (C3: the
    recipe of tests/helpers_glow.py); no golden file reaches 1 MB."""
    import glob
    import json
    from helpers import load_npz_parts, sha256
    from helpers_glow import glow_c3_inputs, glow_c3_state_dict
    for case in GRAD_CASES:
        _grad_golden(case)
    g = load_npz_parts(os.path.join(GOLDEN, "grads_glow_c3.npz"))
    sd = glow_c3_state_dict(np.load(os.path.join(GOLDEN, "glow_c3.npz")))
    assert {k: sha256(v) for k, v in sd.items()} == json.loads(str(g["sd_sha256"]))
    x, y = glow_c3_inputs()
    assert sha256(x.numpy()) == str(g["x_sha256"]) and sha256(y.numpy()) == str(g["y_sha256"])
    for fn in glob.glob(os.path.join(GOLDEN, "grads_glow_*.npz")):
        assert os.path.getsize(fn) < 1 << 20, fn


def _check_grad(name, got, ref):
    ref = ref.detach().double()
    got = got.detach().double().cpu()
    scale = float(ref.abs().max()) or 1.0
    err = (got - ref).abs()
    if float(err.max()) <= 2e-3 * scale:
        return
    # LeakyReLU(0) kinks (ReLU): entries whose pre-activation sits near 0 may take the other branch
    frac = float((err <= 2e-3 * scale).double().mean())
    relf = float((got - ref).norm() / (ref.norm() + 1e-30))
    assert frac >= 0.97 and relf <= 1e-2, f"{name}: max err {float(err.max()):.3e} (scale {scale:.3e}), " \
                                          f"{frac:.4f} within, rel Frobenius {relf:.3e}"


def _check_param(name, grad, g):
    """Against a gradient golden: the whole tensor, or its projections G v, u G and norm |G|."""
    from helpers_glow_grads import grad_projections
    assert grad is not None, name
    if "grad__x__0" in g and name == "x":   # stored in pieces along the batch
        pieces = sorted((k for k in g if k.startswith("grad__x__")), key=lambda k: int(k.rsplit("__", 1)[1]))
        _check_grad(name, grad, torch.from_numpy(np.concatenate([g[k] for k in pieces])))
        return
    if "grad__" + name in g:
        _check_grad(name, grad, torch.from_numpy(np.asarray(g["grad__" + name])))
        return
    # An entry of G v or u G sums a whole row / column of G, so one entry moved by a ReLU kink (see _check_grad) moves
    # every entry of the projection: the fraction-of-entries test has no meaning here; the relative Frobenius error does.
    G = grad.detach().double().cpu().reshape(grad.shape[0], -1)
    v, u = grad_projections(name, tuple(grad.shape))
    for what, got, ref in (("G v", G @ v, g["gradv__" + name]), ("u G", u @ G, g["gradu__" + name]),
                           ("|G|", G.norm().reshape(1), np.asarray(g["gnorm__" + name]).reshape(1))):
        ref = torch.from_numpy(np.asarray(ref, dtype=np.float64))
        relf = float((got - ref).norm() / (ref.norm() + 1e-30))
        assert relf <= 1e-2, f"{name} {what}: rel Frobenius {relf:.3e}"


def _check_model_grads(model, x, y, g):
    xc = x.cuda().requires_grad_(True)
    with torch.enable_grad():
        loss = model.forward_kld(xc, y.cuda())
        loss.backward()
    kld = float(g["kld"])
    assert abs(float(loss.detach()) - kld) <= 2e-5 * abs(kld), (float(loss.detach()), kld)
    _check_param("x", xc.grad, g)
    for n, p in model.named_parameters():
        _check_param(n, p.grad, g)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(GRAD_CASES))
def test_glow_gradients_match_reference(case):
    """forward_kld and every gradient against the reference's fp64 autograd."""
    model, x, y, g = _grad_golden(case)
    _check_model_grads(model.cuda(), x, y, g)


@pytest.mark.gpu
def test_glow_c3_gradients_match_reference():
    """BASELINE config 3 at its real shape (48 blocks, 8 M parameters; the model and 64 images of glow_c3.npz): the
    wgrad kernel runs its longest pixel splits here.  Large tensors are checked through seeded projections and norms."""
    from helpers import load_npz_parts
    from helpers_glow import build_glow_c3, glow_c3_inputs, glow_c3_state_dict
    g = load_npz_parts(os.path.join(GOLDEN, "grads_glow_c3.npz"))
    sd = glow_c3_state_dict(np.load(os.path.join(GOLDEN, "glow_c3.npz")))
    model = build_glow_c3()
    model.load_state_dict({k: torch.from_numpy(v).float() if v.dtype.kind == "f" else torch.from_numpy(v)
                           for k, v in sd.items()}, strict=True)
    x, y = glow_c3_inputs()
    _check_model_grads(model.cuda(), x, y, g)


@pytest.mark.gpu
def test_log_prob_values_identical_with_and_without_grad():
    torch.manual_seed(0)
    x = torch.rand(16, 3, 16, 16, generator=torch.Generator().manual_seed(3)).cuda()
    y = torch.randint(10, (16,), generator=torch.Generator().manual_seed(4)).cuda()
    a, b = build_glow(hidden=64, shape=(3, 16, 16)).cuda(), build_glow(hidden=64, shape=(3, 16, 16)).cuda()
    with torch.enable_grad():
        la = a.log_prob(x, y)            # first call under grad: ActNorm init inside the autograd path
    assert la.requires_grad
    with torch.no_grad():
        lb = b.log_prob(x, y)
    assert torch.equal(la.detach(), lb)
    for (n, p), (_, q) in zip(a.state_dict().items(), b.state_dict().items()):
        assert torch.equal(p, q), n
    with torch.enable_grad():
        la2 = a.log_prob(x, y)
    with torch.no_grad():
        lb2 = a.log_prob(x, y)
    assert torch.equal(la2.detach(), lb2)


def _oracle_spec(model):
    levels = []
    for fl in model.flows:
        lv = []
        for f in fl:
            if isinstance(f, nf.flows.Squeeze):
                lv.append({"type": "Squeeze"})
            else:
                lv.append({"type": "GlowBlock", "channels": f.channels})
        levels.append(lv)
    return {"kind": "MultiscaleFlow", "levels": levels, "class_cond": True}


def _synthetic_images(n, g):
    """Seeded structured images in [0, 1]: a class-dependent oriented stripe pattern, a smooth blob and a little noise."""
    y = torch.randint(10, (n,), generator=g)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, 16), torch.linspace(0, 1, 16), indexing="ij")
    ang = y.float()[:, None, None] * (np.pi / 10)
    stripes = torch.sin(12 * (torch.cos(ang) * xx + torch.sin(ang) * yy))
    cx, cy = torch.rand(n, 1, 1, generator=g), torch.rand(n, 1, 1, generator=g)
    blob = torch.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 0.05)
    col = torch.rand(n, 3, 1, 1, generator=g)
    img = 0.5 + 0.2 * stripes[:, None] * col + 0.25 * blob[:, None] + 0.03 * torch.randn(n, 3, 16, 16, generator=g)
    return img.clamp(0, 1), y


@pytest.mark.gpu
def test_training_loop_of_the_notebook():
    """examples/glow.ipynb cell 4 (Adamax, lr 1e-3, weight decay 1e-5) on a Glow-shaped model; afterwards the packed
    weights must have followed every step: log_prob against the fp64 oracle."""
    from oracle import nf_oracle as O
    model = build_glow(hidden=64, shape=(3, 16, 16)).cuda()
    optimizer = torch.optim.Adamax(model.parameters(), lr=1e-3, weight_decay=1e-5)
    g = torch.Generator().manual_seed(21)
    losses = []
    with torch.enable_grad():
        for it in range(300):
            x, y = _synthetic_images(64, g)
            optimizer.zero_grad()
            loss = model.forward_kld(x.cuda(), y.cuda())
            assert torch.isfinite(loss)
            loss.backward()
            optimizer.step()
            losses.append(float(loss.detach()))
    first, last = np.mean(losses[:5]), np.mean(losses[-20:])
    print(f"\n[glow training] loss {first:.1f} -> {last:.1f} (per image, 768 dims)")
    assert last < first - 0.05 * abs(first), (first, last)
    x, y = _synthetic_images(32, g)
    with torch.no_grad():
        lp = model.log_prob(x.cuda(), y.cuda()).cpu().numpy()
    sd = {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}
    ref = O.log_prob(_oracle_spec(model), sd, x.numpy().astype(np.float64), y.numpy())
    np.testing.assert_allclose(lp, ref, rtol=1e-4)
