"""Stage-by-stage GPU bring-up diagnostics (not a test; prints numbers).  usage: gpu_debug.py <mode>"""
import os, sys, time, traceback
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200"), os.path.join(ROOT, "tests")]
import numpy as np
import torch
torch.set_grad_enabled(False)  # debug runs compare raw outputs; the autograd hook would tag them
import normflows as nf
from normflows.flows.base import NativeFlow
from conftest import load_golden
from helpers import annotate_spec, build_model
from oracle import nf_oracle as O

mode = sys.argv[1] if len(sys.argv) > 1 else "generic"
cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
CASES = ["nsf_ar_d2_h32_l2_k4", "nsf_coupled_d2_h32_l2_k4", "nsf_ar_d5_h128_l3", "nsf_coupled_d5_h128_l3",
         "nsf_ar_d64_h256_l2", "nsf_coupled_d64_h256_l2", "realnvp2d", "affine_block2d", "affine_block6d"]


def report(tag, got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    d = np.abs(got - ref)
    print(f"  {tag:34s} max_abs={np.nanmax(d):.3e} max_rel={np.nanmax(d / (np.abs(ref) + 1e-3)):.3e} "
          f"nan={int(np.isnan(got).sum())}", flush=True)


def per_layer(model, a, n):
    for i in range(n - 1, -1, -1):
        zin = a["x"] if i == n - 1 else a[f"zl_f64__{i + 1}"]
        z, ld = model.flows[i].inverse(cuda(zin))
        torch.cuda.synchronize()
        report(f"layer {i} z ({type(model.flows[i]).__name__[:12]})", z.cpu().numpy(), a[f"zl_f64__{i}"])
        report(f"layer {i} log_det", ld.cpu().numpy(), a[f"ld_f64__{i}"])


def run_cases(use_tc, cases):
    NativeFlow.use_tensor_cores = use_tc
    for name in cases:
        print(f"== {name} use_tc={use_tc}", flush=True)
        try:
            spec, sd, a = load_golden(name)
            model = build_model(annotate_spec(spec, sd), sd).cuda()
            per_layer(model, a, len(model.flows))
            lp = model.log_prob(cuda(a["x"]))
            torch.cuda.synchronize()
            print("  fused layers:", model._stack().fused_layers(), "launches:", model._stack().launch_count())
            report("log_prob (stack)", lp.cpu().numpy(), a["log_prob_f64"])
            print("  kld", float(model.forward_kld(cuda(a["x"]))), "ref", float(a["kld_f64"]))
            if "fwd_x_f64" in a:
                xr, ld = model.forward_and_log_det(cuda(a["z_f64"]))
                report("sampling x", xr.cpu().numpy(), a["fwd_x_f64"])
                report("sampling log_det", ld.cpu().numpy(), a["fwd_ld_f64"])
        except Exception:
            traceback.print_exc()
            print("  !! failed", flush=True)


def rand_model(kind, layers, d=64, hidden=256):
    torch.manual_seed(0)
    fl = []
    for i in range(layers):
        fl.append(nf.flows.AutoregressiveRationalQuadraticSpline(d, 2, hidden) if kind == "ar"
                  else nf.flows.CoupledRationalQuadraticSpline(d, 2, hidden, reverse_mask=bool(i % 2)))
        fl.append(nf.flows.LULinearPermute(d))
    m = nf.NormalizingFlow(nf.distributions.DiagGaussian(d, trainable=False), fl)
    with torch.no_grad():
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    return m.cuda()


def timeit(fn, n=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(n + 1)]
    ev[0].record()
    for i in range(n):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return sorted(ev[i].elapsed_time(ev[i + 1]) for i in range(n))[n // 2]


if mode == "generic":
    run_cases(False, CASES)
elif mode == "fused":
    run_cases(True, ["nsf_ar_d64_h256_l2", "nsf_coupled_d64_h256_l2", "nsf_ar_d5_h128_l3"])
elif mode == "time":
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
    layers = int(sys.argv[3]) if len(sys.argv) > 3 else 32
    for kind in ("ar", "coupled"):
        m = rand_model(kind, layers)
        x = (torch.randn(B, 64) * 1.5).cuda()
        for tc in (True, False):
            NativeFlow.use_tensor_cores = tc
            try:
                ms = timeit(lambda: m.forward_kld(x), n=5 if tc else 2, warm=2 if tc else 1)
                print(f"time {kind} B={B} L={layers} use_tc={tc}: {ms:.2f} ms/pass  {B / ms * 1e3:.3e} samples/s "
                      f"launches={m._stack().launch_count()}", flush=True)
            except Exception:
                traceback.print_exc()
print("done", mode, flush=True)

if mode == "spline":
    import ctypes as C
    from normflows import _lib as L
    B, T, K = 65536, 64, 8
    P = 3 * K - 1
    x = (torch.randn(B, T) * 1.5).cuda()
    params = [torch.randn(B, T * P, device="cuda") for _ in range(2)]  # 2 x 386 MB > L2
    y = torch.empty_like(x)
    ld = torch.zeros(B, device="cuda")
    lib = L.lib()
    for inv in (0, 1):
        def run(i=[0]):
            i[0] += 1
            L.check(lib.nfb_rqs_spline(L.ptr(x), L.ptr(params[i[0] % 2]), L.ptr(y), L.ptr(ld), B, T, K,
                                       C.c_float(3.0), C.c_float(1.0), inv, 1, None))
        ms = timeit(run, n=11, warm=3)
        byt = B * T * (P * 4 + 8) + B * 8
        print(f"spline standalone inverse={inv}: {ms*1e3:.1f} us  {byt/ms/1e6:.1f} GB/s  "
              f"of the H100 SXM data sheet's 3350 = {byt/ms/1e6/3350:.3f}", flush=True)

if mode == "stackdbg":
    spec, sd, a = load_golden("nsf_ar_d64_h256_l2")
    model = build_model(spec, sd).cuda()
    for B in (48, 1, 47):
        x = cuda(a["x"][:B])
        z, ld = model.inverse_and_log_det(x)
        ez = np.abs(z.cpu().numpy() - a["z_f64"][:B])
        eld = np.abs(ld.cpu().numpy() - (a["log_prob_f64"][:B] * 0 + sum(a[f"ld_f64__{i}"][:B] for i in range(4))))
        bad = np.argwhere(ez > 1e-3)
        print(f"B={B}: z max err {ez.max():.3e} ld max err {eld.max():.3e} bad elems {len(bad)} rows {sorted(set(bad[:,0]))[:10]} cols {sorted(set(bad[:,1]))[:20]}", flush=True)
    # repeat several times to see nondeterminism
    x = cuda(a["x"])
    outs = [model.inverse_and_log_det(x)[0].cpu().numpy() for _ in range(5)]
    print("run-to-run max diff:", max(np.abs(o - outs[0]).max() for o in outs))
    # larger batch: compare stack vs oracle on first rows
    xb = np.tile(a["x"], (40, 1))[:1500]
    z, ld = model.inverse_and_log_det(cuda(xb))
    ref = np.tile(a["z_f64"], (40, 1))[:1500]
    ez = np.abs(z.cpu().numpy() - ref).max(axis=1)
    badr = np.argwhere(ez > 1e-3)[:, 0]
    rng_, st = [], None
    for r_ in badr:
        if st is None: st = prev = r_
        elif r_ != prev + 1: rng_.append((st, prev)); st = r_
        prev = r_
    if st is not None: rng_.append((st, prev))
    print("B=1500: bad row ranges:", rng_, "max", ez.max())
    em = np.abs(z.cpu().numpy() - ref)
    for (a0, a1) in rng_[:3]:
        cols = sorted(set(np.argwhere(em[a0:a1 + 1] > 1e-3)[:, 1].tolist()))
        print(f"   rows {a0}-{a1}: {len(cols)} bad cols: {cols}")
        print("   ld err there:", np.abs(ld.cpu().numpy()[a0:a0 + 3] - np.tile(sum(a[f'ld_f64__{i}'] for i in range(4)), 40)[:1500][a0:a0 + 3]))
    for L_ in (1, 3):
        zz = cuda(xb)
        for i in range(L_, -1, -1):
            zz, _ = model.flows[i].inverse(zz)
        if L_ == 3:
            print("per-layer path max err", np.abs(zz.cpu().numpy() - ref).max())

if mode == "bias":
    # signed error of log_prob against the fp64 oracle on the rough test model: is the fused path biased?
    sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tests"))
    from test_gpu_parity import _random_model, _oracle_of
    for kind in ("ar", "coupled"):
        model = _random_model(kind, 64, 4, 256).cuda()
        spec, sd = _oracle_of(model, kind, 64, 4, 256)
        x = torch.randn(3000, 64, generator=torch.Generator().manual_seed(1234)) * 1.5
        ref = O.log_prob(spec, sd, x.numpy().astype(np.float64))
        for tc in (True, False):
            NativeFlow.use_tensor_cores = tc
            lp = model.log_prob(x.cuda()).cpu().numpy().astype(np.float64)
            e = lp - ref
            rel = np.abs(e) / np.abs(ref)
            print(f"bias {kind} tc={tc} comp={os.environ.get('NFB_ACC_COMP_STEP','default')}: mean signed {e.mean():+.3e} median {np.median(e):+.3e} "
                  f"rms {np.sqrt((e**2).mean()):.3e} | rel mean {rel.mean():.2e} p99 {np.quantile(rel,0.99):.2e} max {rel.max():.2e}", flush=True)
        NativeFlow.use_tensor_cores = True

if mode == "timefwd":
    # sampling direction (forward_and_log_det) of the coupled 32-layer stack: fused whole-stack launch vs generic kernels
    B = int(sys.argv[2]) if len(sys.argv) > 2 else 65536
    m = rand_model("coupled", 32)
    z = torch.randn(B, 64).cuda()
    for tc in (True, False):
        NativeFlow.use_tensor_cores = tc
        ms = timeit(lambda: m.forward_and_log_det(z), n=5 if tc else 2, warm=2 if tc else 1)
        print(f"timefwd coupled B={B} L=32 use_tc={tc}: {ms:.2f} ms/pass  {B / ms * 1e3:.3e} samples/s "
              f"launches={m._stack().launch_count()}", flush=True)
    NativeFlow.use_tensor_cores = True
