"""Time training on a Gaussian-mixture base (distributions/base.py GaussianMixture, csrc/nfb_mixture.cu).
    cbd512     examples/change_base_distribution.ipynb's second model (32 x [AffineCouplingBlock(MLP([1, 64, 64, 2])),
               Permute(2, 'swap')] on GaussianMixture(2, 2)): forward_kld + backward + Adam(lr 5e-4, wd 1e-5), batch 512
    cbd65536   the same step at 65 536 rows
    nsf64mix   the BASELINE config-2 model (bench.build_model("ar"): 32 x [autoregressive RQ-NSF d=64 h=256,
               LULinearPermute]) on a trainable GaussianMixture(8, 64): forward_kld + backward + Adam(lr 1e-4), 8 192 rows
    nsf64diag  the same model on a trainable DiagGaussian(64)
    kernel     the stand-alone log_prob and its backward at K = 64, D = 64, 65 536 rows: CUDA-event kernel time of each,
               bytes and FLOPs from the shapes, and the share of the H100 SXM data-sheet peak (3.35 TB/s HBM3, 67 TFLOP/s
               FP32) with the bound that sets it
Each step case prints ms/step (median of CUDA-event-timed steps after warm-up) and peak device memory.  The card's name
and power limit are read in the same run.  When the unmodified reference is installed under oracle/_ref, the same model,
seed and batch are timed through it (eager torch; its mixture holds float64 parameters, as the reference builds them).
    python tools/bench_mixture_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases cbd512,kernel]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_conditional_train import gpu_info  # noqa: E402

CASES = [("cbd512", 512), ("cbd65536", 65536), ("nsf64mix", 8192), ("nsf64diag", 8192), ("kernel", 65536)]
PEAK_BW, PEAK_F32 = 3.35e12, 67e12
KK, KD = 64, 64
# arithmetic per (row, mode, feature) element: the density forms t = (z - mu) inv and ls + t^2 / 2 and accumulates it
# (5 FLOPs); the backward recomputes that twice (log p, then each mode tile's responsibilities), then g_z (4) and the
# two parameter sums (7)
FLOP_FWD, FLOP_BWD = 5, 21


def build(nf, kind):
    """-> (model, (lr, weight decay))"""
    import numpy as np
    import torch
    torch.manual_seed(0)
    np.random.seed(0)
    if kind.startswith("cbd"):
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import helpers_mixture
        return helpers_mixture.cbd(nf), (5e-4, 1e-5)
    sys.path.insert(0, ROOT)
    import bench
    model = bench.build_model("ar")   # (uses whichever `normflows` is imported: same layers, same seed)
    model.q0 = nf.distributions.GaussianMixture(8, bench.D) if kind == "nsf64mix" else \
        nf.distributions.DiagGaussian(bench.D)
    return model, (1e-4, 0.0)


def _median(times):
    times = sorted(times)
    return times[len(times) // 2], times[0], times[-1]


def time_step(nf, kind, batch, steps, warmup):
    import torch
    model, (lr, wd) = build(nf, kind)
    model = model.cuda()
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=wd)
    torch.manual_seed(1)
    if kind.startswith("cbd"):
        xs = [nf.distributions.TwoMoons().sample(batch).float().cuda() for _ in range(4)]
    else:
        xs = [1.5 * torch.randn(batch, model.q0.loc.shape[-1], device="cuda") for _ in range(4)]

    def step(i):
        opt.zero_grad(set_to_none=True)
        loss = model.forward_kld(xs[i % len(xs)])
        loss.backward()
        opt.step()
        return loss

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for i in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss = step(i)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    ms, lo, hi = _median(times)
    return {"model": kind, "batch": batch, "ms_per_step": round(ms, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3),
            "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 3), "loss": round(float(loss), 4)}


def time_kernel(nf, arm, rows, steps, warmup):
    import torch
    torch.manual_seed(0)
    q = nf.distributions.GaussianMixture(KK, KD).cuda()
    z = 1.5 * torch.randn(rows, KD, device="cuda")
    g = torch.randn(rows, device="cuda")
    zz = z.clone().requires_grad_(True)

    def fwd():
        with torch.no_grad():
            return q.log_prob(z)

    lp = q.log_prob(zz)

    def bwd():
        zz.grad = None
        for p in q.parameters():
            p.grad = None
        lp.backward(g, retain_graph=True)

    out = {"model": "kernel", "rows": rows, "n_modes": KK, "dim": KD}
    for name, fn, flop in (("log_prob", fwd, FLOP_FWD), ("backward", bwd, FLOP_BWD)):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        reps = max(steps, 20)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        sec = a.elapsed_time(b) / reps / 1e3
        params = 2 * KK * KD + KK
        # bytes the operation has to move: z (and g_z, g_log_q for the backward), log_q, the parameters (and grads)
        nbytes = 4 * (rows * KD + rows + params) if name == "log_prob" else 4 * (2 * rows * KD + rows + 2 * params)
        flops = flop * rows * KK * KD
        t_bw, t_f = nbytes / PEAK_BW, flops / PEAK_F32
        out[name] = {"ms": round(sec * 1e3, 4), "bytes": nbytes, "flops": flops,
                     "gbytes_per_s": round(nbytes / sec / 1e9, 1), "tflops": round(flops / sec / 1e12, 2)}
        if arm == "native":
            out[name].update({"share_of_peak": round(max(t_bw, t_f) / sec, 3),
                              "bound": "fp32 compute" if t_f > t_bw else "hbm bandwidth"})
    return out


def run_arm(arm, cases, steps, warmup):
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    return [time_kernel(nf, arm, b, steps, warmup) if k == "kernel" else time_step(nf, k, b, steps, warmup)
            for k, b in cases]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated case names (default: all)")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    want = set(a.cases.split(",")) if a.cases else None
    cases = [(k, b) for k, b in CASES if want is None or k in want]
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        print(json.dumps(run_arm(a.arm, cases, a.steps, a.warmup)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixture_train: no CUDA device")
    arms = ["native"] + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
                         else [])
    info = gpu_info()
    res = {}
    for arm in arms:
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps", str(a.steps), "--warmup", str(a.warmup)]
        if a.cases:
            cmd += ["--cases", a.cases]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            res[arm] = [{"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}]
        else:
            res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
    for i, (k, _) in enumerate(cases):
        line = {"metric": "gaussian_mixture", "case": k, **info}
        for arm in arms:
            row = res[arm][i] if len(res[arm]) > i else res[arm][0]
            line[arm] = row
        print(json.dumps(line))


if __name__ == "__main__":
    main()
