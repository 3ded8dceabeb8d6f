"""Time HAIS and a stochastic-normalizing-flow training step (flows/stochastic.py, sampling/hais.py,
csrc/nfb_stochastic.cu).
    hais_d<D>_b<B>  HAIS(linspace(1, 0, B), DiagGaussian(D), GaussianMixture(8, D), 10 leapfrog steps).sample(65 536)
                    under torch.no_grad(), for D in {2, 16, 64} and B in {100, 1000}: ms per call, launches per call
                    (torch.profiler, CUDA kernels), FLOPs per call from the shapes and the achieved rate against the
                    H100 SXM data-sheet FP32 peak (67 TFLOP/s)
    snf_step        NormalizingFlow(DiagGaussian(16), [MaskedAffineFlow, ActNorm, HamiltonianMonteCarlo(GaussianMixture(8,
                    16), 10)] x 2): reverse_kld(8 192) + backward + Adam
The card's name, power limit and clocks are read in the same run.  When the unmodified reference is installed under
oracle/_ref, the same cases are timed through it (eager torch, float32) -- the HAIS cases at 100 betas only: at 1 000
betas a reference call is tens of thousands of autograd calls.
    python tools/bench_stochastic.py [--steps 5] [--warmup 1] [--no-reference] [--cases hais_d2_b100,snf_step]
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

ROWS, K, LEAPFROG = 65536, 8, 10
PEAK_F32 = 67e12
CASES = [f"hais_d{d}_b{b}" for b in (100, 1000) for d in (2, 16, 64)] + ["snf_step"]


def hais_flops(rows, D, betas):
    """Per transition and row: L + 1 evaluations of log p and grad log p of the interpolation (the target's K modes and
    the prior's one: per (mode, feature) 10 FLOPs for the two quadratic passes, 4 for the gradient), and L leapfrog
    updates (10 FLOPs per feature with the momentum draw and the kinetic energies)."""
    T = betas - 2
    return T * rows * ((LEAPFROG + 1) * 14 * D * (K + 1) + LEAPFROG * 10 * D)


def build_hais(nf, D, betas):
    import numpy as np
    import torch
    torch.manual_seed(0)
    loc = np.random.default_rng(0).normal(0, 1.5, (K, D))
    gm = nf.distributions.GaussianMixture(K, D, loc=loc).float().cuda()
    prior = nf.distributions.DiagGaussian(D, trainable=False).cuda()
    return nf.HAIS(torch.linspace(1, 0, betas), prior, gm, LEAPFROG, torch.full((D,), 0.3 / D ** 0.5, device="cuda"),
                   torch.zeros(D, device="cuda"))


def build_snf(nf, D=16):
    import torch
    torch.manual_seed(0)
    gm = nf.distributions.GaussianMixture(K, D).float().cuda()
    flows = []
    for i in range(2):
        b = torch.tensor([(j + i) % 2 for j in range(D)], dtype=torch.float32)
        flows += [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([D, 64, D], init_zeros=True),
                                            nf.nets.MLP([D, 64, D], init_zeros=True)), nf.flows.ActNorm(D),
                  nf.flows.HamiltonianMonteCarlo(gm, LEAPFROG, torch.full((D,), -2.0), torch.zeros(D))]
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows, p=gm).cuda()
    for p in gm.parameters():
        p.requires_grad_(False)
    with torch.enable_grad():   # ActNorm's data-dependent initialisation (the reference's HMC needs grad mode)
        model.reverse_kld(8192)
    return model


def time_case(arm, case, steps, warmup):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    if case.startswith("hais"):
        D, betas = (int(s[1:]) for s in case.split("_")[1:])
        h = build_hais(nf, D, betas)
        grad_ctx = torch.enable_grad if arm == "reference" else torch.no_grad   # the reference needs grad mode

        def step():
            with grad_ctx():
                return h.sample(ROWS)[1]
        flops = hais_flops(ROWS, D, betas)
    else:
        model = build_snf(nf)
        opt = torch.optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
        flops = None

        def step():
            with torch.enable_grad():
                opt.zero_grad()
                loss = model.reverse_kld(8192)
                loss.backward()
                opt.step()
            return loss
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    times.sort()
    ms = times[len(times) // 2]
    res = {"ms_per_call": round(ms, 3), "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3),
           "launches_per_call": launches, "finite": bool(torch.isfinite(out).all())}
    if flops is not None:
        res.update(flops_per_call=flops, tflops=round(flops / (ms * 1e-3) / 1e12, 3),
                   fp32_peak_share=round(flops / (ms * 1e-3) / PEAK_F32, 4))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated case names (default: all)")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    ap.add_argument("--case", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm and case in its own process (the two packages share the name `normflows`)
        print(json.dumps(time_case(a.arm, a.case, a.steps, a.warmup)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_stochastic: no CUDA device")
    has_ref = not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
    want = set(a.cases.split(",")) if a.cases else None
    for case in CASES:
        if want is not None and case not in want:
            continue
        res = {}
        for arm in ["native"] + (["reference"] if has_ref and not case.endswith("b1000") else []):
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--case", case, "--steps", str(a.steps),
                   "--warmup", str(a.warmup)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode:
                res[arm] = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}
            else:
                res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
        print(json.dumps({"metric": "stochastic", "case": case, **gpu_info(), **res}), flush=True)


if __name__ == "__main__":
    main()
