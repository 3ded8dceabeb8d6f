"""Time training steps of Real NVP models on the affine family's wide path (DESIGN §3.13): forward, backward and Adam.
    vae_realnvp40     examples/vae.ipynb with flow_type 'RealNVP' (40 features, 40 MaskedAffineFlows with MLP([40, 40])
                      s / t nets), batch 64 x num_samples 32; the flows' parameters scaled by 0.05 after the notebook's
                      default initialisation, which overflows exp(s) in the first forward (in the reference as well)
    rnvp64_fkl_512    8 x [MaskedAffineFlow(alternating b, MLP([64, 256, 256, 64]) for s and t), ActNorm(64)],
                      forward_kld on 512 rows of a seeded correlated Gaussian
    rnvp64_fkl_65536  the same at 65 536 rows
    rnvp64_rkl_4096   the same model, reverse_kld(4 096) against an 8-mode 64-D GaussianMixture target
Prints one JSON line per case: ms/step (median and range of CUDA-event-timed steps after warm-up), kernel launches per
step (torch.profiler, one separate step), peak device memory, the first and last step's loss, and the card's name and
power limit read in the same run.  When the unmodified reference is installed under oracle/_ref, the same model, seed and
data are timed through it (eager torch, fp32).
    python tools/bench_affine_wide_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases rnvp64_fkl_512,...]
    python tools/bench_affine_wide_train.py --trace DIR --cases rnvp64_fkl_65536   (a torch.profiler trace of one step)
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

CASES = {"vae_realnvp40": 64, "rnvp64_fkl_512": 512, "rnvp64_fkl_65536": 65536, "rnvp64_rkl_4096": 4096}
D = 64


def rnvp64(nf, target=None):
    import torch
    b = torch.tensor([float(j % 2) for j in range(D)])
    flows = []
    for i in range(8):
        s, t = nf.nets.MLP([D, 256, 256, D]), nf.nets.MLP([D, 256, 256, D])
        flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(D)]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(D), flows, p=target)


def build(nf, kind):
    import numpy as np
    import torch
    torch.manual_seed(0)
    if kind == "vae_realnvp40":
        n = 40
        prior = torch.distributions.MultivariateNormal(torch.zeros(n, device="cuda"), torch.eye(n, device="cuda"))
        encoder = nf.distributions.NNDiagGaussian(nf.nets.MLP(np.array([28 ** 2, 512, 256, n * 2])))
        decoder = nf.distributions.NNBernoulliDecoder(nf.nets.MLP(np.array([n, 256, 512, 28 ** 2])))
        b = torch.tensor(n // 2 * [0, 1] + n % 2 * [0])
        flows = []
        for i in range(40):
            s, t = nf.nets.MLP([n, n]), nf.nets.MLP([n, n])
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
        with torch.no_grad():
            for f in flows:
                for p in f.parameters():
                    p.mul_(0.05)
        return nf.NormalizingFlowVAE(prior, encoder, flows, decoder).cuda()
    target = None
    if kind.startswith("rnvp64_rkl"):
        g = torch.Generator().manual_seed(3)
        target = nf.distributions.GaussianMixture(8, D, loc=(2 * torch.randn(8, D, generator=g)).numpy(),
                                                  scale=np.ones((8, D)), trainable=False)
    model = rnvp64(nf, target).cuda()
    x = torch.randn(4096, D, generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():   # ActNorm's data-dependent initialisation on a first batch, in both packages
        model.log_prob(x)
    return model


def batches(kind, rows, n):
    import torch
    g = torch.Generator().manual_seed(1)
    if kind == "vae_realnvp40":
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from bench_vae_train import data
        return data(rows, n)
    A = torch.randn(D, D, generator=g) * 0.3
    return [(torch.randn(rows, D, generator=g) @ A + 1.0).cuda() for _ in range(n)]


def time_arm(arm, kind, steps, warmup, trace=None):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    rows = CASES[kind]
    model = build(nf, kind)
    n = warmup + steps + 2
    xs = batches(kind, rows, n) if not kind.startswith("rnvp64_rkl") else None
    opt = torch.optim.Adam(model.parameters(), lr=1e-4, weight_decay=1e-5)
    torch.manual_seed(0)
    it = iter(range(n))

    def step():
        i = next(it)
        opt.zero_grad()
        if kind == "vae_realnvp40":
            z, log_q, log_p = model(xs[i], 32)
            loss = torch.mean(log_q) - torch.mean(log_p)
        elif xs is None:
            loss = model.reverse_kld(rows)
        else:
            loss = model.forward_kld(xs[i])
        loss.backward()
        opt.step()
        return loss

    first = float(step())
    for _ in range(warmup - 1):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss = step()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    peak = torch.cuda.max_memory_allocated()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    launches = sum(1 for e in ev if "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    out = {"model": kind, "rows": rows * (32 if kind == "vae_realnvp40" else 1)}
    if trace:
        os.makedirs(trace, exist_ok=True)
        prof.export_chrome_trace(os.path.join(trace, f"{kind}_{arm}.json"))
        by = {}
        for e in ev:
            k = e.name[:60]
            by[k] = by.get(k, 0.0) + e.device_time_total / 1e3
        out["top_kernels_ms"] = {k: round(v, 3) for k, v in sorted(by.items(), key=lambda kv: -kv[1])[:8]}
    times.sort()
    out.update({"ms_per_step": round(times[len(times) // 2], 3), "ms_min": round(times[0], 3),
                "ms_max": round(times[-1], 3), "launches_per_step": launches, "peak_mem_gb": round(peak / 2 ** 30, 3),
                "first_loss": round(first, 4), "loss": round(float(loss), 4)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated case names (default: all)")
    ap.add_argument("--trace", help="directory for a torch.profiler trace of one step per arm")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    ap.add_argument("--case", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm and case in its own process (the two packages share the name `normflows`)
        print(json.dumps(time_arm(a.arm, a.case, a.steps, a.warmup, a.trace)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_affine_wide_train: no CUDA device")
    arms = ["native"] + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
                         else [])
    want = set(a.cases.split(",")) if a.cases else None
    info = gpu_info()
    for kind in CASES:
        if want is not None and kind not in want:
            continue
        res = {}
        for arm in arms:
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--case", kind, "--steps", str(a.steps),
                   "--warmup", str(a.warmup)] + (["--trace", a.trace] if a.trace else [])
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode:
                res[arm] = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}
            else:
                res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
        print(json.dumps({"metric": "affine_wide_train_step", "case": kind, **info, **res}), flush=True)


if __name__ == "__main__":
    main()
