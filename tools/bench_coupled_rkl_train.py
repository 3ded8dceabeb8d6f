"""Time reverse-KL training of coupling spline flows: one step (`reverse_kld` + `backward()` + Adam), or a no-grad draw.
    w4096       tests/helpers_coupled_rkl.py case w: 4 x [CoupledRationalQuadraticSpline(6, 2, 64), LULinearPermute(6)]
                on DiagGaussian(6), its 6-D target, reverse_kld(4 096)
    coupled64   16 x [CoupledRationalQuadraticSpline(64, 2, 256, reverse_mask=i % 2), LULinearPermute(64)] on
                DiagGaussian(64), a 64-D Gaussian-chain target, reverse_kld at 4 096 and at 65 536 rows
    sample      the no-grad `sample(65 536)` of the coupled64 model (the forward the training step starts from)
Adam(lr 1e-4).  Prints one JSON line: ms/step (median of CUDA-event-timed steps after warm-up), kernel launches per step
(torch.profiler, one separate step), peak device memory, and the card's name, power limit and SM clock read in the same
run.  When the unmodified reference is installed under oracle/_ref, the same model, seed and batch are timed through it
(eager torch, fp32).
    python tools/bench_coupled_rkl_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases w4096,coupled64]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench_conditional_train import gpu_info  # noqa: E402

CASES = [("w4096", "w4096", 4096), ("coupled64", "coupled64", 4096), ("coupled64_65536", "coupled64", 65536),
         ("sample", "coupled64", 65536)]


def build(nf, kind):
    import torch
    import helpers_coupled_rkl as H
    if kind == "w4096":
        return H.build(nf, "w")
    torch.manual_seed(0)
    flows = []
    for i in range(16):
        flows += [nf.flows.CoupledRationalQuadraticSpline(64, 2, 256, reverse_mask=bool(i % 2)),
                  nf.flows.LULinearPermute(64)]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(64), flows, H.Target64())


def time_arm(arm, name, kind, batch, steps, warmup):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    model = build(nf, kind).cuda()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    torch.manual_seed(0)

    def step():
        if name == "sample":
            with torch.no_grad():
                return model.sample(batch)[1].mean()
        opt.zero_grad(set_to_none=True)
        loss = model.reverse_kld(batch)
        loss.backward()
        opt.step()
        return loss

    for _ in range(warmup):
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
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    times.sort()
    ms = times[len(times) // 2]
    return {"case": name, "batch": batch, "ms_per_step": round(ms, 3), "ms_min": round(times[0], 3),
            "ms_max": round(times[-1], 3), "launches_per_step": launches, "peak_mem_gb": round(peak / 2 ** 30, 3),
            "loss": round(float(loss), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated case names (default: all)")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    want = set(a.cases.split(",")) if a.cases else None
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        print(json.dumps([time_arm(a.arm, n, k, b, a.steps, a.warmup) for n, k, b in CASES
                          if want is None or n in want]))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_coupled_rkl_train: no CUDA device")
    arms = ["native"] + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
                         else [])
    res = {}
    for arm in arms:
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps", str(a.steps), "--warmup", str(a.warmup)]
        if a.cases:
            cmd += ["--cases", a.cases]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            res[arm] = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}
        else:
            res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps({"metric": "coupled_rkl_train_step", **gpu_info(), **res}))


if __name__ == "__main__":
    main()
