"""Time planar and radial flows: one reverse-KL training step (`reverse_kld` + `backward()` + Adam), or a no-grad draw.
    planar16   examples/planar.ipynb: 16 x Planar((2,)) on DiagGaussian(2), TwoModes(2, 0.1), reverse_kld(40, beta=0.5),
               Adam(lr 1e-3, weight decay 1e-4)
    planar32   examples/comparison_plan_rad_aff.ipynb: 32 x Planar((2,)), TwoModes(2.0, 0.2), batch 1 024,
               Adam(lr 1e-3, weight decay 1e-3)
    radial32   the same with Radial((2,))
    sample32   the no-grad `sample(2**20)` of the planar32 model
    vae40      40 x Planar((40,)) on DiagGaussian(40) at 2 048 rows (examples/vae.ipynb's latent size and depth), a 40-D
               standard normal target, the planar16 step
Prints one JSON line: ms/step (median of CUDA-event-timed steps after warm-up), kernel launches per step (torch.profiler,
one separate step), peak device memory, and the card's name and power limit read in the same run.  When the unmodified
reference is installed under oracle/_ref, the same model, seed and batch are timed through it (eager torch, fp32).
    python tools/bench_planar_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases planar16,vae40]
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

CASES = [("planar16", 40), ("planar32", 1024), ("radial32", 1024), ("sample32", 2 ** 20), ("vae40", 2048)]


def build(nf, kind):
    """-> (model, (lr, weight decay), beta)"""
    import torch
    torch.manual_seed(0)
    d = 40 if kind == "vae40" else 2
    K = {"planar16": 16, "vae40": 40}.get(kind, 32)
    layer = (lambda: nf.flows.Radial((d,))) if kind == "radial32" else (lambda: nf.flows.Planar((d,)))

    class StdNormal(torch.nn.Module):
        def log_prob(self, z):
            return -0.5 * torch.sum(z ** 2, 1)
    target = {"planar16": nf.distributions.TwoModes(2, 0.1), "vae40": StdNormal()}.get(kind)
    if target is None:
        target = nf.distributions.TwoModes(2.0, 0.2)
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(d), [layer() for _ in range(K)], target)
    return model, ((1e-3, 1e-4) if kind in ("planar16", "vae40") else (1e-3, 1e-3)), (0.5 if kind == "planar16" else 1.0)


def time_arm(arm, kind, batch, steps, warmup):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    model, (lr, wd), beta = build(nf, kind)
    model = model.cuda()
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=wd)
    torch.manual_seed(0)

    def step():
        if kind == "sample32":
            with torch.no_grad():
                return model.sample(batch)[1].mean()
        opt.zero_grad(set_to_none=True)
        loss = model.reverse_kld(batch, beta=beta)
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
    return {"model": kind, "batch": batch, "ms_per_step": round(ms, 3), "ms_min": round(times[0], 3),
            "ms_max": round(times[-1], 3), "launches_per_step": launches, "peak_mem_gb": round(peak / 2 ** 30, 3),
            "loss": round(float(loss), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated model names (default: all)")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        want = set(a.cases.split(",")) if a.cases else None
        print(json.dumps([time_arm(a.arm, k, b, a.steps, a.warmup) for k, b in CASES if want is None or k in want]))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_planar_train: no CUDA device")
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
    print(json.dumps({"metric": "planar_radial_train_step", **gpu_info(), **res}))


if __name__ == "__main__":
    main()
