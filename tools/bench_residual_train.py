"""Time one residual-flow training step of BASELINE config 5 (16 x Residual(LipschitzMLP([2, 128, 128, 128, 2])),
DiagGaussian(2, trainable=False); the loop of examples/residual.ipynb): `forward_kld(x)` + `backward()` + Adam(lr 3e-4,
weight decay 1e-5), at batch 131 072 (config 5) and 512 (the notebook's), and separately the same step followed by the
notebook's `update_lipschitz(model, 50)`.

Prints one JSON line: ms/step (median of CUDA-event-timed steps after warm-up), samples/s, kernel launches per step
(torch.profiler, one separate step), peak device memory, and the card's name, power limit and SM clock read in the same
run.  The random truncation n of every block is drawn from numpy's generator seeded identically in both arms, so both
run the same number of power-series terms.  When the unmodified reference is installed under oracle/_ref, the same
model, seed and batch are timed through it (eager torch, fp32).

    python tools/bench_residual_train.py [--batches 131072 512] [--steps 10] [--warmup 3] [--no-reference]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def build(nf):
    import torch
    torch.manual_seed(0)
    flows = [nf.flows.Residual(nf.nets.LipschitzMLP([2, 128, 128, 128, 2], init_zeros=True, lipschitz_const=0.9),
                               reduce_memory=True) for _ in range(16)]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows)


def time_arm(arm, batch, steps, warmup, lipschitz):
    import numpy as np
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    dev = torch.device("cuda")
    model = build(nf).to(dev)
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(batch, 2, generator=g) * 1.2).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4, weight_decay=1e-5)
    np.random.seed(0)
    torch.manual_seed(0)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = model.forward_kld(x)
        loss.backward()
        opt.step()
        if lipschitz:
            nf.utils.update_lipschitz(model, 50)
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
    if not torch.isfinite(loss):
        raise RuntimeError("non-finite loss")
    peak = torch.cuda.max_memory_allocated()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    times.sort()
    ms = times[len(times) // 2]
    return {"batch": batch, "update_lipschitz": lipschitz, "ms_per_step": round(ms, 3),
            "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3),
            "samples_per_s": round(batch / ms * 1e3, 1), "launches_per_step": launches,
            "peak_mem_gb": round(peak / 2 ** 30, 2), "loss": round(float(loss), 4)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, sm, sm_max = [s.strip() for s in q.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock_at_end": sm, "sm_clock_max": sm_max}
    except Exception:  # noqa: BLE001 -- recorded as unknown, never guessed
        import torch
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[131072, 512])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        print(json.dumps([time_arm(a.arm, b, a.steps, a.warmup, lip) for b in a.batches for lip in (False, True)]))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_residual_train: no CUDA device")
    arms = ["native"] + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
                         else [])
    res = {}
    for arm in arms:
        cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--steps", str(a.steps), "--warmup", str(a.warmup),
               "--batches", *map(str, a.batches)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            res[arm] = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}
        else:
            res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps({"metric": "residual_c5_train_step", **gpu_info(), **res}))


if __name__ == "__main__":
    main()
