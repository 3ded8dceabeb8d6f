"""Time one Glow training step of BASELINE config 3 (examples/glow.ipynb: L=3, K=16, hidden 256, 3x32x32, 10 classes):
`forward_kld(x, y)` + `backward()` + Adamax(lr 1e-3, weight decay 1e-5), at batch 128 (the notebook's) and 1024.

Prints one JSON line: ms/step (median of CUDA-event-timed steps after warm-up), images/s, kernel launches per step
(torch.profiler, one separate step), peak device memory, algorithmic TFLOP/s and the card's name and power limit read in
the same run.  When the unmodified reference is installed under oracle/_ref, the same model, seed and batch are timed
through it (eager torch; cuDNN convolutions in TF32 when torch.backends.cudnn.allow_tf32, which is recorded).

    python tools/bench_glow_train.py [--batches 128 1024] [--steps 20] [--warmup 5] [--no-reference]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

# multiply-adds of the conditioner convolutions per image (the 1x1 C x C maps are negligible): per level (channels C at
# H x W): K blocks x [3x3 C/2 -> 256, 1x1 256 -> 256, 3x3 256 -> C] ; forward 1.303 GFLOP per image.  A training step
# runs the forward, the recompute in backward, the data and the weight gradient: 4 x that.
def glow_flop_per_image(L_=3, K=16, hidden=256, shape=(3, 32, 32)):
    total = 0
    for i in range(L_):
        C = shape[0] * 2 ** (L_ + 1 - i)
        s = shape[1] // 2 ** (L_ - i) if i > 0 else shape[1] // 2 ** L_
        hw = s * s
        macs = hw * (9 * (C // 2) * hidden + hidden * hidden + 9 * hidden * C)
        total += K * 2 * macs
    return total


def build(nf, merge_cls, L_=3, K=16, hidden=256, shape=(3, 32, 32), ncls=10):
    import torch
    torch.manual_seed(0)
    q0, merges, flows = [], [], []
    for i in range(L_):
        flows.append([nf.flows.GlowBlock(shape[0] * 2 ** (L_ + 1 - i), hidden, split_mode="channel", scale=True)
                      for _ in range(K)] + [nf.flows.Squeeze()])
        if i > 0:
            merges.append(merge_cls())
            ls = (shape[0] * 2 ** (L_ - i), shape[1] // 2 ** (L_ - i), shape[2] // 2 ** (L_ - i))
        else:
            ls = (shape[0] * 2 ** (L_ + 1), shape[1] // 2 ** L_, shape[2] // 2 ** L_)
        q0.append(nf.distributions.ClassCondDiagGaussian(ls, ncls))
    return nf.MultiscaleFlow(q0, flows, merges)


def time_arm(arm, batch, steps, warmup):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
        import normflows as nf
        model = build(nf, nf.flows.Merge)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
        import normflows as nf
        model = build(nf, nf.flows.ImageMerge)
    dev = torch.device("cuda")
    model = model.to(dev)
    g = torch.Generator().manual_seed(1)
    x = torch.rand(batch, 3, 32, 32, generator=g).to(dev)
    y = torch.randint(10, (batch,), generator=g).to(dev)
    with torch.no_grad():
        model.log_prob(x, y)   # ActNorm data-dependent init, outside the timed steps
    opt = torch.optim.Adamax(model.parameters(), lr=1e-3, weight_decay=1e-5)

    def step():
        opt.zero_grad(set_to_none=True)
        loss = model.forward_kld(x, y)
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
    out = {"arm": arm, "batch": batch, "ms_per_step": round(ms, 3), "images_per_s": round(batch / ms * 1e3, 1),
           "launches_per_step": launches, "peak_mem_gb": round(peak / 2 ** 30, 2),
           "tflops_algorithmic": round(4 * glow_flop_per_image() * batch / (ms * 1e-3) / 1e12, 1),
           "loss": round(float(loss), 3)}
    if arm == "reference":
        out["cudnn_allow_tf32"] = bool(torch.backends.cudnn.allow_tf32)
    return out


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
        return name, power
    except Exception:  # noqa: BLE001 -- recorded as unknown, never guessed
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[128, 1024])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        print(json.dumps([time_arm(a.arm, b, a.steps, a.warmup) for b in a.batches]))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_glow_train: no CUDA device")
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
    name, power = gpu_info()
    print(json.dumps({"metric": "glow_c3_train_step", "gpu": name, "power_limit": power,
                      "flop_per_image_forward": glow_flop_per_image(), **res}))


if __name__ == "__main__":
    main()
