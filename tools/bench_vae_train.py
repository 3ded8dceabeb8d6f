"""Time one training step of examples/vae.ipynb's flow-VAE: `nfm(x, num_samples)`, loss mean(log_q) - mean(log_p),
`backward()` and Adam(lr 1e-4, weight decay 1e-4), on seeded synthetic binarised 28 x 28 data.
    vae_planar        the notebook's step: 784-512-256-80 NNDiagGaussian, 40 x Planar((40,)), 40-256-512-784
                      NNBernoulliDecoder, MultivariateNormal prior, batch 64, num_samples 32 (2 048 rows)
    vae_radial        the same with flow_type 'Radial'
    vae_realnvp16     flow_type 'RealNVP' at the 16-feature setting of DESIGN §7's known limitation
    vae_planar_b1024  vae_planar at batch 1 024 (32 768 rows); also times the Bernoulli kernels on their own
Prints one JSON line per case: ms/step (median and range of CUDA-event-timed steps after warm-up), kernel launches per
step (torch.profiler, one separate step), peak device memory, the first step's loss, and the card's name and power limit
read in the same run.  When the unmodified reference is installed under oracle/_ref, the same model, seed and data are
timed through it (eager torch, fp32); both arms draw the same noise, so their first-step losses agree.
    python tools/bench_vae_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases vae_planar,vae_radial]
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

CASES = [("vae_planar", "Planar", 64), ("vae_radial", "Radial", 64), ("vae_realnvp16", "RealNVP", 64),
         ("vae_planar_b1024", "Planar", 1024)]
NUM_SAMPLES = 32
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def build(nf, flow_type):
    """examples/vae.ipynb's model cell (RealNVP: the setting of DESIGN §7's known limitation)."""
    import numpy as np
    import torch
    n_flows, n_bottleneck = 40, 16 if flow_type == "RealNVP" else 40
    prior = torch.distributions.MultivariateNormal(torch.zeros(n_bottleneck, device="cuda"),
                                                   torch.eye(n_bottleneck, device="cuda"))
    encoder = nf.distributions.NNDiagGaussian(nf.nets.MLP(np.array([28 ** 2, 512, 256, n_bottleneck * 2])))
    decoder = nf.distributions.NNBernoulliDecoder(nf.nets.MLP(np.array([n_bottleneck, 256, 512, 28 ** 2])))
    if flow_type == "Planar":
        flows = [nf.flows.Planar((n_bottleneck,)) for _ in range(n_flows)]
    elif flow_type == "Radial":
        flows = [nf.flows.Radial((n_bottleneck,)) for _ in range(n_flows)]
    else:
        b = torch.tensor(n_bottleneck // 2 * [0, 1] + n_bottleneck % 2 * [0])
        flows = []
        for i in range(n_flows):
            s = nf.nets.MLP([n_bottleneck, n_bottleneck], init_zeros=True)
            t = nf.nets.MLP([n_bottleneck, n_bottleneck], init_zeros=True)
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s)]
    return nf.NormalizingFlowVAE(prior, encoder, flows, decoder).cuda()


def data(batch, n_batches):
    """Seeded binarised 28 x 28 images (blobs plus pixel noise), flattened to [n_batches, batch, 784]."""
    import torch
    g = torch.Generator().manual_seed(1)
    yy, xx = torch.meshgrid(torch.arange(28.0), torch.arange(28.0), indexing="ij")
    c = 8 + torch.rand(10, 2, generator=g) * 12
    r = 4 + 3 * torch.rand(10, generator=g)
    T = ((((yy[None] - c[:, 0, None, None]) ** 2 + (xx[None] - c[:, 1, None, None]) ** 2).sqrt() - r[:, None, None])
         .abs() < 1.5).float().reshape(10, 784)
    idx = torch.randint(0, 10, (n_batches * batch,), generator=g)
    flip = (torch.rand(n_batches * batch, 784, generator=g) < 0.03).float()
    return (T[idx] != flip).float().reshape(n_batches, batch, 784).cuda()


def bernoulli_kernels(batch, reps=50):
    """CUDA-event time of nfb_bernoulli_log_prob and its backward at batch x NUM_SAMPLES rows x 784, and their bytes."""
    import torch
    from normflows import _vae
    rows, D = batch * NUM_SAMPLES, 784
    score = torch.randn(rows, D, device="cuda") * 3
    x = (torch.rand(batch, D, device="cuda") > 0.5).float()
    g = torch.randn(rows, device="cuda")
    out, gs = torch.empty(rows, device="cuda"), torch.empty_like(score)
    from normflows import _lib as L
    lib = L.lib()
    fwd = lambda: lib.nfb_bernoulli_log_prob(L.ptr(score), L.ptr(x), rows, D, NUM_SAMPLES, L.ptr(out), L.stream_ptr())
    bwd = lambda: lib.nfb_bernoulli_log_prob_backward(L.ptr(score), L.ptr(x), L.ptr(g), rows, D, NUM_SAMPLES,
                                                      L.ptr(gs), None, L.stream_ptr())
    assert torch.equal(_vae.bernoulli_log_prob(score, x, NUM_SAMPLES), _vae.bernoulli_log_prob(score, x, NUM_SAMPLES))
    res = {}
    # bytes the kernels must move: score [rows, D] and x [batch, D] read, log_p [rows] written (forward); score, x and
    # g read, g_score [rows, D] written (backward)
    nbytes = {"fwd": 4 * (rows * D + batch * D + rows), "bwd": 4 * (2 * rows * D + batch * D + rows)}
    for name, fn in (("fwd", fwd), ("bwd", bwd)):
        for _ in range(5):
            L.check(fn())
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        b.synchronize()
        us = a.elapsed_time(b) * 1e3 / reps
        res[f"bernoulli_{name}_us"] = round(us, 2)
        res[f"bernoulli_{name}_bytes"] = nbytes[name]
        res[f"bernoulli_{name}_hbm_share"] = round(nbytes[name] / (us * 1e-6) / HBM_BYTES_PER_S, 3)
    return res


def time_arm(arm, kind, flow_type, batch, steps, warmup):
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    torch.manual_seed(0)
    nfm = build(nf, flow_type)
    n_batches = warmup + steps + 2
    xs = data(batch, n_batches)
    opt = torch.optim.Adam(nfm.parameters(), lr=1e-4, weight_decay=1e-4)
    torch.manual_seed(0)
    it = iter(range(n_batches))

    def step():
        x = xs[next(it)]
        opt.zero_grad()
        z, log_q, log_p = nfm(x, NUM_SAMPLES)
        loss = torch.mean(log_q) - torch.mean(log_p)
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
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                   and "memcpy" not in e.name.lower() and "memset" not in e.name.lower())
    times.sort()
    out = {"model": kind, "batch": batch, "rows": batch * NUM_SAMPLES, "ms_per_step": round(times[len(times) // 2], 3),
           "ms_min": round(times[0], 3), "ms_max": round(times[-1], 3), "launches_per_step": launches,
           "peak_mem_gb": round(peak / 2 ** 30, 3), "first_loss": round(first, 4), "loss": round(float(loss), 4)}
    if arm == "native" and kind == "vae_planar_b1024":
        out.update(bernoulli_kernels(batch))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated model names (default: all)")
    ap.add_argument("--arm", choices=["native", "reference"], help=argparse.SUPPRESS)
    ap.add_argument("--case", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm and case in its own process (the two packages share the name `normflows`)
        kind, flow_type, batch = next(c for c in CASES if c[0] == a.case)
        print(json.dumps(time_arm(a.arm, kind, flow_type, batch, a.steps, a.warmup)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_vae_train: no CUDA device")
    arms = ["native"] + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
                         else [])
    want = set(a.cases.split(",")) if a.cases else None
    info = gpu_info()
    for kind, _, _ in CASES:
        if want is not None and kind not in want:
            continue
        res = {}
        for arm in arms:
            cmd = [sys.executable, os.path.abspath(__file__), "--arm", arm, "--case", kind, "--steps", str(a.steps),
                   "--warmup", str(a.warmup)]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode:
                res[arm] = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else f"exit {r.returncode}"}
            else:
                res[arm] = json.loads(r.stdout.strip().splitlines()[-1])
        print(json.dumps({"metric": "vae_train_step", "case": kind, **info, **res}), flush=True)


if __name__ == "__main__":
    main()
