"""Time one training step of the stand-alone spline and MAF layers: `forward_kld` + `backward()` + Adam.
    a    examples/conditional_flow.ipynb: ConditionalNormalizingFlow(DiagGaussian(2, trainable=False),
         4 x [AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4), LULinearPermute(2)]),
         Adam(lr 3e-4, weight decay 1e-5), batch 128 (the notebook's) and 65 536
    b    the same with CoupledRationalQuadraticSpline
    circ examples/circular_nsf.ipynb: 20 x CircularAutoregressiveRationalQuadraticSpline(2, 1, 128, [1],
         tail_bound=[5, pi], permute_mask=True) on DiagGaussian(2) (the notebook trains it on UniformGaussian),
         Adam(lr 1e-4, weight decay 1e-4), batch 1 024
    maf  examples/conditional_flow.ipynb's third model: 4 x [MaskedAffineAutoregressive(2, 128, context_features=4,
         num_blocks=2), LULinearPermute(2)] on DiagGaussian(2, trainable=False), Adam(lr 1e-3, weight decay 1e-5),
         batch 128 (the notebook's) and 65 536
    maf16 4 x [MaskedAffineAutoregressive(16, 256, num_blocks=2), LULinearPermute(16)] on DiagGaussian(16), no context,
         Adam(lr 1e-3, weight decay 1e-5), batch 65 536: the D - 1 adjoint passes of each MAF layer dominate
    paper examples/paper_example_nsf.ipynb: 12 x CircularAutoregressiveRationalQuadraticSpline(2, 1, 512, [1],
         num_bins=10, tail_bound=[5, pi], permute_mask=True) on UniformGaussian(2, [1], [1, 2 pi]) with the GaussianVonMises
         target; the step is `reverse_kld(2**14)` + `backward()` + Adam(lr 5e-4), the notebook's (reverse KL: gradients
         through the sampling direction)
    realnvp examples/real_nvp.ipynb: 64 x [MaskedAffineFlow(MLP([2, 4, 2]) s and t), ActNorm(2)] on DiagGaussian(2), the
         TwoModes(2, 0.1) target, `reverse_kld(batch)` + `backward()` + Adam(lr 1e-4, weight decay 1e-6), batch 20 (the
         notebook's) and 4 096
    augmented examples/augmented_flow.ipynb: 32 x [MaskedAffineFlow(MLP([4, 16, 4]) s and t), ActNorm(4)] on
         DiagGaussian(4), target TwoIndependent(TwoMoons(), DiagGaussian(2)), the same step at batch 20
    colab examples/real_nvp_colab.ipynb: 32 x [AffineCouplingBlock(MLP([1, 64, 64, 2])), Permute(2, 'swap')] on
         DiagGaussian(2), Adam(lr 5e-4, weight decay 1e-5), batch 512 (the notebook's) and 65 536 (forward KL: gradients
         through the density direction).  Also timed with DensityFn.use_native_backward = False (the torch restatement
         of the backward, arm "torch_backward"), in the same run
Prints one JSON line: ms/step (median of CUDA-event-timed steps after warm-up), samples/s, kernel launches per step
(torch.profiler, one separate step), peak device memory, and the card's name, power limit and SM clock read in the same
run.  When the unmodified reference is installed under oracle/_ref, the same model, seed and batch are timed through it
(eager torch, fp32).
    python tools/bench_conditional_train.py [--steps 20] [--warmup 5] [--no-reference] [--cases paper,maf]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


CASES = [("a", 128), ("a", 65536), ("b", 128), ("b", 65536), ("circ", 1024), ("maf", 128), ("maf", 65536),
         ("maf16", 65536), ("paper", 16384), ("realnvp", 20), ("realnvp", 4096), ("augmented", 20),
         ("colab", 512), ("colab", 65536)]
TORCH_BACKWARD_CASES = {"colab"}   # cases whose backward has a torch restatement to compare against
NOTEBOOK_LAYERS = 4   # examples/conditional_flow.ipynb: K = 4 (spline + LU) pairs


def build(nf, kind):
    """-> (model, (lr, weight decay), input features, whether the model takes a context)"""
    import math
    import torch
    torch.manual_seed(0)
    if kind == "paper":
        class GaussianVonMises(nf.distributions.Target):   # the notebook's target
            def __init__(self):
                super().__init__(prop_scale=torch.tensor(2 * math.pi), prop_shift=torch.tensor(-math.pi))
                self.n_dims = 2
                self.max_log_prob = -1.99
                self.log_const = -1.5 * math.log(2 * math.pi) - math.log(1.2660658777520082)   # np.i0(1)

            def log_prob(self, x):
                return -0.5 * x[:, 0] ** 2 + torch.cos(x[:, 1] - 3 * x[:, 0]) + self.log_const
        base = nf.distributions.UniformGaussian(2, [1], torch.tensor([1., 2 * math.pi]))
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 512, [1], num_bins=10,
                                                                        tail_bound=torch.tensor([5., math.pi]),
                                                                        permute_mask=True) for _ in range(12)]
        return nf.NormalizingFlow(base, flows, GaussianVonMises()), (5e-4, 0.0), 2, False
    if kind in ("realnvp", "augmented"):
        d, hid, K = (2, 2, 64) if kind == "realnvp" else (4, 4, 32)
        b = torch.Tensor([1 if i % 2 == 0 else 0 for i in range(d)]) if d == 2 else torch.Tensor([1, 1, 0, 0])
        flows = []
        for i in range(K):
            s = nf.nets.MLP([d, hid * d, d], init_zeros=True)
            t = nf.nets.MLP([d, hid * d, d], init_zeros=True)
            flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(d)]
        target = nf.distributions.TwoModes(2, 0.1) if d == 2 else \
            nf.distributions.TwoIndependent(nf.distributions.TwoMoons(), nf.distributions.DiagGaussian(2))
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(d), flows, target), (1e-4, 1e-6), d, False
    if kind == "colab":
        flows = []
        for _ in range(32):
            flows += [nf.flows.AffineCouplingBlock(nf.nets.MLP([1, 64, 64, 2], init_zeros=True)),
                      nf.flows.Permute(2, mode='swap')]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows), (5e-4, 1e-5), 2, False
    if kind == "circ":
        flows = [nf.flows.CircularAutoregressiveRationalQuadraticSpline(2, 1, 128, [1], tail_bound=torch.tensor([5., math.pi]),
                                                                        permute_mask=True) for _ in range(20)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows), (1e-4, 1e-4), 2, False
    if kind == "maf16":
        flows = []
        for _ in range(NOTEBOOK_LAYERS):
            flows += [nf.flows.MaskedAffineAutoregressive(16, 256, num_blocks=2), nf.flows.LULinearPermute(16)]
        return nf.NormalizingFlow(nf.distributions.DiagGaussian(16), flows), (1e-3, 1e-5), 16, False
    flows = []
    for _ in range(NOTEBOOK_LAYERS):
        if kind == "a":
            flows.append(nf.flows.AutoregressiveRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
        elif kind == "b":
            flows.append(nf.flows.CoupledRationalQuadraticSpline(2, 2, 128, num_context_channels=4))
        else:
            flows.append(nf.flows.MaskedAffineAutoregressive(2, 128, context_features=4, num_blocks=2))
        flows.append(nf.flows.LULinearPermute(2))
    lr = (1e-3, 1e-5) if kind == "maf" else (3e-4, 1e-5)
    return nf.ConditionalNormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows), lr, 2, True


def time_arm(arm, kind, batch, steps, warmup):
    import numpy as np
    import torch
    if arm == "reference":
        sys.path.insert(0, REF_DIR)
    else:
        sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import normflows as nf
    if arm == "torch_backward":
        from normflows._autograd import DensityFn
        DensityFn.use_native_backward = False
    dev = torch.device("cuda")
    model, (lr, wd), dim, conditional = build(nf, kind)
    model = model.to(dev)
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(batch, dim, generator=g) * 1.2).to(dev)
    ctx = torch.cat([torch.randn(batch, 2, generator=g), 0.5 + 0.5 * torch.rand(batch, 2, generator=g)], 1).to(dev) \
        if conditional else None
    if kind in ("realnvp", "augmented"):
        model.sample(num_samples=2 ** 7)   # the notebooks' ActNorm initialisation
    opt = torch.optim.Adam(model.parameters(), lr=lr, weight_decay=wd)
    np.random.seed(0)
    torch.manual_seed(0)

    def step():
        opt.zero_grad(set_to_none=True)
        if kind in ("paper", "realnvp", "augmented"):
            loss = model.reverse_kld(batch)
        else:
            loss = model.forward_kld(x) if ctx is None else model.forward_kld(x, ctx)
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
    return {"model": kind, "batch": batch, "ms_per_step": round(ms, 3),
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--cases", help="comma-separated model names (default: all)")
    ap.add_argument("--arm", choices=["native", "torch_backward", "reference"], help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:   # one arm in its own process (the two packages share the name `normflows`)
        want = set(a.cases.split(",")) if a.cases else None
        if a.arm == "torch_backward":
            want = (want or TORCH_BACKWARD_CASES) & TORCH_BACKWARD_CASES
        print(json.dumps([time_arm(a.arm, k, b, a.steps, a.warmup) for k, b in CASES if want is None or k in want]))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_conditional_train: no CUDA device")
    cases = set(a.cases.split(",")) if a.cases else None
    arms = ["native"] + (["torch_backward"] if cases is None or cases & TORCH_BACKWARD_CASES else []) + (["reference"] if not a.no_reference and os.path.isdir(os.path.join(REF_DIR, "normflows"))
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
    print(json.dumps({"metric": "conditional_spline_train_step", **gpu_info(), **res}))


if __name__ == "__main__":
    main()
