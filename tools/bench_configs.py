"""Timings of the BASELINE.json parity-test configurations that are NOT the bench line:
  C1  Real NVP 2-D (examples/real_nvp.ipynb cell 2 with K=8): 8 x [MaskedAffineFlow(MLP[2,4,2]), ActNorm(2)],
      batch 4096, forward_kld
  C3  Glow (examples/glow.ipynb cell 2): L=3, K=16, hidden 256, 3x32x32 images, batch 1024, forward_kld
  C2' the Coupled RQ-NSF variant of the bench line (SURVEY 8d reports both)
Device-resident inputs, CUDA events, median of the timed calls.  Prints one JSON line per configuration:
    python tools/bench_configs.py [c1 c2 c3 c5]"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "normalizing-flows_b200"))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import normflows as nf  # noqa: E402

torch.set_grad_enabled(False)


def timed(fn, warmup=5, iters=30):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def real_nvp():
    torch.manual_seed(0)
    b = torch.Tensor([1 if i % 2 == 0 else 0 for i in range(2)])
    flows = []
    for i in range(8):
        s = nf.nets.MLP([2, 4, 2], init_zeros=True)
        t = nf.nets.MLP([2, 4, 2], init_zeros=True)
        flows += [nf.flows.MaskedAffineFlow(b if i % 2 == 0 else 1 - b, t, s), nf.flows.ActNorm(2)]
    m = nf.NormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows).cuda()
    x = nf.distributions.TwoMoons().sample(4096).cuda()
    m.forward_kld(x)  # ActNorm data-dependent init (one-time)
    ms = timed(lambda: m.forward_kld(x), iters=200)
    return {"config": "C1 Real NVP 2-D, 8 x [MaskedAffineFlow(MLP[2,4,2]) + ActNorm], batch 4096, forward_kld",
            "ms": ms, "samples_per_s": 4096 / ms * 1e3, "launches": m._stack().launch_count()}


def glow():
    torch.manual_seed(0)
    L_, K, hidden, shape, ncls = 3, 16, 256, (3, 32, 32), 10
    q0, merges, flows = [], [], []
    for i in range(L_):
        fl = [nf.flows.GlowBlock(shape[0] * 2 ** (L_ + 1 - i), hidden, split_mode="channel", scale=True)
              for _ in range(K)] + [nf.flows.Squeeze()]
        flows += [fl]
        if i > 0:
            merges += [nf.flows.ImageMerge()]
            ls = (shape[0] * 2 ** (L_ - i), shape[1] // 2 ** (L_ - i), shape[2] // 2 ** (L_ - i))
        else:
            ls = (shape[0] * 2 ** (L_ + 1), shape[1] // 2 ** L_, shape[2] // 2 ** L_)
        q0 += [nf.distributions.ClassCondDiagGaussian(ls, ncls)]
    m = nf.MultiscaleFlow(q0, flows, merges).cuda()
    x = torch.rand(1024, *shape).cuda()
    y = torch.randint(ncls, (1024,)).cuda()
    m.forward_kld(x, y)  # ActNorm init
    ms = timed(lambda: m.forward_kld(x, y), warmup=2, iters=8)
    return {"config": "C3 Glow L=3 K=16 hidden 256, 3x32x32, batch 1024, forward_kld (one nfb_glow_block call per GlowBlock: folded 1x1 conv, fused wgmma conditioner, tap-form coupling)",
            "ms": ms, "images_per_s": 1024 / ms * 1e3, "tflops_algorithmic": 1.303e9 * 1024 / ms / 1e9}


def coupled_nsf():
    import bench
    m = bench.build_model("coupled", 32).cuda()
    x = (torch.randn(65536, 64, generator=torch.Generator().manual_seed(1234)) * 1.5).cuda()
    ms = timed(lambda: m.forward_kld(x))
    return {"config": "C2' Coupled RQ-NSF d=64, 32 x [spline + LULinearPermute], batch 65536, forward_kld",
            "ms": ms, "samples_per_s": 65536 / ms * 1e3, "launches": m._stack().launch_count()}


def residual_flow():
    """BASELINE config 5: 16 x Residual(LipschitzMLP([2, 128, 128, 128, 2])) (examples/residual.ipynb), batch 131 072,
    forward_kld in TRAINING mode = the stochastic (Russian-roulette + Hutchinson) log-det estimator of
    flows/residual.py:163-217, and in eval mode = the exact 2 x 2 Jacobian path (:148-161)."""
    import numpy as np
    torch.manual_seed(0)
    np.random.seed(0)
    flows = [nf.flows.Residual(nf.nets.LipschitzMLP([2, 128, 128, 128, 2], init_zeros=True, lipschitz_const=0.9),
                               reduce_memory=True) for _ in range(16)]
    m = nf.NormalizingFlow(nf.distributions.DiagGaussian(2, trainable=False), flows).cuda()
    x = nf.distributions.TwoMoons().sample(131072).cuda()
    m.train()
    ms_train = timed(lambda: m.forward_kld(x), warmup=2, iters=8)
    m.eval()
    ms_eval = timed(lambda: m.forward_kld(x), warmup=2, iters=8)
    return {"config": "C5 Residual flow 2-D, 16 x iResBlock(LipschitzMLP[2,128,128,128,2]), batch 131072, forward_kld",
            "ms_stochastic_estimator": ms_train, "samples_per_s_stochastic": 131072 / ms_train * 1e3,
            "ms_exact_2x2": ms_eval, "samples_per_s_exact": 131072 / ms_eval * 1e3}


CONFIGS = (("c1", real_nvp), ("c2", coupled_nsf), ("c3", glow), ("c5", residual_flow))

if __name__ == "__main__":
    which = sys.argv[1:] or ["c1", "c2", "c3", "c5"]
    for name, fn in CONFIGS:
        if name in which:
            print(json.dumps(fn()), flush=True)
