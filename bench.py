#!/usr/bin/env python
"""bench.py -- samples/sec of `forward_kld` on the flagship neural-spline stack (BASELINE.json metric).

    python bench.py --gpus 1 --steps 20 --warmup 5          # ours, one H100
    torchrun --nproc-per-node N ... bench.py --gpus N ...    # data parallel: batch sharded, one all-reduce
    python bench.py --impl reference ...                     # CPU arm: the unmodified reference on the host cores
    python bench.py --impl reference-eager ...               # the unmodified reference, PyTorch eager on cuda:0

Workload (configs[1] of BASELINE.json; SURVEY 8d): 32 x [AutoregressiveRationalQuadraticSpline(64, 2
blocks, 256 hidden, 8 bins, tail 3) + LULinearPermute(64)], DiagGaussian(64) base, batch 65 536 per GPU,
fp32 in/out, synthetic inputs x = 1.5 * randn, random-init weights moved off identity-init
(sigma 0.03 on the conditioners, 0.01 on the LU factors) so that splines/tails are non-degenerate.  (SURVEY 8d's
sigma = 0.05 recipe was written for 4-layer stacks: at 32 layers it makes the map explode -- forward_kld = 19 431,
|z| up to 122, and the reference's own fp32 run then differs from its fp64 run by 1.5e-2 -- so the flagship uses
the milder perturbation: forward_kld = 301.7, reference fp32-vs-fp64 <= 6e-6.)
One "step" = one full `forward_kld` pass over one batch (all 64 layers + base density + mean).

Timed region: W warm-up steps, then exactly K steps between barrier+synchronize, CUDA events on the
launching stream, max over ranks.  Inputs rotate through NBUF distinct device batches whose total size
(160 MB) exceeds L2 (so no step re-reads its input from L2); the packed weights cycle through L2 as they
do in real use.  `e2e` is the same pass through the C-ABI host entry point (`nfb_flow_forward_kld_host`):
pinned host batch -> H2D -> kernels -> D2H of the scalar loss, every step.
--dump-outputs DIR writes what the timed paths returned in their last step (DIR/forward_kld.npy: the loss of the
device path; DIR/forward_kld_host.npy: the loss of the host entry point), float64.  Inputs and weights are seeded,
so two builds run with the same arguments can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]

D, LAYERS, HIDDEN, BLOCKS, BINS, TAIL = 64, 32, 256, 2, 8, 3.0
BATCH = 65536
KIND = os.environ.get("NFB_BENCH_KIND", "ar")  # "ar" (BASELINE config 2) or "coupled"
# algorithmic work per sample per [spline block + LU] (SURVEY 8d table): GEMM flops 2*sum(in*out)
FLOPS_PER_SAMPLE_LAYER = {"ar": 1_327_104, "coupled": 933_888}
MIN_BYTES_PER_SAMPLE_LAYER = 520  # z in + z out + log_q r/w
METRIC = "samples/sec forward_kld, 32-layer RQ-NSF d=64 batch=65536"


def workload_name(batch=BATCH):
    return (f"{'Autoregressive' if KIND == 'ar' else 'Coupled'} RQ-NSF d={D}, {LAYERS} x "
            f"[spline block(2 blocks, hidden {HIDDEN}, {BINS} bins) + LULinearPermute], "
            f"batch {batch}/GPU, forward_kld (BASELINE.json configs[1])")


def build_model(kind=KIND, layers=LAYERS, seed=0):
    import torch
    import normflows as nf
    torch.manual_seed(seed)
    fl = []
    for i in range(layers):
        if kind == "ar":
            fl.append(nf.flows.AutoregressiveRationalQuadraticSpline(D, BLOCKS, HIDDEN, num_bins=BINS, tail_bound=TAIL))
        else:
            fl.append(nf.flows.CoupledRationalQuadraticSpline(D, BLOCKS, HIDDEN, num_bins=BINS, tail_bound=TAIL,
                                                             reverse_mask=bool(i % 2)))
        fl.append(nf.flows.LULinearPermute(D))
    model = nf.NormalizingFlow(nf.distributions.DiagGaussian(D, trainable=False), fl)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for name, p in model.named_parameters():
            p.add_((0.01 if ".linear." in name else 0.03) * torch.randn(p.shape, generator=g))
    return model


def oracle_spec(kind=KIND, layers=LAYERS):
    t = "AutoregressiveRationalQuadraticSpline" if kind == "ar" else "CoupledRationalQuadraticSpline"
    return {"kind": "NormalizingFlow", "q0": {"shape": [D]},
            "flows": [{"type": t, "num_bins": BINS, "tail_bound": TAIL}, {"type": "LULinearPermute"}] * layers}


class ClockSampler(threading.Thread):
    """Samples nvidia-smi SM clocks / throttle reasons during the timed region (read-only queries)."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.rows, self._stop_evt = index, [], threading.Event()

    def run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self._stop_evt.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}",
                                      "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=5)
                parts = [s.strip() for s in out.stdout.strip().split(",")]
                if len(parts) >= 6:
                    self.rows.append(parts)
            except Exception:
                pass
            self._stop_evt.wait(0.1)

    def stop(self):
        self._stop_evt.set()
        self.join(timeout=6)
        sm = sorted(int(r[0]) for r in self.rows if r[0].isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(r[2 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None,
                "sm_max_mhz": int(self.rows[0][1]) if self.rows and self.rows[0][1].isdigit() else None,
                "reasons": reasons, "samples": len(self.rows)}


# ---------------------------------------------------------------------------------------------------------
# CPU legs.  `--impl reference` and the GPU line's `cpu_baseline` both time the UNMODIFIED reference package
# (oracle/_ref/normflows, installed by __graft_entry__.build() through oracle/reference.py) on the host cores.
# The batch is data-parallel, so it is sharded over worker processes exactly like the GPU arm shards it over
# GPUs: every worker builds the same model (same seed) with the reference's own classes and runs
# `model.forward_kld(x_shard)` under no_grad.  The oracle port (oracle/nf_oracle.py) is the fallback only when
# oracle/_ref is absent (kind "port").
# ---------------------------------------------------------------------------------------------------------
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
_W = {}


def usable_cpus():
    """Host cores this process may actually use: min(affinity, cgroup CPU quota).  A container can show many more
    logical CPUs than its cgroup quota (cpu.max) lets it run; sizing the worker pool by os.cpu_count() would then
    oversubscribe the quota and throttle."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            n = min(n, max(1, int(int(q) / int(p))))
    except Exception:
        pass
    return max(1, n)


def reference_available():
    return os.path.isfile(os.path.join(REF_DIR, "normflows", "__init__.py"))


def _use_reference_package():
    """Put the unmodified reference first on sys.path (worker processes / the eager-CUDA leg only)."""
    assert "normflows" not in sys.modules or sys.modules["normflows"].__file__.startswith(REF_DIR)
    sys.path.insert(0, REF_DIR)
    import normflows as nf
    assert nf.__file__.startswith(REF_DIR), nf.__file__
    return nf


def _ref_worker_init(kind, threads, rows, seed, use_ref):
    import torch
    torch.set_num_threads(threads)
    torch.set_grad_enabled(False)
    _W["rows"] = rows
    g = torch.Generator().manual_seed(seed)
    if use_ref:
        _use_reference_package()
        _W["model"] = build_model(kind)
        _W["x"] = torch.randn(rows, D, generator=g) * 1.5
        _W["step"] = lambda: float(_W["model"].forward_kld(_W["x"]))
    else:
        import numpy as np
        from threadpoolctl import threadpool_limits
        from oracle import nf_oracle as O
        model = build_model(kind)  # our parameter containers: only the state_dict is used
        sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
        spec, x = oracle_spec(kind), (torch.randn(rows, D, generator=g) * 1.5).numpy()

        def step():
            with threadpool_limits(limits=threads):
                return float(O.forward_kld(spec, sd, x))
        _W["step"] = step


def _ref_worker_main(conn, kind, threads, rows, seed, use_ref):
    _ref_worker_init(kind, threads, rows, seed, use_ref)
    conn.send("ready")
    while True:
        msg = conn.recv()
        if msg == "stop":
            return
        t0 = time.perf_counter()
        kld = _W["step"]()
        conn.send((time.perf_counter() - t0, kld))


class CpuReference:
    """Persistent worker processes (one pipe each); one `step()` = one forward_kld pass over `rows_total` rows
    sharded over the workers, timed as the wall-clock until the slowest worker is done (what a data-parallel CPU
    job sees)."""

    def __init__(self, rows_total, kind=KIND):
        import multiprocessing as mp
        self.cores = usable_cpus()
        self.threads = int(os.environ.get("NFB_REF_THREADS", 4 if self.cores >= 8 else self.cores))
        self.workers = max(1, self.cores // self.threads)
        self.rows = max(1, rows_total // self.workers)
        self.rows_total = self.rows * self.workers
        self.use_ref = reference_available()
        ctx = mp.get_context("spawn")
        self.procs, self.conns = [], []
        for i in range(self.workers):
            parent, child = ctx.Pipe()
            p = ctx.Process(target=_ref_worker_main, daemon=True,
                            args=(child, kind, self.threads, self.rows, 1234 + i, self.use_ref))
            p.start()
            self.procs.append(p)
            self.conns.append(parent)
        for c in self.conns:
            assert c.recv() == "ready"

    def step(self):
        t0 = time.perf_counter()
        for c in self.conns:
            c.send("go")
        res = [c.recv() for c in self.conns]
        return time.perf_counter() - t0, res[0][1]

    def close(self):
        for c in self.conns:
            c.send("stop")
        for p in self.procs:
            p.join(timeout=10)

    def describe(self, steps, warmup, wall):
        what = ("unmodified reference package (oracle/_ref/normflows, torch CPU fp32) model.forward_kld under no_grad"
                if self.use_ref else "oracle/nf_oracle.py (numpy fp32 port; oracle/_ref absent) forward_kld")
        return (f"{what}; {self.workers} worker processes x {self.threads} torch threads, {self.rows} rows each = "
                f"{self.rows_total} rows per step, {warmup} warm-up + {steps} timed steps ({wall:.1f} s wall incl. start-up)")


def time_cpu_reference(rows_total, steps, warmup, kind=KIND):
    t_start = time.time()
    ref = CpuReference(rows_total, kind)
    try:
        for _ in range(warmup):
            ref.step()
        times, kld = [], None
        for _ in range(steps):
            dt, kld = ref.step()
            times.append(dt)
    finally:
        ref.close()
    total = sum(times)
    value = ref.rows_total * steps / total
    base = {"value": value, "unit": "samples/s", "cores": ref.workers * ref.threads, "logical_cpus": os.cpu_count(),
            "kind": "reference" if ref.use_ref else "port",
            "sample": ref.describe(steps, warmup, time.time() - t_start) + f"; kld={kld:.4f}",
            "rows_per_step": ref.rows_total, "same_config": ref.rows_total == BATCH}
    return base, total / steps


def cpu_baseline(kind=KIND):
    """GPU line's `cpu_baseline` (rank 0, N = 1): 1 warm-up + 2 timed passes of the reference over a bounded sample
    (16 384 rows = 4096 per worker at 16 usable cores)."""
    return time_cpu_reference(16384 if usable_cpus() >= 8 else 4096, steps=2, warmup=1, kind=kind)


def run_reference(args):
    """--impl reference: the unmodified reference's CPU path on all host cores, same metric / workload / batch.
    One step = one forward_kld pass over the batch sharded over worker processes (65 536 rows for short runs, a
    16 384-row sample -- 4096 rows per worker -- when K + W > 4; 4096 rows on hosts with < 8 usable cores)."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    steps = max(1, args.steps)
    # full batch when the run is short; otherwise a bounded sample (>= 4096 rows per worker process) so that
    # warm-up + K steps end within a few minutes on a 16-core host
    cores = usable_cpus()
    if cores < 8:
        rows = min(args.batch, 4096)
    elif cores >= 16 and steps + max(1, args.warmup) <= 4:
        rows = args.batch
    else:
        rows = min(args.batch, 16384)
    base, dt = time_cpu_reference(rows, steps, max(1, args.warmup))
    line = {"impl": "reference", "metric": METRIC, "value": base["value"],
            "unit": "samples/s", "n_gpus": args.gpus, "steps": steps, "warmup": max(1, args.warmup),
            "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_name(args.batch), "sample": f"{base['rows_per_step']} rows per step",
                       "same_config": base["same_config"]},
            "cpu_baseline": base,
            "e2e": {"value": base["value"], "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def run_reference_eager_cuda(args):
    """--impl reference-eager: the unmodified reference in PyTorch eager mode on cuda:0 -- the denominator of
    north_star's >= 10x target (BASELINE.md section 4).  10 warm-up + 50 timed passes, CUDA events, median."""
    import torch
    nf = _use_reference_package()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    model = build_model().to(dev)
    g = torch.Generator().manual_seed(1234)
    x = (torch.randn(args.batch, D, generator=g) * 1.5).to(dev)
    for _ in range(10):
        loss = model.forward_kld(x)
    torch.cuda.synchronize()
    ts = []
    for _ in range(max(1, args.steps)):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loss = model.forward_kld(x)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    med = ts[len(ts) // 2]
    print(json.dumps({"impl": "reference-eager", "package": nf.__file__, "version": nf.__version__,
                      "device": torch.cuda.get_device_name(0), "batch": args.batch, "steps": len(ts),
                      "ms_per_step_median": med, "ms_per_step_min": ts[0], "value": args.batch / (med * 1e-3),
                      "unit": "samples/s", "loss": float(loss), "tf32": torch.backends.cuda.matmul.allow_tf32}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "reference-eager"])
    ap.add_argument("--batch", type=int, default=BATCH, help="rows per GPU (weak scaling)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-reference-eager", action="store_true")
    ap.add_argument("--no-train-step", action="store_true")
    ap.add_argument("--no-extra-configs", action="store_true", help="skip BASELINE configs C1 / C2' / C3 / C5 (extra keys)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's outputs as DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    if args.impl == "reference":
        return run_reference(args)
    if args.impl == "reference-eager":
        return run_reference_eager_cuda(args)

    import numpy as np
    import torch
    import torch.distributed as dist
    import normflows as nf
    from normflows.parallel import forward_kld_dp
    torch.set_grad_enabled(False)  # the metric is the forward pass (SURVEY 8d: timed under torch.no_grad())

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert world == args.gpus, f"launched {world} ranks for --gpus {args.gpus}"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
        # NCCL sets channels up lazily over the first collectives (hundreds of ms when the GPU is busy):
        # keep that out of the warm-up/timed steps
        t = torch.ones(2, dtype=torch.float64, device=dev)
        for _ in range(20):
            dist.all_reduce(t)
        torch.cuda.synchronize()
        dist.barrier()
    warmup = max(3, args.warmup)
    steps = args.steps
    B = args.batch

    model = build_model().to(dev)
    nbuf = max(2, (160 << 20) // (B * D * 4) + 1)  # rotating inputs: 160 MB in total, over three times the 50 MB L2
    g = torch.Generator().manual_seed(1234 + rank)
    xs_host = [(torch.randn(B, D, generator=g) * 1.5).pin_memory() for _ in range(2)]
    xs = [(torch.randn(B, D, generator=g) * 1.5).to(dev) for _ in range(nbuf)]

    dp_mode = os.environ.get("NFB_BENCH_DP", "async")  # async | sync | none(debug: no collective)

    def step(i):
        if dp_mode == "none":
            return model.forward_kld(xs[i % nbuf])
        return forward_kld_dp(model, xs[i % nbuf], async_op=(dp_mode == "async"))

    def value_of(l):
        return l.result() if hasattr(l, "result") else l

    for i in range(warmup):
        loss = value_of(step(i))
    stack = model._stack()
    launches_per_step = stack.launch_count()
    fused = stack.fused_layers()
    assert len(fused) == 2 * LAYERS, "flagship stack must run on the fused tensor-core kernel"
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    sampler = ClockSampler(local)
    sampler.start()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record()
    t_host0 = time.perf_counter()
    for i in range(steps):
        loss = step(i)
    loss = value_of(loss)  # stream-waits for the last collective; every step's loss was reduced on device
    host_enqueue_ms = (time.perf_counter() - t_host0) * 1e3 / steps  # CPU time to enqueue one step
    ev1.record()
    torch.cuda.synchronize()
    elapsed_ms = ev0.elapsed_time(ev1)
    if world > 1:
        dist.barrier()
        t = torch.tensor([elapsed_ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        elapsed_ms = float(t)
    loss_val = float(loss)
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "forward_kld.npy"), np.array([loss_val], dtype=np.float64))

    # ---- e2e through the host-buffer C-ABI entry point (H2D + kernels + D2H each step) ----
    for i in range(3):
        model.forward_kld_host(xs_host[i % 2], dev)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    for i in range(steps):
        e2e_loss = model.forward_kld_host(xs_host[i % 2], dev)  # synchronous: returns the host float
    e2e_s = time.perf_counter() - t0
    if args.dump_outputs and rank == 0:
        np.save(os.path.join(args.dump_outputs, "forward_kld_host.npy"), np.array([float(e2e_loss)], dtype=np.float64))
    if world > 1:
        t = torch.tensor([e2e_s], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        e2e_s = float(t)
    clocks = sampler.stop()

    # ---- roofline of the dominant kernel (fused spline block), timed live with CUDA events ----
    roof = None
    if rank == 0:
        import ctypes as C
        from normflows import _lib as L
        # The dominant kernel is the persistent whole-stack launch (all 32 [LU + spline block] pairs, one
        # kernel): time it alone, back to back, inputs rotating as above.
        h = stack._h
        n_l = 10
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        outs = [torch.empty_like(xs[0]) for _ in range(2)]
        ld = torch.zeros(B, device=dev)
        for i in range(2):
            L.check(L.lib().nfb_flow_transform(h, L.NFB_INVERSE, L.ptr(xs[i % nbuf]), L.ptr(outs[i % 2]), L.ptr(ld),
                                               B, L.stream_ptr()))
        torch.cuda.synchronize()
        e0.record()
        for i in range(n_l):
            L.check(L.lib().nfb_flow_transform(h, L.NFB_INVERSE, L.ptr(xs[i % nbuf]), L.ptr(outs[i % 2]), L.ptr(ld),
                                               B, L.stream_ptr()))
        e1.record()
        torch.cuda.synchronize()
        k_ms = e0.elapsed_time(e1) / n_l  # includes a 65 K-element fill and a 2 KB memset (~4 us)
        # NVIDIA's data sheet for the H100 SXM: 989 TFLOP/s dense FP16 (700 W card).  A data-sheet rate, not a measured
        # one: `clocks` shows the SM clock the run actually had.
        peak = 989.0
        flops = FLOPS_PER_SAMPLE_LAYER[KIND] * B * LAYERS
        achieved = flops / (k_ms * 1e-3) / 1e12
        roof = {"kernel": "nfb::fused_rqs_kernel, whole stack in one persistent launch: 32 x (LULinearPermute + MADE "
                          "conditioner + RQ spline + log-det), (layer, tile) work units",
                "bound": "tensor", "achieved": achieved, "peak": peak, "unit": "TFLOP/s", "frac": achieved / peak,
                "kernel_ms": k_ms, "peak_source": "H100 SXM data sheet, dense FP16",
                "note": "algorithmic = dense fp32-equivalent GEMM flops of the reference (1.327 MFLOP/sample/layer x 32 "
                        "layers, SURVEY 8d).  The kernel runs every product as 3 fp16 tensor-core passes (split "
                        "precision with power-of-two operand scaling, needed for the rtol 1e-4 bar) so frac <= 1/3 by "
                        "construction, and skips the all-zero [64 x 64] blocks of the MADE masks"}

    # ---- training step (extra key; every rank takes part): forward_kld + native backward (tensor-core dgrad /
    # wgrad, analytic spline adjoint) + DDP-style bucketed gradient all-reduce (NCCL when world > 1) + Adam step.
    # The optimizer step invalidates the packed weights, so each timed step includes the device-side repack. ----
    train = None
    if not args.no_train_step:
        from normflows.parallel import GradientBuckets
        try:
            torch.set_grad_enabled(True)
            params = list(model.parameters())
            opt = torch.optim.Adam(params, lr=1e-6)
            buckets = GradientBuckets(params)

            def tstep(i):
                opt.zero_grad(set_to_none=True)
                l = model.forward_kld(xs[i % nbuf])
                l.backward()
                buckets.start(B).finish()
                opt.step()
                return l
            for i in range(2):
                tl = tstep(i)
            torch.cuda.synchronize()
            if world > 1:
                dist.barrier()
            t0e, t1e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n_t = 5
            t0e.record()
            for i in range(n_t):
                tl = tstep(i)
            t1e.record()
            torch.cuda.synchronize()
            t_ms = t0e.elapsed_time(t1e) / n_t
            if world > 1:
                tt = torch.tensor([t_ms], device=dev)
                dist.all_reduce(tt, op=dist.ReduceOp.MAX)
                t_ms = float(tt)
            train = {"ms_per_step": t_ms, "value": world * B / (t_ms * 1e-3), "unit": "samples/s", "loss": float(tl.detach()),
                     "what": "forward_kld + loss.backward() (libnfb200 nfb_flow_log_prob_backward) + bucketed gradient "
                             "all-reduce + Adam step + repack of the packed weights, batch %d/GPU, 2 warm-up + %d timed" % (B, n_t)}
        except Exception as e:  # an extra key must never take the headline down
            train = {"unavailable": repr(e)[:300]}
        finally:
            torch.set_grad_enabled(False)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    value = world * B * steps / (elapsed_ms * 1e-3)
    e2e_value = world * B * steps / e2e_s
    line = {"metric": METRIC, "value": value,
            "unit": "samples/s", "n_gpus": world, "steps": steps, "warmup": warmup,
            "ms_per_step": elapsed_ms / steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "f32", "data": "synthetic",
            "config": {"workload": workload_name(B),
                       "global_batch": world * B, "parallelism": f"dp{world}", "dp_collective": dp_mode,
                       "l2_policy": f"{nbuf} rotating input batches ({nbuf * B * D * 4 >> 20} MiB > L2)",
                       "loss": loss_val},
            "e2e": {"value": e2e_value, "unit": "samples/s", "h2d_bytes_per_step": B * D * 4,
                    "d2h_bytes_per_step": 4, "ms_per_step": e2e_s / steps * 1e3, "loss": e2e_loss,
                    "api": "nfb_flow_forward_kld_host (pinned host batch; chunked H2D overlapped with the kernel)"
                           + ("" if world == 1 else "; at N > 1 every rank calls it on its own shard and no collective is "
                              "included (throughput of N independent host calls, not forward_kld_dp end to end)")},
            "host_enqueue_ms_per_step": host_enqueue_ms,
            "gpu_launches": launches_per_step * steps, "gpu_launches_per_step": launches_per_step,
            "clocks": clocks, "roofline": roof, "train_step": train}
    if world == 1 and not args.no_extra_configs:
        # the other BASELINE configurations (parity-test cases, not bench lines), as `extra` keys: C1 Real NVP,
        # C2' coupled variant, C3 Glow, C5 residual flow -- tools/bench_configs.py, in a subprocess (fresh model state)
        try:
            out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_configs.py")], capture_output=True,
                                 text=True, timeout=900)
            line["extra"] = [json.loads(ln) for ln in out.stdout.splitlines() if ln.startswith("{")]
        except Exception as e:
            line["extra"] = {"unavailable": repr(e)[:200]}
    if world == 1 and reference_available() and not args.no_reference_eager:
        # the denominator of north_star's >= 10x target: the unmodified reference, PyTorch eager, same GPU
        try:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--impl", "reference-eager",
                                  "--steps", "50", "--batch", str(B)], capture_output=True, text=True, timeout=600)
            ref = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
            line["reference_eager"] = {
                "value": ref["value"], "unit": "samples/s", "ms_per_step": ref["ms_per_step_median"],
                "loss": ref["loss"], "how": "oracle/_ref/normflows (unmodified) model.forward_kld under no_grad on "
                "cuda:0, same model/seed/batch, 10 warm-up + 50 timed passes, CUDA events, median",
                "speedup_device": value / ref["value"], "speedup_e2e": e2e_value / ref["value"], "target": 10.0}
        except Exception as e:  # reported, never fatal
            line["reference_eager"] = {"unavailable": repr(e)[:200]}
    if not args.no_cpu_baseline and world == 1:  # reported baseline: rank 0 at N = 1 only
        line["cpu_baseline"], _ = cpu_baseline()
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
