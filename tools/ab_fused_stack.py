#!/usr/bin/env python
"""Same-box A/B of two builds of libnfb200.so on the flagship workload (bench.py), with a bit-for-bit output check.

    python tools/ab_fused_stack.py --base-lib OTHER/libnfb200.so --out DIR [--rounds 5]

The base build is loaded through NFB200_LIB; the new build is the in-tree library.  Each round runs

    bench.py --steps 50 --warmup 5 --no-cpu-baseline --no-reference-eager --no-extra-configs --dump-outputs DIR

once per build, alternating the order from round to round, and collects `value`, `roofline.kernel_ms`, `ms_per_step`,
`train_step.ms_per_step` and `clocks`.  The forward_kld / forward_kld_host dumps of every run must be bit-identical
between the builds.  Then, in three child processes per build, the per-row log_prob of the bench model on one seeded
batch and the sampling-direction output of a seeded 4-layer autoregressive stack are dumped and compared bit for bit (a
scalar loss can hide a per-row difference), together with gradients: one forward_kld(x).backward() of the bench model
(`ar` and `coupled`, x.grad, every parameter gradient and launch_count()) and the stand-alone conditioner backward
(ResidualNet / MADE, with and without a context), MaskedAffineAutoregressive.inverse and the autoregressive spline
layers' sampling direction (with and without periodic features).  Split-K weight gradients and shared-table spline
gradients are reduced with atomics, so a gradient the base build does not reproduce bit for bit between its own runs
is set against that run-to-run difference instead (compare_grads).  The card's name, power limit and max SM clock are read with a
read-only nvidia-smi query.  Everything goes to DIR/ab.json; the summary is printed.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH_ARGS = ["--steps", "50", "--warmup", "5", "--no-cpu-baseline", "--no-reference-eager", "--no-extra-configs"]


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), (s.strip() for s in out.split(","))))


def env_for(lib):
    env = dict(os.environ)
    env.pop("NFB200_LIB", None)
    if lib:
        env["NFB200_LIB"] = lib
    return env


def run_bench(lib, dump):
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + BENCH_ARGS + ["--dump-outputs", dump],
                       cwd=ROOT, env=env_for(lib), capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise SystemExit(f"bench.py failed ({p.returncode}) with NFB200_LIB={lib}")
    res = None
    for line in p.stdout.splitlines():
        line = line.strip()
        if line.startswith("{"):
            try:
                res = json.loads(line)
            except ValueError:
                pass
    if res is None:
        raise SystemExit("bench.py printed no JSON result line")
    return {"value": res["value"], "kernel_ms": res["roofline"]["kernel_ms"], "ms_per_step": res["ms_per_step"],
            "train_ms": res["train_step"]["ms_per_step"], "clocks": res.get("clocks")}


def dump_rows(out):
    """Child process: per-row outputs of the library NFB200_LIB selects, on seeded inputs."""
    sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
    import numpy as np
    import torch
    import bench
    torch.set_grad_enabled(False)
    os.makedirs(out, exist_ok=True)
    model = bench.build_model("ar").cuda()
    x = (torch.randn(bench.BATCH + 37, bench.D, generator=torch.Generator().manual_seed(4321)) * 1.5).cuda()
    np.save(os.path.join(out, "log_prob.npy"), model.log_prob(x).cpu().numpy())
    assert model._stack().fused_layers() == list(range(2 * bench.LAYERS))
    small = bench.build_model("ar", layers=4, seed=5).cuda()
    z = torch.randn(4096 + 37, bench.D, generator=torch.Generator().manual_seed(99)).cuda()
    xs, ld = small.forward_and_log_det(z)
    np.save(os.path.join(out, "sample_x.npy"), xs.cpu().numpy())
    np.save(os.path.join(out, "sample_logdet.npy"), ld.cpu().numpy())
    dump_grads(out, x)


def dump_grads(out, x):
    """Gradients of every native backward that runs on the shared ResidualNet / MADE backward, on seeded inputs."""
    import numpy as np
    import torch
    import bench
    import normflows as nf
    from normflows.nets import MADE, ResidualNet
    torch.set_grad_enabled(True)
    grads, launches = {}, {}

    def run(name, module, f, *inputs):
        module.zero_grad(set_to_none=True)
        ins = [t.cuda().requires_grad_(True) if t is not None else None for t in inputs]
        outs = f(*ins)
        g = torch.Generator().manual_seed(17)
        sum((o * torch.randn(o.shape, generator=g).cuda()).sum() for o in outs).backward()
        for i, t in enumerate(ins):
            if t is not None:
                grads[f"{name}/in{i}"] = t.grad
        for k, p in module.named_parameters():
            if p.grad is not None:
                grads[f"{name}/{k}"] = p.grad

    for kind in ("ar", "coupled"):
        model = bench.build_model(kind).cuda()
        model.zero_grad(set_to_none=True)
        xg = x.clone().requires_grad_(True)
        model.forward_kld(xg).backward()
        launches[kind] = model._stack().launch_count()
        grads[f"{kind}/x"] = xg.grad
        for k, p in model.named_parameters():
            if p.grad is not None:
                grads[f"{kind}/{k}"] = p.grad
    g = torch.Generator().manual_seed(23)
    rows = 1061
    for ctx in (False, True):
        cf = 5 if ctx else None
        c = torch.randn(rows, 5, generator=g) if ctx else None
        torch.manual_seed(3)
        for name, net, din in ((f"resnet_ctx{int(ctx)}", ResidualNet(3, 7, 64, cf, 2), 3),
                               (f"made_ctx{int(ctx)}", MADE(4, 64, cf, 2, output_multiplier=3), 4)):
            net = net.cuda()
            run(name, net, lambda a, b: [net(a, b)], torch.randn(rows, din, generator=g), c)
        torch.manual_seed(5)
        maf = nf.flows.MaskedAffineAutoregressive(5, 64, context_features=3 if ctx else None, num_blocks=2).cuda()
        c3 = torch.randn(rows, 3, generator=g) if ctx else None
        run(f"maf_ctx{int(ctx)}", maf, lambda a, b: list(maf.inverse(a, b)), torch.randn(rows, 5, generator=g), c3)
    torch.manual_seed(7)
    ar = nf.flows.AutoregressiveRationalQuadraticSpline(5, 2, 48, num_context_channels=3, num_bins=8, tail_bound=2.5,
                                                        permute_mask=True).cuda()
    run("ar_sampling", ar, lambda a, b: list(ar(a, b)), torch.randn(rows, 5, generator=g) * 1.2,
        torch.randn(rows, 3, generator=g))
    car = nf.flows.CircularAutoregressiveRationalQuadraticSpline(5, 2, 48, [1, 3], num_bins=8,
                                                                 tail_bound=torch.tensor([2.5, 3., 3.5, 4., 4.5])).cuda()
    run("ar_sampling_periodic", car, lambda a: list(car(a)), torch.randn(rows, 5, generator=g) * 1.2)
    np.savez(os.path.join(out, "grads.npz"), **{k: v.detach().cpu().numpy() for k, v in grads.items()})
    with open(os.path.join(out, "launches.json"), "w") as fh:
        json.dump(launches, fh)


DUMP_RUNS = 3


def compare_grads(out, builds):
    """Gradients the base build reproduces bit for bit must be bit-identical in every new run.  For the others, d_new
    (largest |new run 0 - base run j| over the base runs) is set against d_base (largest difference between two base
    runs): both are maxima of the same atomic-reduction noise over as many pairs, so for an unchanged computation
    either is the larger about equally often, and a systematic change shows as d_new >> d_base."""
    import numpy as np
    runs = {name: [np.load(os.path.join(out, f"rows_{name}_{i}", "grads.npz")) for i in range(DUMP_RUNS)]
            for name in builds}
    base, new = runs["base"], runs["new"]
    assert all(sorted(r.files) == sorted(base[0].files) for rs in runs.values() for r in rs), "different gradient sets"
    rep = {"compared": 0, "bit_identical": 0, "base_nondeterministic": 0, "new_larger": 0, "new_equal": 0,
           "new_smaller": 0, "worst_ratio": 0.0, "failed": []}
    for k in base[0].files:
        rep["compared"] += 1
        b = [r[k] for r in base]
        n = [r[k] for r in new]
        if all(x.tobytes() == b[0].tobytes() for x in b):
            if all(x.tobytes() == b[0].tobytes() for x in n):
                rep["bit_identical"] += 1
            else:
                rep["failed"].append(k)
            continue
        rep["base_nondeterministic"] += 1
        d_base = max(float(np.abs(b[i] - b[j]).max()) for i in range(len(b)) for j in range(i))
        d_new = max(float(np.abs(n[0] - x).max()) for x in b)
        rep["new_larger" if d_new > d_base else "new_equal" if d_new == d_base else "new_smaller"] += 1
        rep["worst_ratio"] = max(rep["worst_ratio"], d_new / d_base)
    rep["launches"] = {name: [json.load(open(os.path.join(out, f"rows_{name}_{i}", "launches.json")))
                              for i in range(DUMP_RUNS)] for name in builds}
    rep["launches_equal"] = all(v == rep["launches"]["base"][0] for vs in rep["launches"].values() for v in vs)
    return rep


def same_bits(a, b):
    import numpy as np
    a, b = np.load(a), np.load(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base-lib", help="the other build of libnfb200.so (A)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--dump-rows", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.dump_rows:
        return dump_rows(args.out)
    base = os.path.abspath(args.base_lib)
    assert os.path.exists(base), base
    os.makedirs(args.out, exist_ok=True)
    builds = {"base": base, "new": None}
    report = {"gpu": gpu_info(), "runs": {"base": [], "new": []}, "identical": {}}
    print("gpu:", report["gpu"], flush=True)

    for r in range(args.rounds):
        order = ["base", "new"] if r % 2 == 0 else ["new", "base"]
        for name in order:
            d = os.path.join(args.out, f"{name}_{r}")
            res = run_bench(builds[name], d)
            report["runs"][name].append(res)
            print(f"round {r} {name}: kernel_ms {res['kernel_ms']:.3f} ms_per_step {res['ms_per_step']:.3f} "
                  f"train_ms {res['train_ms']:.3f} value {res['value']:.0f} sm_mhz {res['clocks'] and res['clocks'].get('sm_mhz')}", flush=True)
    for f in ("forward_kld.npy", "forward_kld_host.npy"):
        ref = os.path.join(args.out, "base_0", f)
        report["identical"][f] = all(same_bits(ref, os.path.join(args.out, f"{n}_{r}", f))
                                     for n in builds for r in range(args.rounds))
    for i in range(DUMP_RUNS):
        for name, lib in builds.items():
            subprocess.run([sys.executable, os.path.abspath(__file__), "--dump-rows", "--out",
                            os.path.join(args.out, f"rows_{name}_{i}")], cwd=ROOT, env=env_for(lib), check=True)
    for f in ("log_prob.npy", "sample_x.npy", "sample_logdet.npy"):
        report["identical"][f] = same_bits(os.path.join(args.out, "rows_base_0", f),
                                           os.path.join(args.out, "rows_new_0", f))
    report["grads"] = compare_grads(args.out, builds)
    report["identical"]["grads"] = not report["grads"]["failed"] and report["grads"]["launches_equal"]

    km = {n: [x["kernel_ms"] for x in report["runs"][n]] for n in builds}
    ms = {n: [x["ms_per_step"] for x in report["runs"][n]] for n in builds}
    tm = {n: [x["train_ms"] for x in report["runs"][n]] for n in builds}
    report["summary"] = {
        "train_ms_median": {n: statistics.median(tm[n]) for n in builds},
        "train_ms_range": {n: [min(tm[n]), max(tm[n])] for n in builds},
        "kernel_ms_median": {n: statistics.median(km[n]) for n in builds},
        "kernel_ms_range": {n: [min(km[n]), max(km[n])] for n in builds},
        "ms_per_step_median": {n: statistics.median(ms[n]) for n in builds},
        "kernel_speedup_median": statistics.median(km["base"]) / statistics.median(km["new"]),
        "slowest_new_beats_fastest_base": max(km["new"]) < min(km["base"]),
    }
    with open(os.path.join(args.out, "ab.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"gpu": report["gpu"], "identical": report["identical"], "summary": report["summary"],
                      "grads": report["grads"]}, indent=1))
    if not all(report["identical"].values()):
        raise SystemExit("outputs differ between the builds")


if __name__ == "__main__":
    main()
