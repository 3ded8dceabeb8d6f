#!/usr/bin/env python
"""Same-box A/B of two builds of libnfb200.so on the flagship workload (bench.py), with a bit-for-bit output check.

    python tools/ab_fused_stack.py --base-lib OTHER/libnfb200.so --out DIR [--rounds 5]

The base build is loaded through NFB200_LIB; the new build is the in-tree library.  Each round runs

    bench.py --steps 50 --warmup 5 --no-cpu-baseline --no-reference-eager --no-extra-configs --no-train-step
             --dump-outputs DIR

once per build, alternating the order from round to round, and collects `value`, `roofline.kernel_ms`, `ms_per_step`
and `clocks`.  The forward_kld / forward_kld_host dumps of every run must be bit-identical between the builds.  Then,
in a child process per build, the per-row log_prob of the bench model on one seeded batch and the sampling-direction
output of a seeded 4-layer autoregressive stack are dumped and compared bit for bit (a scalar loss can hide a per-row
difference).  The card's name, power limit and max SM clock are read with a read-only nvidia-smi query.  Everything
goes to DIR/ab.json; the summary is printed.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BENCH_ARGS = ["--steps", "50", "--warmup", "5", "--no-cpu-baseline", "--no-reference-eager", "--no-extra-configs",
              "--no-train-step"]


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
            "clocks": res.get("clocks")}


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
                  f"value {res['value']:.0f} sm_mhz {res['clocks'] and res['clocks'].get('sm_mhz')}", flush=True)
    for f in ("forward_kld.npy", "forward_kld_host.npy"):
        ref = os.path.join(args.out, "base_0", f)
        report["identical"][f] = all(same_bits(ref, os.path.join(args.out, f"{n}_{r}", f))
                                     for n in builds for r in range(args.rounds))
    for name, lib in builds.items():
        subprocess.run([sys.executable, os.path.abspath(__file__), "--dump-rows", "--out",
                        os.path.join(args.out, f"rows_{name}")], cwd=ROOT, env=env_for(lib), check=True)
    for f in ("log_prob.npy", "sample_x.npy", "sample_logdet.npy"):
        report["identical"][f] = same_bits(os.path.join(args.out, "rows_base", f), os.path.join(args.out, "rows_new", f))

    km = {n: [x["kernel_ms"] for x in report["runs"][n]] for n in builds}
    ms = {n: [x["ms_per_step"] for x in report["runs"][n]] for n in builds}
    report["summary"] = {
        "kernel_ms_median": {n: statistics.median(km[n]) for n in builds},
        "kernel_ms_range": {n: [min(km[n]), max(km[n])] for n in builds},
        "ms_per_step_median": {n: statistics.median(ms[n]) for n in builds},
        "kernel_speedup_median": statistics.median(km["base"]) / statistics.median(km["new"]),
        "slowest_new_beats_fastest_base": max(km["new"]) < min(km["base"]),
    }
    with open(os.path.join(args.out, "ab.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    print(json.dumps({"gpu": report["gpu"], "identical": report["identical"], "summary": report["summary"]}, indent=1))
    if not all(report["identical"].values()):
        raise SystemExit("outputs differ between the builds")


if __name__ == "__main__":
    main()
