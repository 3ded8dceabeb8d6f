#!/usr/bin/env python
"""Where a (layer, 64-row tile) unit of the fused spline kernel spends its cycles, per role.

    make -C normalizing-flows_b200/csrc CLOCKS=1 OUT=../libnfb200_clocks.so
    NFB200_LIB=normalizing-flows_b200/libnfb200_clocks.so python tools/fused_phase_clocks.py [--passes 5]

The CLOCKS=1 build of the library stamps the SM clock between the phases of `nfb::fused_rqs_kernel` (csrc/nfb_fused_rqs.cu,
NFB_PHASE_CLOCKS) and sums the differences per role.  This tool runs warmed `forward_kld` passes of the flagship stack
(bench.build_model) at the bench batch and prints the cycles per unit of every phase: mean over all units, for each
consumer warpgroup and for the producer warp.  The stamps cost time themselves, so the sum per unit is somewhat above the
product kernel's.  The card's name, power limit and SM clock are read with a read-only nvidia-smi query.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]

PHASES = ["claim / dependency wait", "tile load, row units, first A operand", "LU stage", "hidden: ring wait",
          "hidden: wgmma issue -> complete", "hidden: epilogues + barriers", "final: ring wait",
          "final: wgmma issue -> complete", "final: pair tail (wait for a pair's last products)",
          "final: staging + barriers", "final: spline", "log-det, store, publish", "producer: empty-slot wait",
          "producer: other"]
ROLES = ["warpgroup 0", "warpgroup 1", "producer"]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), (s.strip() for s in out.split(","))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=5)
    ap.add_argument("--kind", default="ar", choices=["ar", "coupled"])
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("fused_phase_clocks: no CUDA device; the phase clocks are read on the GPU")
    import bench
    from normflows import _lib
    lib = _lib.lib()
    try:
        read = lib.nfb_phase_clocks_read
    except AttributeError:
        raise SystemExit(f"fused_phase_clocks: {_lib.LIB_PATH} has no phase clocks; build it with `make CLOCKS=1 "
                         "OUT=../libnfb200_clocks.so` and select it with NFB200_LIB")
    read.argtypes, read.restype = [C.c_void_p, C.c_int], C.c_int
    phases = PHASES
    try:
        n = lib.nfb_phase_clocks_count()
    except AttributeError:   # a build from before the pair-tail phase: its pair tails are inside issue -> complete
        phases = [p for p in PHASES if not p.startswith("final: pair tail")]
        n = len(phases) + 1
    assert n == len(phases) + 1, f"{_lib.LIB_PATH}: {n - 1} phases, this tool knows {len(phases)}"
    torch.set_grad_enabled(False)
    model = bench.build_model(args.kind).cuda()
    x = (torch.randn(bench.BATCH, bench.D, generator=torch.Generator().manual_seed(1)) * 1.5).cuda()
    for _ in range(3):
        model.forward_kld(x)
    assert read(None, 1) == 0
    during = None
    for i in range(args.passes):
        model.forward_kld(x)
        if i == args.passes // 2:
            during = gpu_info()   # while the queue is busy: the SM clock under load
    buf = ((C.c_ulonglong * n) * 3)()
    assert read(C.byref(buf), 1) == 0
    print("gpu:", during)
    print(f"{args.kind} stack, batch {bench.BATCH}, {args.passes} passes; SM cycles per unit")
    units = [buf[r][n - 1] for r in range(3)]
    print(f"{'phase':50s}" + "".join(f"{r:>14s}" for r in ROLES))
    for ph, name in enumerate(phases):
        print(f"{name:50s}" + "".join(f"{buf[r][ph] / max(1, units[r]):14.0f}" for r in range(3)))
    print(f"{'sum':50s}" + "".join(f"{sum(buf[r][:n - 1]) / max(1, units[r]):14.0f}" for r in range(3)))
    print(f"{'units':50s}" + "".join(f"{units[r]:14d}" for r in range(3)))


if __name__ == "__main__":
    main()
