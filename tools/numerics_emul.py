"""Offline numerics study (CPU, numpy/torch): emulate the fused kernel's split-precision GEMMs inside the fp64 oracle
and measure the log_prob error of the 32-layer bench model on chosen rows.  Everything except the conditioner GEMMs
stays in fp64, so the numbers isolate the operand-split error of each candidate scheme.
    python tools/numerics_emul.py [row_lo row_hi]
"""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
import numpy as np, torch, bench
from oracle import nf_oracle as O

def rnd(x, dt):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dt).to(torch.float64).numpy()

def split(x, dt, n=2, scale=1.0):
    parts, rem = [], np.asarray(x, dtype=np.float32).astype(np.float64) * scale
    for _ in range(n):
        p = rnd(rem, dt)
        parts.append(p)
        rem = rem - p
    return parts

SCHEME = {"name": "fp64"}
def emu_linear(x, w, b=None):
    s = SCHEME["name"]
    x32 = np.asarray(x, dtype=np.float32).astype(np.float64)   # activations are fp32 in the kernel
    if s == "fp64":
        y = x @ w.T
    elif s == "fp32in":
        y = x32 @ w.T
    elif s in ("bf16x3", "bf16x4", "fp16x3", "fp16x3s"):
        dt = torch.bfloat16 if s.startswith("bf16") else torch.float16
        sa = sw = 1.0
        if s == "fp16x3s":   # power-of-two scales that centre the operands in fp16's range
            sw = 2.0 ** (13 - np.ceil(np.log2(np.abs(w).max() + 1e-30)))
            sa = 2.0 ** (10 - np.ceil(np.log2(np.abs(x32).max(axis=1, keepdims=True) + 1e-30)))   # per-row exponent
        ah, al = split(x32 * sa, dt)
        wh, wl = split(w, dt, scale=sw)
        y = ah @ wh.T + al @ wh.T + ah @ wl.T
        if s == "bf16x4":
            y = y + al @ wl.T
        y = y / (sa * sw)
    if b is not None:
        y = y + b
    return y

O.linear = emu_linear

def main():
    lo, hi = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (6800, 7056)
    kind = "ar"
    model = bench.build_model(kind)
    sd = {k: v.detach().numpy() for k, v in model.state_dict().items()}
    spec = bench.oracle_spec(kind)
    x = (torch.randn(65536 + 77, 64, generator=torch.Generator().manual_seed(1234)) * 1.5).numpy().astype(np.float64)[lo:hi]
    SCHEME["name"] = "fp64"
    truth = O.log_prob(spec, sd, x)
    for s in ("fp32in", "bf16x3", "bf16x4", "fp16x3", "fp16x3s"):
        SCHEME["name"] = s
        lp = O.log_prob(spec, sd, x)
        rel = np.abs(lp - truth) / np.abs(truth)
        w = np.argsort(rel)[-3:][::-1]
        print(f"{s:8s} rel max {rel.max():.2e} p99 {np.quantile(rel,.99):.2e} median {np.median(rel):.2e}  worst rows {[(int(lo+i), float('%.2e'%rel[i])) for i in w]}", flush=True)
    # the reference's own fp32 arithmetic on the same rows (oracle in float32 == reference fp32 to ~1e-6)
    SCHEME["name"] = "fp64"
    O.linear = lambda x, w, b=None: (x @ w.T + b) if b is not None else x @ w.T
    lp32 = O.log_prob(spec, sd, x.astype(np.float32)).astype(np.float64)
    rel = np.abs(lp32 - truth) / np.abs(truth)
    print(f"oracle-fp32 rel max {rel.max():.2e} p99 {np.quantile(rel,.99):.2e} median {np.median(rel):.2e}; row 6927: {rel[6927-lo] if lo <= 6927 < hi else None}")

if __name__ == "__main__":
    main()
