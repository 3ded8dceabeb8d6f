"""Offline emulation of the PLANNED fp16-split numerics of the fused kernel (per-row power-of-two unit u = 2^-e_r from
the row's input magnitude, static per-GEMM power-of-two scales from guaranteed infinity-norm bounds, 3-term 2-way
fp16 split for conditioner GEMMs, 4-term for the LU map), inside the fp64 oracle.  CPU only."""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "normalizing-flows_b200")]
import numpy as np, torch, bench
from oracle import nf_oracle as O

def f16(x):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.float16).to(torch.float64).numpy()
def split16(x):
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    hi = f16(x); lo = f16(x - hi)
    return hi, lo
def cl2(v):
    return int(np.ceil(np.log2(max(float(v), 1e-30))))

STATS = {"amax": [], "amed": []}
def gemm(a_true, u, w, pa, pw, four=False):
    """a_true [B,K] fp32-valued, u [B,1] row unit; returns the true-scale product W a (fp64 accumulate)."""
    a = np.asarray(a_true, dtype=np.float32).astype(np.float64) * u * 2.0 ** pa
    assert np.abs(a).max() < 65504, ("A overflow", np.abs(a).max())
    STATS["amax"].append(np.abs(a).max()); STATS["amed"].append(np.median(np.abs(a[a != 0])))
    ah, al = split16(a)
    wh, wl = split16(w * 2.0 ** pw)
    assert np.abs(w).max() * 2.0 ** pw < 65504
    y = ah @ wh.T + al @ wh.T + ah @ wl.T
    if four:
        y = y + al @ wl.T
    return y / (u * 2.0 ** (pa + pw))

def plan(norms, bmaxs, b_in0):
    """-> per-GEMM (pa, pw) from guaranteed bounds; norms[g] = (max row L1, max abs) of the effective matrix."""
    n = len(norms)
    bounds_in = [b_in0]
    B_h = norms[0][0] * b_in0 + bmaxs[0]
    g = 1
    while g + 1 < n - 1 + 1 and g + 1 <= n - 2:   # blocks: (g, g+1)
        bounds_in.append(B_h)
        B_t = norms[g][0] * B_h + bmaxs[g]
        bounds_in.append(B_t)
        B_h = B_h + norms[g + 1][0] * B_t + bmaxs[g + 1]
        g += 2
    bounds_in.append(B_h)  # final layer input
    pa = [14 - cl2(b) for b in bounds_in]
    pw = [13 - cl2(nm[1]) for nm in norms]
    # GEMMs that accumulate onto the residual stream (0, 2, 4, ...) share pa + pw
    hs = [0] + list(range(2, n - 1, 2))
    P = min(pa[i] + pw[i] for i in hs)
    for i in hs:
        d = pa[i] + pw[i] - P
        pw[i] -= d   # (lower the weight scale first; 10+ binades of slack there)
    return pa, pw, bounds_in

def made_emul(x, u, sd, p, b_in0):
    names = [p + "initial_layer."]
    nb = O._num_blocks(sd, p)
    for i in range(nb):
        names += [f"{p}blocks.{i}.linear_layers.0.", f"{p}blocks.{i}.linear_layers.1."]
    names.append(p + "final_layer.")
    W = [sd[q + "weight"] * sd[q + "mask"] for q in names]
    b = [sd[q + "bias"] for q in names]
    # input of GEMMs 1..n-2 is post-ReLU (>= 0): |W a| <= max(sum w+, sum w-) |a|_inf  (tighter than the L1 norm)
    def rown(w, nonneg):
        if nonneg:
            return max(np.maximum(w, 0).sum(axis=1).max(), np.maximum(-w, 0).sum(axis=1).max())
        return np.abs(w).sum(axis=1).max()
    norms = [(rown(w, 0 < g < len(W) - 1), np.abs(w).max()) for g, w in enumerate(W)]
    pa, pw, bounds = plan(norms, [np.abs(v).max() for v in b], b_in0)
    h = gemm(x, u, W[0], pa[0], pw[0]) + b[0]
    for i in range(nb):
        t = gemm(np.maximum(h, 0), u, W[1 + 2 * i], pa[1 + 2 * i], pw[1 + 2 * i]) + b[1 + 2 * i]
        h = h + gemm(np.maximum(t, 0), u, W[2 + 2 * i], pa[2 + 2 * i], pw[2 + 2 * i]) + b[2 + 2 * i]
    return gemm(h, u, W[-1], pa[-1], pw[-1]) + b[-1], (pa, pw, bounds)

def log_prob_emul(spec, sd, x, verbose=False):
    z = x.copy(); lq = np.zeros(len(x))
    n = len(spec["flows"])
    i = n - 1
    while i >= 0:
        L = spec["flows"][i]
        if L["type"] == "LULinearPermute":   # unit = LU map then the spline block before it in list order
            zmax = np.abs(z).max(axis=1, keepdims=True)
            e = np.clip(np.ceil(np.log2(np.maximum(zmax, 1e-30))), 0, 40)
            u = 2.0 ** -e
            lower, upper, diag = O.lu_matrices(sd, f"flows.{i}.", np.float64)
            Wm = (lower @ upper)
            perm = sd[f"flows.{i}.permutation._permutation"]
            zp = z[:, perm]
            n_lu = np.abs(Wm).sum(axis=1).max()
            pa, pw = 14, 13 - cl2(np.abs(Wm).max())
            z = gemm(zp, u, Wm, pa, pw, four=True) + sd[f"flows.{i}.linear.bias"]
            lq += np.sum(np.log(diag))
            b_in0 = n_lu + np.abs(sd[f"flows.{i}.linear.bias"]).max()
            i -= 1
            L = spec["flows"][i]
        else:
            zmax = np.abs(z).max(axis=1, keepdims=True)
            u = 2.0 ** -np.clip(np.ceil(np.log2(np.maximum(zmax, 1e-30))), 0, 40)
            b_in0 = 1.0
        assert L["type"] == "AutoregressiveRationalQuadraticSpline"
        p = f"flows.{i}.mprqat.autoregressive_net."
        params, info = made_emul(z, u, sd, p, b_in0)
        if verbose and i >= n - 3:
            print("layer", i, "pa", info[0], "pw", info[1], "bounds", ["%.1f" % b for b in info[2]])
        params = params.reshape(len(z), 64, 23)
        uw, uh, ud = O._split_params(params, 8, None)
        z, lad = O.unconstrained_rqs(z, uw, uh, ud, inverse=False, tail_bound=3.0)
        lq += lad.sum(axis=1)
        i -= 1
    return lq + O.diag_gaussian_log_prob(z, sd, "q0.")

def main():
    lo, hi = (int(sys.argv[1]), int(sys.argv[2])) if len(sys.argv) > 2 else (6800, 7056)
    model = bench.build_model("ar")
    sd = {k: v.detach().numpy().astype(np.float64) if v.dtype.is_floating_point else v.numpy() for k, v in model.state_dict().items()}
    spec = bench.oracle_spec("ar")
    x = (torch.randn(65536 + 77, 64, generator=torch.Generator().manual_seed(1234)) * 1.5).numpy().astype(np.float64)[lo:hi]
    truth = O.log_prob(spec, sd, x)
    lp = log_prob_emul(spec, sd, x, verbose=True)
    rel = np.abs(lp - truth) / np.abs(truth)
    w = np.argsort(rel)[-3:][::-1]
    print(f"fp16 planned scheme: rel max {rel.max():.2e} p99 {np.quantile(rel,.99):.2e} median {np.median(rel):.2e} worst {[(int(lo+i), float('%.2e'%rel[i])) for i in w]}")
    print("scaled A operand: max over GEMMs %.3g, median-of-medians %.3g, min median %.3g" % (max(STATS["amax"]), np.median(STATS["amed"]), min(STATS["amed"])))
    # robustness: a row with absurd inputs must stay finite
    xb = x[:4].copy(); xb[0, 0] = 1e6; xb[1, 3] = -3e4; xb[2] *= 1e-6
    lpb = log_prob_emul(spec, sd, xb); tb = O.log_prob(spec, sd, xb)
    print("absurd rows: emul", lpb, "truth", tb)

if __name__ == "__main__":
    main()
