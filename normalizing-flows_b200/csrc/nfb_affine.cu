// nfb_affine.cu -- the affine family for low-dimensional flows (D <= 16), whole stack in ONE kernel.
//
// One thread per sample keeps z[D] and the running log-det in registers and walks the layer list:
//   MaskedAffineFlow      flows/affine/coupling.py:208-229   (s,t = MLPs on b*z; non-finite -> NaN)
//   AffineCouplingBlock   flows/affine/coupling.py:253-267 -> AffineCoupling :113-171
//   AffineConstFlow/ActNorm (after init)  flows/affine/coupling.py:38-54
//   Permute               flows/mixing.py:31-54
// HBM traffic per sample is D*4 bytes in, D*4 out (+4 for log_q) for the entire stack -- the
// reference launches ~26 ATen ops per layer (SURVEY 3.5).  MLP weights are read through the
// read-only path with warp-uniform addresses (broadcast).
#include "nfb_kernels.h"
#include "nfb_affine_bwd.cuh"

namespace nfb {

__device__ __forceinline__ void mlp_eval(const AffMlp& m, const float* in, float* out, float slope) {
    float a[kAffMaxW], b[kAffMaxW];
    const int n0 = m.sizes[0];
    for (int i = 0; i < n0; ++i) a[i] = in[i];
    float* cur = a;
    float* nxt = b;
    for (int l = 0; l < m.n_layers; ++l) {
        const int ni = m.sizes[l], no = m.sizes[l + 1];
        const float* w = m.w[l];
        const float* bias = m.b[l];
        const bool last = (l + 1 == m.n_layers);
        for (int o = 0; o < no; ++o) {
            float acc = __ldg(bias + o);
            for (int i = 0; i < ni; ++i) acc = fmaf(cur[i], __ldg(w + o * ni + i), acc);
            nxt[o] = last ? acc : (acc >= 0.f ? acc : acc * slope);
        }
        float* tmp = cur; cur = nxt; nxt = tmp;
    }
    const int no = m.sizes[m.n_layers];
    for (int o = 0; o < no; ++o) out[o] = cur[o];
}

// direction: 0 = "inverse" (density pass: ops applied last-to-first), 1 = "forward" (sampling)
__global__ void __launch_bounds__(128)
affine_stack_kernel(const AffineOp* __restrict__ ops, int n_ops, const float* __restrict__ zin,
                    float* __restrict__ zout, float* __restrict__ logq, long long rows, int d,
                    int accumulate, int direction) {
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= rows) return;
    float z[kAffMaxD];
    for (int j = 0; j < d; ++j) z[j] = zin[row * d + j];
    float ld = 0.f;
    for (int k = 0; k < n_ops; ++k) {
        const AffineOp& op = ops[direction ? k : (n_ops - 1 - k)];
        if (op.type == kOpMasked) {
            float zm[kAffMaxD], s[kAffMaxD], t[kAffMaxD];
            for (int j = 0; j < d; ++j) zm[j] = __ldg(op.p0 + j) * z[j];
            if (op.s.n_layers) mlp_eval(op.s, zm, s, op.slope); else for (int j = 0; j < d; ++j) s[j] = 0.f;
            if (op.t.n_layers) mlp_eval(op.t, zm, t, op.slope_t); else for (int j = 0; j < d; ++j) t[j] = 0.f;
            for (int j = 0; j < d; ++j) {
                const float b = __ldg(op.p0 + j);
                const float sj = isfinite(s[j]) ? s[j] : __int_as_float(0x7fc00000);
                const float tj = isfinite(t[j]) ? t[j] : __int_as_float(0x7fc00000);
                if (direction) {
                    z[j] = zm[j] + (1.f - b) * (z[j] * expf(sj) + tj);
                    ld += (1.f - b) * sj;
                } else {
                    z[j] = zm[j] + (1.f - b) * (z[j] - tj) * expf(-sj);
                    ld -= (1.f - b) * sj;
                }
            }
        } else if (op.type == kOpConst) {
            float ssum = 0.f;
            for (int j = 0; j < d; ++j) {
                const float s = __ldg(op.p0 + j), t = __ldg(op.p1 + j);
                z[j] = direction ? z[j] * expf(s) + t : (z[j] - t) * expf(-s);
                ssum += s;
            }
            ld += direction ? ssum : -ssum;
        } else if (op.type == kOpCoupling) {
            const int h = (d + 1) / 2;                 // torch.chunk(2): first chunk ceil(d/2)
            const bool inv_split = (op.flags >> 3) & 1;  // channel_inv: z1 is the SECOND chunk
            const int o1 = inv_split ? h : 0, n1 = inv_split ? d - h : h;
            const int o2 = inv_split ? 0 : h, n2 = d - n1;
            float param[2 * kAffMaxD];
            mlp_eval(op.s, z + o1, param, op.slope);
            if (!(op.flags & 1)) {
                for (int j = 0; j < n2; ++j) z[o2 + j] += direction ? param[j] : -param[j];
            } else {
                const int smap = (op.flags >> 1) & 3;
                for (int j = 0; j < n2; ++j) {
                    const float shift = param[2 * j], sc = param[2 * j + 1];
                    float& v = z[o2 + j];
                    if (smap == 0) {
                        if (direction) { v = v * expf(sc) + shift; ld += sc; }
                        else { v = (v - shift) * expf(-sc); ld -= sc; }
                    } else {
                        const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
                        const float lsg = logf(sg);
                        const bool div = (smap == 1) == (direction != 0);
                        if (direction) v = div ? v / sg + shift : v * sg + shift;
                        else v = div ? (v - shift) / sg : (v - shift) * sg;
                        ld += div ? -lsg : lsg;
                    }
                }
            }
        } else {  // permute
            const int* idx = direction ? op.fwd_idx : op.inv_idx;
            float tmp[kAffMaxD];
            for (int j = 0; j < d; ++j) tmp[j] = z[__ldg(idx + j)];
            for (int j = 0; j < d; ++j) z[j] = tmp[j];
        }
    }
    for (int j = 0; j < d; ++j) zout[row * d + j] = z[j];
    if (logq) logq[row] = accumulate ? logq[row] + ld : ld;
}

int launch_affine_stack(const void* ops_dev, int n_ops, const float* zin, float* zout, float* logq,
                        long long rows, int d, int accumulate, int direction, cudaStream_t st) {
    NFB_CHECK(d >= 1 && d <= kAffMaxD, NFB_ERR_UNSUPPORTED, "affine stack: dim %d > %d", d, kAffMaxD);
    if (rows == 0) return NFB_OK;
    affine_stack_kernel<<<(unsigned)((rows + 127) / 128), 128, 0, st>>>(
        static_cast<const AffineOp*>(ops_dev), n_ops, zin, zout, logq, rows, d, accumulate, direction);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

size_t affine_op_size() { return sizeof(AffineOp); }

// ---------------------------------------------------------------------------------------------------------------
// Sampling-direction backward (direction = 1).  Kernel A (affine_bwd_rows_kernel), one thread per row: recompute the
// stack from z with the forward kernel's own expressions, keeping every op's input row and every Linear's input
// activations and pre-activations in the workspace; then walk the ops in reverse, apply the element adjoints
// (nfb_affine_bwd.cuh) and back-propagate through the MLPs, overwriting each pre-activation with its output cotangent.
// Kernel B (affine_bwd_partial_kernel + affine_bwd_finish_kernel) reduces sum_rows delta a^T and sum_rows delta for
// every Linear, and the column sums of the AffineConst ops, in a fixed order: warp-per-element partial sums over
// kAffSegRows-row segments, then a fixed-order sum of the segments.  No atomics, so two calls give identical bits.
// ---------------------------------------------------------------------------------------------------------------
#define AFF_U(u, r) ws[(size_t)(u) * R + (r)]

// mlp_eval's arithmetic, also storing the Linear inputs (u_act) and pre-activations (u_del) of row r
__device__ __forceinline__ void mlp_eval_store(const AffMlp& m, const float* in, float* out, float slope, float* ws,
                                               long long R, long long r, const int* u_act, const int* u_del) {
    float a[kAffMaxW], b[kAffMaxW];
    const int n0 = m.sizes[0];
    for (int i = 0; i < n0; ++i) { a[i] = in[i]; AFF_U(u_act[0] + i, r) = a[i]; }
    float* cur = a;
    float* nxt = b;
    for (int l = 0; l < m.n_layers; ++l) {
        const int ni = m.sizes[l], no = m.sizes[l + 1];
        const float* w = m.w[l];
        const float* bias = m.b[l];
        const bool last = (l + 1 == m.n_layers);
        for (int o = 0; o < no; ++o) {
            float acc = __ldg(bias + o);
            for (int i = 0; i < ni; ++i) acc = fmaf(cur[i], __ldg(w + o * ni + i), acc);
            AFF_U(u_del[l] + o, r) = acc;
            nxt[o] = last ? acc : (acc >= 0.f ? acc : acc * slope);
            if (!last) AFF_U(u_act[l + 1] + o, r) = nxt[o];
        }
        float* tmp = cur; cur = nxt; nxt = tmp;
    }
    const int no = m.sizes[m.n_layers];
    for (int o = 0; o < no; ++o) out[o] = cur[o];
}

// back-propagate the output cotangents (already in u_del[last]) to the input: g_in[n0]; hidden cotangents are written
// over their pre-activations (LeakyReLU derivative: 1 where pre > 0, else slope -- torch's leaky_relu_backward)
__device__ __forceinline__ void mlp_backward_row(const AffMlp& m, float slope, float* ws, long long R, long long r,
                                                 const int* u_del, float* g_in) {
    float acc[kAffMaxW];
    for (int l = m.n_layers - 1; l >= 0; --l) {
        const int ni = m.sizes[l], no = m.sizes[l + 1];
        const float* w = m.w[l];
        for (int i = 0; i < ni; ++i) acc[i] = 0.f;
        for (int o = 0; o < no; ++o) {
            const float dl = AFF_U(u_del[l] + o, r);
            for (int i = 0; i < ni; ++i) acc[i] = fmaf(__ldg(w + o * ni + i), dl, acc[i]);
        }
        if (l > 0) {
            for (int i = 0; i < ni; ++i) {
                float& p = AFF_U(u_del[l - 1] + i, r);
                p = p > 0.f ? acc[i] : acc[i] * slope;
            }
        } else {
            for (int i = 0; i < ni; ++i) g_in[i] = acc[i];
        }
    }
}

__global__ void __launch_bounds__(128)
affine_bwd_rows_kernel(const AffineOp* __restrict__ ops, const AffBwdOp* __restrict__ bops, int n_ops,
                       const float* __restrict__ zin, const float* __restrict__ gx, const float* __restrict__ gld,
                       float* __restrict__ gz, float* __restrict__ ws, long long R, int d) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    float z[kAffMaxD];
    for (int j = 0; j < d; ++j) z[j] = zin[r * d + j];
    // ---- recompute (affine_stack_kernel, direction = 1) ----
    for (int k = 0; k < n_ops; ++k) {
        const AffineOp& op = ops[k];
        const AffBwdOp& bo = bops[k];
        for (int j = 0; j < d; ++j) AFF_U(bo.u_z + j, r) = z[j];
        if (op.type == kOpMasked) {
            float zm[kAffMaxD], s[kAffMaxD], t[kAffMaxD];
            for (int j = 0; j < d; ++j) zm[j] = __ldg(op.p0 + j) * z[j];
            if (op.s.n_layers) mlp_eval_store(op.s, zm, s, op.slope, ws, R, r, bo.u_act[0], bo.u_del[0]);
            else for (int j = 0; j < d; ++j) s[j] = 0.f;
            if (op.t.n_layers) mlp_eval_store(op.t, zm, t, op.slope_t, ws, R, r, bo.u_act[1], bo.u_del[1]);
            else for (int j = 0; j < d; ++j) t[j] = 0.f;
            for (int j = 0; j < d; ++j) {
                const float b = __ldg(op.p0 + j);
                const float sj = isfinite(s[j]) ? s[j] : __int_as_float(0x7fc00000);
                const float tj = isfinite(t[j]) ? t[j] : __int_as_float(0x7fc00000);
                z[j] = zm[j] + (1.f - b) * (z[j] * expf(sj) + tj);
            }
        } else if (op.type == kOpConst) {
            for (int j = 0; j < d; ++j) z[j] = z[j] * expf(__ldg(op.p0 + j)) + __ldg(op.p1 + j);
        } else if (op.type == kOpCoupling) {
            const int h = (d + 1) / 2;
            const bool inv_split = (op.flags >> 3) & 1;
            const int o1 = inv_split ? h : 0, n1 = inv_split ? d - h : h;
            const int o2 = inv_split ? 0 : h, n2 = d - n1;
            float param[2 * kAffMaxD];
            mlp_eval_store(op.s, z + o1, param, op.slope, ws, R, r, bo.u_act[0], bo.u_del[0]);
            if (!(op.flags & 1)) {
                for (int j = 0; j < n2; ++j) z[o2 + j] += param[j];
            } else {
                const int smap = (op.flags >> 1) & 3;
                for (int j = 0; j < n2; ++j) {
                    const float shift = param[2 * j], sc = param[2 * j + 1];
                    float& v = z[o2 + j];
                    if (smap == 0) {
                        v = v * expf(sc) + shift;
                    } else {
                        const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
                        v = smap == 1 ? v / sg + shift : v * sg + shift;
                    }
                }
            }
        } else {
            float tmp[kAffMaxD];
            for (int j = 0; j < d; ++j) tmp[j] = z[__ldg(op.fwd_idx + j)];
            for (int j = 0; j < d; ++j) z[j] = tmp[j];
        }
    }
    // ---- adjoint, ops in reverse ----
    float g[kAffMaxD];
    for (int j = 0; j < d; ++j) g[j] = gx ? gx[r * d + j] : 0.f;
    const float gam = gld ? gld[r] : 0.f;
    for (int k = n_ops - 1; k >= 0; --k) {
        const AffineOp& op = ops[k];
        const AffBwdOp& bo = bops[k];
        for (int j = 0; j < d; ++j) z[j] = AFF_U(bo.u_z + j, r);
        if (op.type == kOpMasked) {
            const int ls = op.s.n_layers - 1, lt = op.t.n_layers - 1;
            float gs[kAffMaxD], gt[kAffMaxD];
            for (int j = 0; j < d; ++j) {
                const float s = ls >= 0 ? AFF_U(bo.u_del[0][ls] + j, r) : 0.f;
                const float t = lt >= 0 ? AFF_U(bo.u_del[1][lt] + j, r) : 0.f;
                float sh, th;
                masked_affine_adjoint<float>(z[j], __ldg(op.p0 + j), s, t, g[j], gam, sh, th, g[j]);
                if (ls >= 0) AFF_U(bo.u_del[0][ls] + j, r) = sh;
                if (lt >= 0) AFF_U(bo.u_del[1][lt] + j, r) = th;
                gs[j] = gt[j] = 0.f;
            }
            if (ls >= 0) mlp_backward_row(op.s, op.slope, ws, R, r, bo.u_del[0], gs);
            if (lt >= 0) mlp_backward_row(op.t, op.slope_t, ws, R, r, bo.u_del[1], gt);
            for (int j = 0; j < d; ++j) g[j] += __ldg(op.p0 + j) * (gs[j] + gt[j]);
        } else if (op.type == kOpConst) {
            for (int j = 0; j < d; ++j) {
                float cs, ct;
                affine_const_adjoint<float>(z[j], __ldg(op.p0 + j), g[j], gam, g[j], cs, ct);
                AFF_U(bo.u_del[0][0] + j, r) = cs;
                AFF_U(bo.u_del[1][0] + j, r) = ct;
            }
        } else if (op.type == kOpCoupling) {
            const int h = (d + 1) / 2;
            const bool inv_split = (op.flags >> 3) & 1;
            const int o1 = inv_split ? h : 0, n1 = inv_split ? d - h : h;
            const int o2 = inv_split ? 0 : h, n2 = d - n1;
            const int scale = op.flags & 1, smap = (op.flags >> 1) & 3;
            const int lp = op.s.n_layers - 1;
            for (int j = 0; j < n2; ++j) {
                float gv, gsh, gsc;
                if (scale) {
                    const float sc = AFF_U(bo.u_del[0][lp] + 2 * j + 1, r);
                    coupling_adjoint<float>(1, smap, z[o2 + j], sc, g[o2 + j], gam, gv, gsh, gsc);
                    AFF_U(bo.u_del[0][lp] + 2 * j, r) = gsh;
                    AFF_U(bo.u_del[0][lp] + 2 * j + 1, r) = gsc;
                } else {
                    coupling_adjoint<float>(0, 0, z[o2 + j], 0.f, g[o2 + j], gam, gv, gsh, gsc);
                    AFF_U(bo.u_del[0][lp] + j, r) = gsh;
                }
                g[o2 + j] = gv;
            }
            float g1[kAffMaxD];
            mlp_backward_row(op.s, op.slope, ws, R, r, bo.u_del[0], g1);
            for (int j = 0; j < n1; ++j) g[o1 + j] += g1[j];
        } else {  // x[j] = z[fwd[j]]  ->  g_z[i] = g_x[inv[i]]
            float tmp[kAffMaxD];
            for (int j = 0; j < d; ++j) tmp[j] = g[__ldg(op.inv_idx + j)];
            for (int j = 0; j < d; ++j) g[j] = tmp[j];
        }
    }
    if (gz) for (int j = 0; j < d; ++j) gz[r * d + j] = g[j];
}

// Density-direction backward (direction = 0), the same workspace plan and reduction: recompute the stack from x taking
// the ops last-to-first with the forward kernel's inverse expressions, then walk them first-to-last with the density
// adjoints of nfb_affine_bwd.cuh.  Like the sampling kernel it keeps its own copy of the per-op arithmetic, so that
// affine_stack_kernel's code stays as it is.
__global__ void __launch_bounds__(128)
affine_density_bwd_rows_kernel(const AffineOp* __restrict__ ops, const AffBwdOp* __restrict__ bops, int n_ops,
                               const float* __restrict__ xin, const float* __restrict__ gzo,
                               const float* __restrict__ gld, float* __restrict__ gx, float* __restrict__ ws,
                               long long R, int d) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    float z[kAffMaxD];
    for (int j = 0; j < d; ++j) z[j] = xin[r * d + j];
    // ---- recompute (affine_stack_kernel, direction = 0) ----
    for (int k = n_ops - 1; k >= 0; --k) {
        const AffineOp& op = ops[k];
        const AffBwdOp& bo = bops[k];
        for (int j = 0; j < d; ++j) AFF_U(bo.u_z + j, r) = z[j];
        if (op.type == kOpMasked) {
            float zm[kAffMaxD], s[kAffMaxD], t[kAffMaxD];
            for (int j = 0; j < d; ++j) zm[j] = __ldg(op.p0 + j) * z[j];
            if (op.s.n_layers) mlp_eval_store(op.s, zm, s, op.slope, ws, R, r, bo.u_act[0], bo.u_del[0]);
            else for (int j = 0; j < d; ++j) s[j] = 0.f;
            if (op.t.n_layers) mlp_eval_store(op.t, zm, t, op.slope_t, ws, R, r, bo.u_act[1], bo.u_del[1]);
            else for (int j = 0; j < d; ++j) t[j] = 0.f;
            for (int j = 0; j < d; ++j) {
                const float b = __ldg(op.p0 + j);
                const float sj = isfinite(s[j]) ? s[j] : __int_as_float(0x7fc00000);
                const float tj = isfinite(t[j]) ? t[j] : __int_as_float(0x7fc00000);
                z[j] = zm[j] + (1.f - b) * (z[j] - tj) * expf(-sj);
            }
        } else if (op.type == kOpConst) {
            for (int j = 0; j < d; ++j) z[j] = (z[j] - __ldg(op.p1 + j)) * expf(-__ldg(op.p0 + j));
        } else if (op.type == kOpCoupling) {
            const int h = (d + 1) / 2;
            const bool inv_split = (op.flags >> 3) & 1;
            const int o1 = inv_split ? h : 0, n1 = inv_split ? d - h : h;
            const int o2 = inv_split ? 0 : h, n2 = d - n1;
            float param[2 * kAffMaxD];
            mlp_eval_store(op.s, z + o1, param, op.slope, ws, R, r, bo.u_act[0], bo.u_del[0]);
            if (!(op.flags & 1)) {
                for (int j = 0; j < n2; ++j) z[o2 + j] += -param[j];
            } else {
                const int smap = (op.flags >> 1) & 3;
                for (int j = 0; j < n2; ++j) {
                    const float shift = param[2 * j], sc = param[2 * j + 1];
                    float& v = z[o2 + j];
                    if (smap == 0) {
                        v = (v - shift) * expf(-sc);
                    } else {
                        const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
                        v = smap == 1 ? (v - shift) * sg : (v - shift) / sg;
                    }
                }
            }
        } else {
            float tmp[kAffMaxD];
            for (int j = 0; j < d; ++j) tmp[j] = z[__ldg(op.inv_idx + j)];
            for (int j = 0; j < d; ++j) z[j] = tmp[j];
        }
    }
    // ---- adjoint, ops first-to-last ----
    float g[kAffMaxD];
    for (int j = 0; j < d; ++j) g[j] = gzo ? gzo[r * d + j] : 0.f;
    const float gam = gld ? gld[r] : 0.f;
    for (int k = 0; k < n_ops; ++k) {
        const AffineOp& op = ops[k];
        const AffBwdOp& bo = bops[k];
        for (int j = 0; j < d; ++j) z[j] = AFF_U(bo.u_z + j, r);
        if (op.type == kOpMasked) {
            const int ls = op.s.n_layers - 1, lt = op.t.n_layers - 1;
            float gs[kAffMaxD], gt[kAffMaxD];
            for (int j = 0; j < d; ++j) {
                const float s = ls >= 0 ? AFF_U(bo.u_del[0][ls] + j, r) : 0.f;
                const float t = lt >= 0 ? AFF_U(bo.u_del[1][lt] + j, r) : 0.f;
                float sh, th;
                masked_affine_density_adjoint<float>(z[j], __ldg(op.p0 + j), s, t, g[j], gam, sh, th, g[j]);
                if (ls >= 0) AFF_U(bo.u_del[0][ls] + j, r) = sh;
                if (lt >= 0) AFF_U(bo.u_del[1][lt] + j, r) = th;
                gs[j] = gt[j] = 0.f;
            }
            if (ls >= 0) mlp_backward_row(op.s, op.slope, ws, R, r, bo.u_del[0], gs);
            if (lt >= 0) mlp_backward_row(op.t, op.slope_t, ws, R, r, bo.u_del[1], gt);
            for (int j = 0; j < d; ++j) g[j] += __ldg(op.p0 + j) * (gs[j] + gt[j]);
        } else if (op.type == kOpConst) {
            for (int j = 0; j < d; ++j) {
                float cs, ct;
                affine_const_density_adjoint<float>(z[j], __ldg(op.p0 + j), __ldg(op.p1 + j), g[j], gam, g[j], cs, ct);
                AFF_U(bo.u_del[0][0] + j, r) = cs;
                AFF_U(bo.u_del[1][0] + j, r) = ct;
            }
        } else if (op.type == kOpCoupling) {
            const int h = (d + 1) / 2;
            const bool inv_split = (op.flags >> 3) & 1;
            const int o1 = inv_split ? h : 0, n1 = inv_split ? d - h : h;
            const int o2 = inv_split ? 0 : h, n2 = d - n1;
            const int scale = op.flags & 1, smap = (op.flags >> 1) & 3;
            const int lp = op.s.n_layers - 1;
            for (int j = 0; j < n2; ++j) {
                float gv, gsh, gsc;
                if (scale) {
                    float& ush = AFF_U(bo.u_del[0][lp] + 2 * j, r);
                    float& usc = AFF_U(bo.u_del[0][lp] + 2 * j + 1, r);
                    coupling_density_adjoint<float>(1, smap, z[o2 + j], ush, usc, g[o2 + j], gam, gv, gsh, gsc);
                    ush = gsh;
                    usc = gsc;
                } else {
                    float& up = AFF_U(bo.u_del[0][lp] + j, r);
                    coupling_density_adjoint<float>(0, 0, z[o2 + j], up, 0.f, g[o2 + j], gam, gv, gsh, gsc);
                    up = gsh;
                }
                g[o2 + j] = gv;
            }
            float g1[kAffMaxD];
            mlp_backward_row(op.s, op.slope, ws, R, r, bo.u_del[0], g1);
            for (int j = 0; j < n1; ++j) g[o1 + j] += g1[j];
        } else {  // x[j] = z[inv[j]]  ->  g_z[i] = g_x[fwd[i]]
            float tmp[kAffMaxD];
            for (int j = 0; j < d; ++j) tmp[j] = g[__ldg(op.fwd_idx + j)];
            for (int j = 0; j < d; ++j) g[j] = tmp[j];
        }
    }
    if (gx) for (int j = 0; j < d; ++j) gx[r * d + j] = g[j];
}

__device__ __forceinline__ int aff_find_item(const AffRedItem* items, int n_items, long long e) {
    int lo = 0, hi = n_items - 1;   // last item with e_off <= e
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (items[mid].e_off <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// one warp per (element, row segment): lanes stride the segment's rows, then a fixed butterfly
__global__ void __launch_bounds__(256)
affine_bwd_partial_kernel(const AffRedItem* __restrict__ items, int n_items, long long n_elem,
                          const float* __restrict__ ws, long long R, float* __restrict__ partial) {
    const long long e = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (e >= n_elem) return;
    const AffRedItem it = items[aff_find_item(items, n_items, e)];
    const long long k = e - it.e_off;
    const long long nw = (long long)it.n_out * it.n_in;
    const int o = (int)(k < nw ? k / it.n_in : k - nw);
    const int i = k < nw ? (int)(k % it.n_in) : -1;
    const long long r0 = (long long)blockIdx.y * kAffSegRows, r1 = min(R, r0 + kAffSegRows);
    float acc = 0.f;
    for (long long r = r0 + lane; r < r1; r += 32) {
        const float dl = AFF_U(it.u_del + o, r);
        acc = i >= 0 ? fmaf(dl, AFF_U(it.u_act + i, r), acc) : acc + dl;
    }
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) partial[(size_t)blockIdx.y * n_elem + e] = acc;
}

__global__ void affine_bwd_finish_kernel(const AffRedItem* __restrict__ items, int n_items, long long n_elem,
                                         const float* __restrict__ partial, int n_seg, int accumulate) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_elem) return;
    const AffRedItem it = items[aff_find_item(items, n_items, e)];
    const long long k = e - it.e_off;
    const long long nw = (long long)it.n_out * it.n_in;
    float* dst = k < nw ? (it.dw ? it.dw + k : nullptr) : (it.db ? it.db + (k - nw) : nullptr);
    if (!dst) return;
    float s = 0.f;
    for (int g = 0; g < n_seg; ++g) s += partial[(size_t)g * n_elem + e];
    *dst = accumulate ? *dst + s : s;
}
#undef AFF_U

int launch_affine_bwd_rows(const void* ops_dev, const void* bops_dev, int n_ops, int direction, const float* zin,
                           const float* gx, const float* gld, float* gz, float* ws, long long R, int d, cudaStream_t st) {
    if (R == 0) return NFB_OK;
    const AffineOp* ops = static_cast<const AffineOp*>(ops_dev);
    const AffBwdOp* bops = static_cast<const AffBwdOp*>(bops_dev);
    if (direction)
        affine_bwd_rows_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(ops, bops, n_ops, zin, gx, gld, gz, ws, R, d);
    else
        affine_density_bwd_rows_kernel<<<(unsigned)((R + 127) / 128), 128, 0, st>>>(ops, bops, n_ops, zin, gx, gld, gz,
                                                                                     ws, R, d);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// partial sums (skipped when R = 0) + the fixed-order finish: with R = 0 and accumulate = 0 it writes zeros
int launch_affine_bwd_reduce(const void* items_dev, int n_items, long long n_elem, const float* ws, long long R,
                             float* partial, int accumulate, cudaStream_t st) {
    if (n_elem == 0) return NFB_OK;
    const int n_seg = (int)((R + kAffSegRows - 1) / kAffSegRows);
    const AffRedItem* items = static_cast<const AffRedItem*>(items_dev);
    if (n_seg > 0) {
        affine_bwd_partial_kernel<<<dim3((unsigned)((n_elem + 7) / 8), (unsigned)n_seg), 256, 0, st>>>(
            items, n_items, n_elem, ws, R, partial);
        NFB_LAUNCH_CHECK();
    }
    affine_bwd_finish_kernel<<<(unsigned)((n_elem + 255) / 256), 256, 0, st>>>(items, n_items, n_elem, partial, n_seg,
                                                                                accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
