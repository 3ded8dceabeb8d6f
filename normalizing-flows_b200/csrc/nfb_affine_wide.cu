// nfb_affine_wide.cu -- element kernels of the affine family's wide path: stacks with more than kAffMaxD features or a
// net wider than kAffMaxW, which affine_stack_kernel's one-thread-per-row design cannot hold in registers.  The host
// (nfb_api.cu, affine_wide_apply / affine_wide_backward) runs such a group layer by layer: the s / t nets (param_map of
// the coupling block) on gemm_tc_kernel, the coupling arithmetic here.  Per layer:
//   affine_wide_mask_kernel     zm = b z, the masked input of a MaskedAffineFlow's nets
//   affine_wide_elem_kernel     the op's output and log-det (formulas: nfb_affine_wide.cuh); one warp per row, lanes
//                               over the features, a fixed butterfly for the row's log-det sum, added into log_det
//   affine_wide_adjoint_kernel  one thread per element: g_z (direct part, in place over the output cotangent) and the
//                               cotangents of the nets' outputs (in place over s / t / param) or AffineConstFlow's per-row
//                               contributions (nfb_affine_bwd.cuh)
// Permute is a column gather (launch_gather_cols).
#include "nfb_kernels.h"
#include "nfb_affine_wide.cuh"

namespace nfb {

namespace {
struct OpCoupling : CouplingSplit {   // the split and the scale flags of a coupling op (AffineOp::flags)
    int scale, smap;
    __device__ explicit OpCoupling(const AffineOp& op, int d)
        : CouplingSplit(d, (op.flags >> 3) & 1), scale(op.flags & 1), smap((op.flags >> 1) & 3) {}
};
}  // namespace

__global__ void __launch_bounds__(256)
affine_wide_mask_kernel(const float* __restrict__ z, const float* __restrict__ b, float* __restrict__ zm, long long n,
                        int d) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) zm[i] = __ldg(b + (int)(i % d)) * z[i];
}

// S / T: the nets' outputs [rows, d] (null: the net is absent, its term 0); coupling: S = param [rows, (1 + scale) n2]
__global__ void __launch_bounds__(256)
affine_wide_elem_kernel(const AffineOp op, int d, int dir, const float* __restrict__ zin, const float* __restrict__ S,
                        const float* __restrict__ T, float* __restrict__ zout, float* __restrict__ ld, long long rows) {
    const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;   // (uniform over the warp)
    const float* z = zin + r * d;
    float* x = zout + r * d;
    float acc = 0.f;
    if (op.type == kOpMasked) {
        for (int j = lane; j < d; j += 32) {
            float o, l;
            masked_affine_elem<float>(dir, z[j], __ldg(op.p0 + j), S ? S[r * d + j] : 0.f, T ? T[r * d + j] : 0.f, o, l);
            x[j] = o;
            acc += l;
        }
    } else if (op.type == kOpConst) {
        for (int j = lane; j < d; j += 32) {
            float o, l;
            affine_const_elem<float>(dir, z[j], __ldg(op.p0 + j), __ldg(op.p1 + j), o, l);
            x[j] = o;
            acc += l;
        }
    } else {
        const OpCoupling c(op, d);
        const float* P = S + r * (long long)((1 + c.scale) * c.n2);
        for (int j = lane; j < d; j += 32) {
            const int k = j - c.o2;
            if (k < 0 || k >= c.n2) { x[j] = z[j]; continue; }
            float o, l;
            coupling_elem<float>(dir, c.scale, c.smap, z[j], c.scale ? P[2 * k] : P[k], c.scale ? P[2 * k + 1] : 0.f, o, l);
            x[j] = o;
            acc += l;
        }
    }
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0 && ld) ld[r] += acc;
}

// zin: the op's input in direction dir; G: the cotangent of its output, overwritten by the direct part of g_z;
// gld: the log-det cotangent per row (null: 0).  Masked: S / T (null when the net is absent) overwritten by the
// cotangents of the nets' outputs.  Const: S / T receive the per-row contributions to g_s / g_t.  Coupling: S = param,
// overwritten by its cotangent; the identity half of G is left as it is.
__global__ void __launch_bounds__(256)
affine_wide_adjoint_kernel(const AffineOp op, int d, int dir, const float* __restrict__ zin, float* __restrict__ S,
                           float* __restrict__ T, float* __restrict__ G, const float* __restrict__ gld, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * d) return;
    const long long r = i / d;
    const int j = (int)(i - r * d);
    const float z = zin[i], g = G[i], gam = gld ? gld[r] : 0.f;
    if (op.type == kOpMasked) {
        const float b = __ldg(op.p0 + j), s = S ? S[i] : 0.f, t = T ? T[i] : 0.f;
        float sh, th, gz;
        if (dir) masked_affine_adjoint<float>(z, b, s, t, g, gam, sh, th, gz);
        else masked_affine_density_adjoint<float>(z, b, s, t, g, gam, sh, th, gz);
        G[i] = gz;
        if (S) S[i] = sh;
        if (T) T[i] = th;
    } else if (op.type == kOpConst) {
        float gz, cs, ct;
        if (dir) affine_const_adjoint<float>(z, __ldg(op.p0 + j), g, gam, gz, cs, ct);
        else affine_const_density_adjoint<float>(z, __ldg(op.p0 + j), __ldg(op.p1 + j), g, gam, gz, cs, ct);
        G[i] = gz;
        S[i] = cs;
        T[i] = ct;
    } else {
        const OpCoupling c(op, d);
        const int k = j - c.o2;
        if (k < 0 || k >= c.n2) return;
        float* P = S + r * (long long)((1 + c.scale) * c.n2);
        float gv, gsh, gsc;
        if (c.scale) {
            if (dir) coupling_adjoint<float>(1, c.smap, z, P[2 * k + 1], g, gam, gv, gsh, gsc);
            else coupling_density_adjoint<float>(1, c.smap, z, P[2 * k], P[2 * k + 1], g, gam, gv, gsh, gsc);
            P[2 * k] = gsh;
            P[2 * k + 1] = gsc;
        } else {
            if (dir) coupling_adjoint<float>(0, 0, z, 0.f, g, gam, gv, gsh, gsc);
            else coupling_density_adjoint<float>(0, 0, z, P[k], 0.f, g, gam, gv, gsh, gsc);
            P[k] = gsh;
        }
        G[i] = gv;
    }
}

int launch_affine_wide_mask(const float* z, const float* b, float* zm, long long rows, int d, cudaStream_t st) {
    const long long n = rows * d;
    if (n == 0) return NFB_OK;
    affine_wide_mask_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(z, b, zm, n, d);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_affine_wide_elem(const AffineOp& op, int d, int dir, const float* zin, const float* S, const float* T,
                            float* zout, float* ld, long long rows, cudaStream_t st) {
    if (rows == 0) return NFB_OK;
    affine_wide_elem_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(op, d, dir, zin, S, T, zout, ld, rows);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_affine_wide_adjoint(const AffineOp& op, int d, int dir, const float* zin, float* S, float* T, float* G,
                               const float* gld, long long rows, cudaStream_t st) {
    const long long n = rows * d;
    if (n == 0) return NFB_OK;
    affine_wide_adjoint_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(op, d, dir, zin, S, T, G, gld, rows);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
