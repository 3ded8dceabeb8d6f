// nfb_planar.cu -- stacks of planar and radial flows (Rezende & Mohamed 2015; reference flows/planar.py, radial.py) in
// ONE kernel launch, and the sampling direction's backward.
//
// One thread per row keeps z[D] (D <= 64) and the running log-det in registers and walks the layer list, like
// affine_stack_kernel.  The per-layer constants depend on the parameters only -- planar k (u_hat = u + k w) and
// psi = w.u_hat, radial |alpha| and log(1 + exp(beta)) - |alpha| -- and are formed on the device by every CTA, for a
// tile of kPlanarTile layers at a time, into shared memory: nothing waits on the host, and a parameter update needs no
// repack.  The backward's recompute forms them with the same functions (nfb_planar_bwd.cuh).
//   sampling (direction 1):  planar x = z + u_hat h(w.z + b), ld += log|1 + psi h'(w.z + b)|      planar.py:51-64
//                            radial x = z + h (z - z0), ld += (d-1) log(1 + h) + log(1 + h + h_)  radial.py:37-46
//   density (direction 0):   leaky-ReLU planar only, planar.py:66-81 (the host refuses any other layer)
// The row loops run to a compile-time bound MAXD (guarded by j < d), so z[] stays in registers.
#include "nfb_kernels.h"
#include "nfb_planar_bwd.cuh"

namespace nfb {

constexpr int kPlanarTile = 256;   // layers whose constants one CTA holds in shared memory at a time

__device__ __forceinline__ float2 planar_layer_consts(const PlanarOp& op, int d) {
    float c0, c1;
    if (op.type == kRadial) radial_consts<float>(__ldg(op.alpha), __ldg(op.b), c0, c1);
    else planar_consts<float>(op.a, op.w, d, c0, c1);
    return make_float2(c0, c1);
}

// constants of layers [t0, t0 + nt) of the application order (order[i] = index of the i-th applied layer) into cst
__device__ __forceinline__ void planar_tile_consts(const PlanarOp* ops, int n_ops, int t0, int nt, int direction, int d,
                                                   float2* cst) {
    __syncthreads();   // the previous tile's constants are no longer read
    for (int i = threadIdx.x; i < nt; i += blockDim.x) {
        const int k = direction ? t0 + i : n_ops - 1 - (t0 + i);
        cst[i] = planar_layer_consts(ops[k], d);
    }
    __syncthreads();
}

// one layer of the sampling direction on the row z (shared by the forward and the backward's recompute)
template <int MAXD>
__device__ __forceinline__ void planar_apply_fwd(const PlanarOp& op, float2 c, float* z, int d, float& ld) {
    if (op.type == kRadial) {   // (z - z0 is formed twice rather than held: registers)
        float r2 = 0.f;
#pragma unroll
        for (int j = 0; j < MAXD; ++j)
            if (j < d) { const float dz = z[j] - __ldg(op.a + j); r2 = fmaf(dz, dz, r2); }
        const float r = sqrtf(r2);
        const float s = c.x + r;
        const float h = c.y / s;
        const float h_ = -c.y * r / (s * s);
#pragma unroll
        for (int j = 0; j < MAXD; ++j)
            if (j < d) z[j] = fmaf(h, z[j] - __ldg(op.a + j), z[j]);
        ld += (float)(d - 1) * logf(1.f + h) + logf(1.f + h + h_);
    } else {
        float lin = 0.f;
#pragma unroll
        for (int j = 0; j < MAXD; ++j)
            if (j < d) lin = fmaf(__ldg(op.w + j), z[j], lin);
        lin += __ldg(op.b);
        float h, hp, hd, hpp;
        planar_act<float>(op.type, op.slope, lin, h, hp, hd, hpp);
#pragma unroll
        for (int j = 0; j < MAXD; ++j)
            if (j < d) z[j] = fmaf(__ldg(op.a + j) + c.x * __ldg(op.w + j), h, z[j]);
        ld += logf(fabsf(1.f + c.y * hp));
    }
}

// one leaky-ReLU planar layer of the density direction (planar.py:66-81): a = h'(lin), z_ = z - a u_hat lin / (1 + a psi)
template <int MAXD>
__device__ __forceinline__ void planar_apply_inv(const PlanarOp& op, float2 c, float* z, int d, float& ld) {
    float lin = 0.f;
#pragma unroll
    for (int j = 0; j < MAXD; ++j)
        if (j < d) lin = fmaf(__ldg(op.w + j), z[j], lin);
    lin += __ldg(op.b);
    const float a = lin < 0.f ? (op.slope - 1.f) + 1.f : 1.f;
    const float inner = a * c.y;
    const float t = lin / (1.f + inner);
#pragma unroll
    for (int j = 0; j < MAXD; ++j)
        if (j < d) z[j] -= a * (__ldg(op.a + j) + c.x * __ldg(op.w + j)) * t;
    ld -= logf(fabsf(1.f + inner));
}

template <int MAXD>
__global__ void __launch_bounds__(128)
planar_stack_kernel(const PlanarOp* __restrict__ ops, int n_ops, const float* __restrict__ zin, float* __restrict__ zout,
                    float* __restrict__ logq, long long rows, int d, int accumulate, int direction) {
    __shared__ float2 cst[kPlanarTile];
    const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = row < rows;   // (every thread takes part in the constants' barriers)
    float z[MAXD];
#pragma unroll
    for (int j = 0; j < MAXD; ++j) z[j] = (live && j < d) ? zin[row * d + j] : 0.f;
    float ld = 0.f;
    for (int t0 = 0; t0 < n_ops; t0 += kPlanarTile) {
        const int nt = min(kPlanarTile, n_ops - t0);
        planar_tile_consts(ops, n_ops, t0, nt, direction, d, cst);
        if (!live) continue;
        for (int i = 0; i < nt; ++i) {
            const PlanarOp& op = ops[direction ? t0 + i : n_ops - 1 - (t0 + i)];
            if (direction) planar_apply_fwd<MAXD>(op, cst[i], z, d, ld);
            else planar_apply_inv<MAXD>(op, cst[i], z, d, ld);
        }
    }
    if (!live) return;
#pragma unroll
    for (int j = 0; j < MAXD; ++j)
        if (j < d) zout[row * d + j] = z[j];
    if (logq) logq[row] = accumulate ? logq[row] + ld : ld;
}

// ---------------------------------------------------------------------------------------------------------------
// Sampling-direction backward.  planar_bwd_rows_kernel, one thread per row: recompute the stack from z (the forward's
// own code), keeping each layer's input row in the workspace; then walk the layers in reverse with the element
// adjoints of nfb_planar_bwd.cuh, leaving each row's contributions to the parameter gradients in the workspace:
//   planar  units [u_off, +D) z, [+D, +2D) g (cotangent of the layer's output), +2D c, +2D+1 h(lin), +2D+2 e
//   radial  units [u_off, +D) z overwritten by g_dz, +D the beta_hat term, +D+1 the alpha_hat term
// launch_affine_bwd_reduce then sums them over the rows in a fixed order (items built by the host), and
// planar_bwd_chain_kernel takes the sums through the parameter-only maps u_hat(u, w), softplus(beta) and |alpha|.
// ---------------------------------------------------------------------------------------------------------------
#define PL_U(u, r) ws[(size_t)(u) * R + (r)]

template <int MAXD>
__global__ void __launch_bounds__(128)
planar_bwd_rows_kernel(const PlanarOp* __restrict__ ops, int n_ops, const float* __restrict__ zin,
                       const float* __restrict__ gx, const float* __restrict__ gld, float* __restrict__ gz,
                       float* __restrict__ ws, long long R, int d) {
    __shared__ float2 cst[kPlanarTile];
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = r < R;
    float z[MAXD];
#pragma unroll
    for (int j = 0; j < MAXD; ++j) z[j] = (live && j < d) ? zin[r * d + j] : 0.f;
    // ---- recompute ----
    float ld = 0.f;
    for (int t0 = 0; t0 < n_ops; t0 += kPlanarTile) {
        const int nt = min(kPlanarTile, n_ops - t0);
        planar_tile_consts(ops, n_ops, t0, nt, 1, d, cst);
        if (!live) continue;
        for (int i = 0; i < nt; ++i) {
            const PlanarOp& op = ops[t0 + i];
#pragma unroll
            for (int j = 0; j < MAXD; ++j)
                if (j < d) PL_U(op.u_off + j, r) = z[j];
            planar_apply_fwd<MAXD>(op, cst[i], z, d, ld);
        }
    }
    // ---- adjoint, layers in reverse (the layer's input row is read from the workspace where it is used) ----
    float g[MAXD];
#pragma unroll
    for (int j = 0; j < MAXD; ++j) g[j] = (live && j < d && gx) ? gx[r * d + j] : 0.f;
    const float gam = (live && gld) ? gld[r] : 0.f;
    const float dm1 = (float)(d - 1);
    const int n_tiles = (n_ops + kPlanarTile - 1) / kPlanarTile;
    for (int t = n_tiles - 1; t >= 0; --t) {
        const int t0 = t * kPlanarTile, nt = min(kPlanarTile, n_ops - t0);
        planar_tile_consts(ops, n_ops, t0, nt, 1, d, cst);
        if (!live) continue;
        for (int i = nt - 1; i >= 0; --i) {
            const PlanarOp& op = ops[t0 + i];
            const float2 c = cst[i];
            const int u0 = op.u_off;
            if (op.type == kRadial) {
                float r2 = 0.f, gdot = 0.f;
#pragma unroll
                for (int j = 0; j < MAXD; ++j)
                    if (j < d) {
                        const float dz = PL_U(u0 + j, r) - __ldg(op.a + j);
                        r2 = fmaf(dz, dz, r2);
                        gdot = fmaf(g[j], dz, gdot);
                    }
                float h, cr, gbh, gah;
                radial_row_adjoint<float>(sqrtf(r2), c.x, c.y, dm1, gdot, gam, h, cr, gbh, gah);
#pragma unroll
                for (int j = 0; j < MAXD; ++j)
                    if (j < d) {
                        const float gdz = h * g[j] + cr * (PL_U(u0 + j, r) - __ldg(op.a + j));
                        PL_U(u0 + j, r) = gdz;
                        g[j] += gdz;
                    }
                PL_U(u0 + d, r) = gbh;
                PL_U(u0 + d + 1, r) = gah;
            } else {
                float lin = 0.f, gu = 0.f;
#pragma unroll
                for (int j = 0; j < MAXD; ++j)
                    if (j < d) {
                        lin = fmaf(__ldg(op.w + j), PL_U(u0 + j, r), lin);
                        gu = fmaf(g[j], __ldg(op.a + j) + c.x * __ldg(op.w + j), gu);
                    }
                lin += __ldg(op.b);
                float cl, hv, e;
                planar_row_adjoint<float>(op.type, op.slope, lin, c.y, gu, gam, cl, hv, e);
#pragma unroll
                for (int j = 0; j < MAXD; ++j)
                    if (j < d) {
                        PL_U(u0 + d + j, r) = g[j];
                        g[j] = fmaf(cl, __ldg(op.w + j), g[j]);
                    }
                PL_U(u0 + 2 * d, r) = cl;
                PL_U(u0 + 2 * d + 1, r) = hv;
                PL_U(u0 + 2 * d + 2, r) = e;
            }
        }
    }
    if (live && gz) {
#pragma unroll
        for (int j = 0; j < MAXD; ++j)
            if (j < d) gz[r * d + j] = g[j];
    }
}
#undef PL_U

// one thread per layer: the reduced sums through the parameter-only maps, into the gradient slots
__global__ void planar_bwd_chain_kernel(const PlanarOp* __restrict__ ops, const PlanarGradOut* __restrict__ outs,
                                        int n_ops, const float* __restrict__ sums, int d) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_ops) return;
    const PlanarOp op = ops[k];
    const PlanarGradOut o = outs[k];
    const float* S = sums + op.s_off;
    if (op.type == kRadial) {
        float gb, ga;
        radial_param_chain<float>(__ldg(op.alpha), __ldg(op.b), S[d], S[d + 1], gb, ga);
        if (o.g[0]) *o.g[0] = gb;
        if (o.g[1]) *o.g[1] = ga;
        if (o.g[2])
            for (int j = 0; j < d; ++j) o.g[2][j] = -S[j];
    } else {
        planar_param_chain<float>(op.a, op.w, d, S, S[d], S + d + 1, S[2 * d + 2], o.g[0], o.g[1], o.g[2]);
    }
}

template <int MAXD>
static void planar_stack_launch(const PlanarOp* ops, int n_ops, const float* zin, float* zout, float* logq,
                                long long rows, int d, int accumulate, int direction, cudaStream_t st) {
    planar_stack_kernel<MAXD><<<(unsigned)((rows + 127) / 128), 128, 0, st>>>(ops, n_ops, zin, zout, logq, rows, d,
                                                                              accumulate, direction);
}

template <int MAXD>
static void planar_bwd_launch(const PlanarOp* ops, int n_ops, const float* zin, const float* gx, const float* gld,
                              float* gz, float* ws, long long R, int d, cudaStream_t st) {
    planar_bwd_rows_kernel<MAXD><<<(unsigned)((R + 127) / 128), 128, 0, st>>>(ops, n_ops, zin, gx, gld, gz, ws, R, d);
}

#define PLANAR_DISPATCH(fn, d, ...)                                     \
    do {                                                                \
        if ((d) <= 2) fn<2>(__VA_ARGS__);                               \
        else if ((d) <= 4) fn<4>(__VA_ARGS__);                          \
        else if ((d) <= 8) fn<8>(__VA_ARGS__);                          \
        else if ((d) <= 16) fn<16>(__VA_ARGS__);                        \
        else if ((d) <= 32) fn<32>(__VA_ARGS__);                        \
        else fn<64>(__VA_ARGS__);                                       \
    } while (0)

int launch_planar_stack(const void* ops_dev, int n_ops, const float* zin, float* zout, float* logq, long long rows,
                        int d, int accumulate, int direction, cudaStream_t st) {
    NFB_CHECK(d >= 1 && d <= kPlanarMaxD, NFB_ERR_UNSUPPORTED, "planar/radial stack: dim %d > %d", d, kPlanarMaxD);
    if (rows == 0) return NFB_OK;
    PLANAR_DISPATCH(planar_stack_launch, d, static_cast<const PlanarOp*>(ops_dev), n_ops, zin, zout, logq, rows, d,
                    accumulate, direction, st);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_planar_bwd_rows(const void* ops_dev, int n_ops, const float* zin, const float* gx, const float* gld,
                           float* gz, float* ws, long long R, int d, cudaStream_t st) {
    NFB_CHECK(d >= 1 && d <= kPlanarMaxD, NFB_ERR_UNSUPPORTED, "planar/radial stack: dim %d > %d", d, kPlanarMaxD);
    if (R == 0) return NFB_OK;
    PLANAR_DISPATCH(planar_bwd_launch, d, static_cast<const PlanarOp*>(ops_dev), n_ops, zin, gx, gld, gz, ws, R, d, st);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_planar_bwd_chain(const void* ops_dev, const void* outs_dev, int n_ops, const float* sums, int d,
                            cudaStream_t st) {
    if (n_ops == 0) return NFB_OK;
    planar_bwd_chain_kernel<<<(unsigned)((n_ops + 127) / 128), 128, 0, st>>>(
        static_cast<const PlanarOp*>(ops_dev), static_cast<const PlanarGradOut*>(outs_dev), n_ops, sums, d);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
