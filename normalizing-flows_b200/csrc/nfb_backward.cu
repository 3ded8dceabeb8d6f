// nfb_backward.cu -- element-wise and reduction kernels of the TRAINING pass of the neural-spline stacks
// (SURVEY 8f-1: `loss.backward()` of examples/neural_spline_flow.ipynb cell 4), the parts that are not GEMMs:
//   * analytic backward of the rational-quadratic spline element (csrc/nfb_spline_bwd.cuh; utils/splines.py:100-219)
//     for conditioner-parameterised features (rows x T x (3K-1) parameter gradients) and for the unconditional CDF
//     of the coupling layer's identity features (neural_spline/coupling.py:221-253: parameters shared by the batch,
//     gradient = sum over rows),
//   * DiagGaussian.log_prob backward (distributions/base.py:94-103),
//   * column sums (bias gradients), LU-factor gradients of LULinearPermute (flows/mixing.py:402-412,514-532).
// The dense products (recompute / dgrad / wgrad of every Linear) run on the tensor core: csrc/nfb_gemm_tc.cu.
// All of these are HBM-bound streaming kernels: coalesced through shared-memory staging where the natural access
// is strided (23 parameters per element), one pass over the data.
#include "nfb_kernels.h"
#include "nfb_maf_bwd.cuh"
#include "nfb_spline_bwd.cuh"

namespace nfb {

namespace {
constexpr int kP = 23;  // 3K - 1 for K = 8
}

// One thread per (row, feature) element, 256 consecutive elements per block; the block's 256 x 23 parameter slab is
// contiguous in memory: staged through shared memory with coalesced loads, read at the conflict-free odd stride 23,
// gradients written back the same way.  INV: the inverse spline of the sampling direction (rqs_inv_fwd_bwd): xin is its
// input z, g_out the cotangent of its output x, gx receives g_z.
template <int K, typename T>
__device__ __forceinline__ void rqs_dir_fwd_bwd(bool inv, T x, const T (&lw)[K], const T (&lh)[K], const T (&ud)[K - 1],
                                                T tail, T gy, T glad, T& y, T& lad, T& gx, T (&glw)[K], T (&glh)[K],
                                                T (&gud)[K - 1]) {
    if (inv) rqs_inv_fwd_bwd<K, T>(x, lw, lh, ud, tail, gy, glad, y, lad, gx, glw, glh, gud);
    else rqs_fwd_bwd<K, T>(x, lw, lh, ud, tail, gy, glad, y, lad, gx, glw, glh, gud);
}

template <bool INV>
__global__ void __launch_bounds__(256) spline_bwd_rows_kernel(
    const float* __restrict__ xin, int ldx, const float* __restrict__ params, const float* __restrict__ g_out,
    const float* __restrict__ g_lq, const int* __restrict__ fidx, long long rows, int T, float tail, float wh_scale,
    float* __restrict__ g_params, float* __restrict__ gx) {
    __shared__ float sp[256 * kP];
    const long long e0 = (long long)blockIdx.x * 256;
    const long long n_el = rows * T;
    const long long n_valid = n_el - e0 < 256 ? n_el - e0 : 256;
    const float* src = params + e0 * kP;
    for (int i = threadIdx.x; i < n_valid * kP; i += 256) sp[i] = __ldg(src + i);
    __syncthreads();
    const long long e = e0 + threadIdx.x;
    float glw[8], glh[8], gud[7];
    if (e < n_el) {
        const long long row = e / T;
        const int t = (int)(e - row * T);
        const int col = fidx ? fidx[t] : t;
        const float* p = sp + threadIdx.x * kP;
        const float s2 = wh_scale * kLog2e;
        float lw[8], lh[8], ud[7];
#pragma unroll
        for (int k = 0; k < 8; ++k) { lw[k] = p[k] * s2; lh[k] = p[8 + k] * s2; }
#pragma unroll
        for (int k = 0; k < 7; ++k) ud[k] = p[16 + k];
        float y, lad, g;
        rqs_dir_fwd_bwd<8, float>(INV, xin[row * ldx + col], lw, lh, ud, tail, g_out[row * ldx + col], g_lq[row], y, lad,
                                  g, glw, glh, gud);
        gx[row * ldx + col] = g;
#pragma unroll
        for (int k = 0; k < 8; ++k) { glw[k] *= s2; glh[k] *= s2; }
    }
    __syncthreads();
    if (e < n_el) {
        float* p = sp + threadIdx.x * kP;
#pragma unroll
        for (int k = 0; k < 8; ++k) { p[k] = glw[k]; p[8 + k] = glh[k]; }
#pragma unroll
        for (int k = 0; k < 7; ++k) p[16 + k] = gud[k];
    }
    __syncthreads();
    float* dst = g_params + e0 * kP;
    for (int i = threadIdx.x; i < n_valid * kP; i += 256) dst[i] = sp[i];
}
int launch_spline_bwd_rows(const float* xin, int ldx, const float* params, const float* g_out, const float* g_lq,
                           const int* fidx, long long rows, int T, int K, float tail, float wh_scale, float* g_params,
                           float* gx, cudaStream_t st, int inverse) {
    NFB_CHECK(K == 8, NFB_ERR_UNSUPPORTED, "spline backward: num_bins %d != 8", K);
    const long long n = rows * T;
    if (n == 0) return NFB_OK;
    (inverse ? spline_bwd_rows_kernel<true> : spline_bwd_rows_kernel<false>)<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        xin, ldx, params, g_out, g_lq, fidx, rows, T, tail, wh_scale, g_params, gx);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Unconditional CDF of the identity features: table [n_id][23] shared by every row.  grid = (row chunks, n_id);
// each thread walks rows of its chunk for ONE feature and keeps 23 partial sums; block reduce, 23 atomics per block.
// INV: the inverse CDF of the sampling direction (see spline_bwd_rows_kernel).
template <bool INV>
__global__ void __launch_bounds__(256) spline_bwd_shared_kernel(
    const float* __restrict__ xin, int ldx, const float* __restrict__ table, const float* __restrict__ g_out,
    const float* __restrict__ g_lq, const int* __restrict__ fidx, long long rows, long long rows_per_block, float tail,
    float* __restrict__ g_table, float* __restrict__ gx) {
    const int i = blockIdx.y;
    const int col = fidx[i];
    const float* tb = table + i * kP;
    float lw[8], lh[8], ud[7];
#pragma unroll
    for (int k = 0; k < 8; ++k) { lw[k] = __ldg(tb + k) * kLog2e; lh[k] = __ldg(tb + 8 + k) * kLog2e; }
#pragma unroll
    for (int k = 0; k < 7; ++k) ud[k] = __ldg(tb + 16 + k);
    float acc[kP];
#pragma unroll
    for (int k = 0; k < kP; ++k) acc[k] = 0.f;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
    for (long long row = r0 + threadIdx.x; row < r1; row += 256) {
        float glw[8], glh[8], gud[7], y, lad, g;
        rqs_dir_fwd_bwd<8, float>(INV, xin[row * ldx + col], lw, lh, ud, tail, g_out[row * ldx + col], g_lq[row], y, lad,
                                  g, glw, glh, gud);
        gx[row * ldx + col] = g;
#pragma unroll
        for (int k = 0; k < 8; ++k) { acc[k] += glw[k]; acc[8 + k] += glh[k]; }
#pragma unroll
        for (int k = 0; k < 7; ++k) acc[16 + k] += gud[k];
    }
    __shared__ float red[8][kP];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < kP; ++k) {
        const float v = warp_sum(acc[k]);
        if (lane == 0) red[w][k] = v;
    }
    __syncthreads();
    if (threadIdx.x < kP) {
        float s = 0.f;
        for (int j = 0; j < 8; ++j) s += red[j][threadIdx.x];
        atomicAdd(g_table + i * kP + threadIdx.x, s * (threadIdx.x < 16 ? kLog2e : 1.f));
    }
}
int launch_spline_bwd_shared(const float* xin, int ldx, const float* table, const float* g_out, const float* g_lq,
                             const int* fidx, long long rows, int n_id, int K, float tail, float* g_table, float* gx,
                             cudaStream_t st, int inverse) {
    NFB_CHECK(K == 8, NFB_ERR_UNSUPPORTED, "spline backward: num_bins %d != 8", K);
    if (rows == 0 || n_id == 0) return NFB_OK;
    const long long rpb = 2048;
    dim3 grid((unsigned)((rows + rpb - 1) / rpb), (unsigned)n_id);
    (inverse ? spline_bwd_shared_kernel<true> : spline_bwd_shared_kernel<false>)<<<grid, 256, 0, st>>>(
        xin, ldx, table, g_out, g_lq, fidx, rows, rpb, tail, g_table, gx);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// ---- stand-alone splines (nfb_rqs_spline / nfb_rqs_spline_tails): density direction (rqs_adjoint_params) and, with
// INV, the sampling direction (rqs_inverse_adjoint_params: x is then the spline's input z, gy the cotangent of its
// output, gx receives g_z).  gin, when given, is added to gy (the fixed-point passes of nfb_ar_rqs_sampling_backward).
// Per-row parameters: one thread per (row, feature) element, 256 consecutive elements per block; the block's
// 256 x P parameter slab is contiguous: staged through shared memory with coalesced loads (P = 2K + nd), the gradient
// slab written back the same way.  KT = 8: the templated fast path (K known at compile time); KT = 0: any K <= 32.
template <int KMAX, bool INV>
__device__ __forceinline__ void spline_element(int K, int nd, bool circ, float x, const float* p, float wh_scale,
                                               float tail, float gy, float gld, float& g, float* gp) {
    float y, lad;
    if (INV)
        rqs_inverse_adjoint_params<KMAX, float>(K, nd, circ, x, p, wh_scale, tail, gy, gld, y, lad, g, gp);
    else
        rqs_adjoint_params<KMAX, float>(K, nd, circ, x, p, wh_scale, tail, gy, gld, y, lad, g, gp);
}

template <int KT, bool INV>
__device__ __forceinline__ void spline_adjoint_rows_body(
    const float* __restrict__ x, const float* __restrict__ params, const float* __restrict__ gy,
    const float* __restrict__ gin, const float* __restrict__ g_ld, long long rows, int feats, int K, int nd,
    const float* __restrict__ tail, const int* __restrict__ circ, float tail0, float wh_scale,
    float* __restrict__ g_params, float* __restrict__ gx) {
    constexpr int KMAX = KT ? KT : 32;
    if (KT) K = KT;
    extern __shared__ float sp[];
    const int P = 2 * K + nd;
    const long long e0 = (long long)blockIdx.x * 256;
    const long long n_el = rows * feats;
    const int n_valid = (int)(n_el - e0 < 256 ? n_el - e0 : 256);
    const float* src = params + e0 * P;
    for (int i = threadIdx.x; i < n_valid * P; i += 256) sp[i] = __ldg(src + i);
    __syncthreads();
    const long long e = e0 + threadIdx.x;
    float gp[3 * KMAX + 1];
    if (e < n_el) {
        const long long row = e / feats;
        const int f = (int)(e - row * feats);
        float g;
        spline_element<KMAX, INV>(K, nd, circ ? circ[f] != 0 : false, x[e], sp + threadIdx.x * P, wh_scale,
                                  tail ? tail[f] : tail0, (gy ? gy[e] : 0.f) + (gin ? gin[e] : 0.f),
                                  g_ld ? g_ld[row] : 0.f, g, gp);
        if (gx) gx[e] = g;
    }
    __syncthreads();
    if (e < n_el)
        for (int k = 0; k < P; ++k) sp[threadIdx.x * P + k] = gp[k];
    __syncthreads();
    if (g_params) {
        float* dst = g_params + e0 * P;
        for (int i = threadIdx.x; i < n_valid * P; i += 256) dst[i] = sp[i];
    }
}

// One parameter table [feats][P] shared by every row (the unconditional CDF of the coupling layers): grid = (row
// chunks, feats); each thread walks rows of its chunk for ONE feature and keeps P partial sums, block reduction, one
// atomic per table entry and block (g_table zeroed by the caller).
template <int KT, bool INV>
__device__ __forceinline__ void spline_adjoint_shared_body(
    const float* __restrict__ x, const float* __restrict__ table, const float* __restrict__ gy,
    const float* __restrict__ gin, const float* __restrict__ g_ld, long long rows, long long rows_per_block, int feats,
    int K, int nd, const float* __restrict__ tail, const int* __restrict__ circ, float tail0, float wh_scale,
    float* __restrict__ g_table, float* __restrict__ gx) {
    constexpr int KMAX = KT ? KT : 32;
    if (KT) K = KT;
    extern __shared__ float red[];  // [8][P]
    const int P = 2 * K + nd;
    const int f = blockIdx.y;
    float p[3 * KMAX + 1], acc[3 * KMAX + 1], gp[3 * KMAX + 1];
    for (int k = 0; k < P; ++k) { p[k] = __ldg(table + (long long)f * P + k); acc[k] = 0.f; }
    const bool c = circ ? circ[f] != 0 : false;
    const float tb = tail ? tail[f] : tail0;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
    for (long long row = r0 + threadIdx.x; row < r1; row += 256) {
        const long long e = row * feats + f;
        float g;
        spline_element<KMAX, INV>(K, nd, c, x[e], p, wh_scale, tb, (gy ? gy[e] : 0.f) + (gin ? gin[e] : 0.f),
                                  g_ld ? g_ld[row] : 0.f, g, gp);
        if (gx) gx[e] = g;
        for (int k = 0; k < P; ++k) acc[k] += gp[k];
    }
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int k = 0; k < P; ++k) {
        const float v = warp_sum(acc[k]);
        if (lane == 0) red[w * P + k] = v;
    }
    __syncthreads();
    if (g_table)
        for (int k = threadIdx.x; k < P; k += 256) {
            float s = 0.f;
            for (int j = 0; j < 8; ++j) s += red[j * P + k];
            atomicAdd(g_table + (long long)f * P + k, s);
        }
}

#define NFB_SPLINE_ROWS_ARGS                                                                                         \
    const float* __restrict__ x, const float* __restrict__ params, const float* __restrict__ gy,                     \
        const float* __restrict__ gin, const float* __restrict__ g_ld, long long rows, int feats, int K, int nd,     \
        const float* __restrict__ tail, const int* __restrict__ circ, float tail0, float wh_scale,                   \
        float *__restrict__ g_params, float *__restrict__ gx
#define NFB_SPLINE_SHARED_ARGS                                                                                       \
    const float* __restrict__ x, const float* __restrict__ table, const float* __restrict__ gy,                      \
        const float* __restrict__ gin, const float* __restrict__ g_ld, long long rows, long long rows_per_block,     \
        int feats, int K, int nd, const float* __restrict__ tail, const int* __restrict__ circ, float tail0,         \
        float wh_scale, float *__restrict__ g_table, float *__restrict__ gx
template <int KT>
__global__ void __launch_bounds__(256) spline_adjoint_rows_kernel(NFB_SPLINE_ROWS_ARGS) {
    spline_adjoint_rows_body<KT, false>(x, params, gy, gin, g_ld, rows, feats, K, nd, tail, circ, tail0, wh_scale,
                                        g_params, gx);
}
template <int KT>
__global__ void __launch_bounds__(256) spline_inverse_adjoint_rows_kernel(NFB_SPLINE_ROWS_ARGS) {
    spline_adjoint_rows_body<KT, true>(x, params, gy, gin, g_ld, rows, feats, K, nd, tail, circ, tail0, wh_scale,
                                       g_params, gx);
}
template <int KT>
__global__ void __launch_bounds__(256) spline_adjoint_shared_kernel(NFB_SPLINE_SHARED_ARGS) {
    spline_adjoint_shared_body<KT, false>(x, table, gy, gin, g_ld, rows, rows_per_block, feats, K, nd, tail, circ,
                                          tail0, wh_scale, g_table, gx);
}
template <int KT>
__global__ void __launch_bounds__(256) spline_inverse_adjoint_shared_kernel(NFB_SPLINE_SHARED_ARGS) {
    spline_adjoint_shared_body<KT, true>(x, table, gy, gin, g_ld, rows, rows_per_block, feats, K, nd, tail, circ,
                                         tail0, wh_scale, g_table, gx);
}
#undef NFB_SPLINE_ROWS_ARGS
#undef NFB_SPLINE_SHARED_ARGS

namespace {
template <bool INV>
int spline_adjoint_launch(const float* x, const float* params, int shared, const float* gy, const float* gin,
                          const float* g_ld, long long rows, int feats, int K, int nd, const float* tail, const int* circ,
                          float tail0, float wh_scale, float* g_params, float* gx, cudaStream_t st) {
    NFB_CHECK(K >= 1 && K <= 32, NFB_ERR_ARG, "rqs backward: num_bins %d out of range [1,32]", K);
    NFB_CHECK(nd == K - 1 || nd == K || nd == K + 1, NFB_ERR_ARG, "rqs backward: %d derivative parameters for %d bins",
              nd, K);
    const int P = 2 * K + nd;
    if (shared && g_params) NFB_CUDA(cudaMemsetAsync(g_params, 0, (size_t)feats * P * 4, st));
    if (rows == 0 || feats == 0) return NFB_OK;
    const bool fast = K == 8;
    auto rows8 = INV ? spline_inverse_adjoint_rows_kernel<8> : spline_adjoint_rows_kernel<8>;
    auto rows0 = INV ? spline_inverse_adjoint_rows_kernel<0> : spline_adjoint_rows_kernel<0>;
    auto shared8 = INV ? spline_inverse_adjoint_shared_kernel<8> : spline_adjoint_shared_kernel<8>;
    auto shared0 = INV ? spline_inverse_adjoint_shared_kernel<0> : spline_adjoint_shared_kernel<0>;
    if (!shared) {
        // dynamic shared memory up to the K = 32 tails-list slab (256 x 97 floats), set once per device
        static PerDevice per_dev;
        if (per_dev.ensure([] {
                const int most = 256 * (3 * 32 + 1) * 4;
                auto r8 = INV ? spline_inverse_adjoint_rows_kernel<8> : spline_adjoint_rows_kernel<8>;
                auto r0 = INV ? spline_inverse_adjoint_rows_kernel<0> : spline_adjoint_rows_kernel<0>;
                cudaError_t e = cudaFuncSetAttribute(r8, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
                return e != cudaSuccess ? e : cudaFuncSetAttribute(r0, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
            }) < 0)
            return NFB_ERR_CUDA;
        const long long n = rows * feats;
        const size_t smem = (size_t)256 * P * 4;
        const unsigned grid = (unsigned)((n + 255) / 256);
        (fast ? rows8 : rows0)<<<grid, 256, smem, st>>>(x, params, gy, gin, g_ld, rows, feats, K, nd, tail, circ, tail0,
                                                        wh_scale, g_params, gx);
    } else {
        const long long rpb = 2048;
        const dim3 grid((unsigned)((rows + rpb - 1) / rpb), (unsigned)feats);
        const size_t smem = (size_t)8 * P * 4;
        (fast ? shared8 : shared0)<<<grid, 256, smem, st>>>(x, params, gy, gin, g_ld, rows, rpb, feats, K, nd, tail,
                                                            circ, tail0, wh_scale, g_params, gx);
    }
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
}  // namespace

int launch_spline_adjoint(const float* x, const float* params, int shared, const float* gy, const float* g_ld,
                          long long rows, int feats, int K, int nd, const float* tail, const int* circ, float tail0,
                          float wh_scale, float* g_params, float* gx, cudaStream_t st) {
    return spline_adjoint_launch<false>(x, params, shared, gy, nullptr, g_ld, rows, feats, K, nd, tail, circ, tail0,
                                        wh_scale, g_params, gx, st);
}
int launch_spline_inverse_adjoint(const float* z, const float* params, int shared, const float* gx, const float* gin,
                                  const float* g_ld, long long rows, int feats, int K, int nd, const float* tail,
                                  const int* circ, float tail0, float wh_scale, float* g_params, float* gz,
                                  cudaStream_t st) {
    return spline_adjoint_launch<true>(z, params, shared, gx, gin, g_ld, rows, feats, K, nd, tail, circ, tail0, wh_scale,
                                       g_params, gz, st);
}

// Adjoint of PeriodicFeaturesElementwise (utils/nn.py:64-130; forward: nfb_kernels.cu periodic_features_kernel).
// grid = (row chunks, dim): each thread walks rows of its chunk for one column, writes gx and, for a periodic column,
// keeps the partial sums of d/dw0 = g sin(s x), d/dw1 = g cos(s x), d/db = g; block reduction, three atomics per block
// (g_w / g_b zeroed by the caller).
__global__ void __launch_bounds__(256) periodic_features_bwd_kernel(
    const float* __restrict__ x, const float* __restrict__ gy, long long rows, long long rows_per_block, int dim,
    const int* __restrict__ slot, const float* __restrict__ w, const float* __restrict__ scale, float* __restrict__ gx,
    float* __restrict__ g_w, float* __restrict__ g_b) {
    const int j = blockIdx.y;
    const int k = slot[j];
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = r0 + rows_per_block < rows ? r0 + rows_per_block : rows;
    const float s = k >= 0 ? scale[k] : 0.f, w0 = k >= 0 ? w[2 * k] : 0.f, w1 = k >= 0 ? w[2 * k + 1] : 0.f;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (long long r = r0 + threadIdx.x; r < r1; r += 256) {
        const long long e = r * dim + j;
        const float g = gy[e];
        if (k < 0) {
            if (gx) gx[e] = g;
            continue;
        }
        float sn, cs;
        sincosf(s * x[e], &sn, &cs);
        if (gx) gx[e] = g * s * (w0 * cs - w1 * sn);
        a0 = fmaf(g, sn, a0); a1 = fmaf(g, cs, a1); a2 += g;
    }
    if (k < 0) return;
    __shared__ float red[3][8];
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    const int wi = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { red[0][wi] = a0; red[1][wi] = a1; red[2][wi] = a2; }
    __syncthreads();
    if (threadIdx.x < 3) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[threadIdx.x][i];
        if (threadIdx.x < 2) { if (g_w) atomicAdd(g_w + 2 * k + threadIdx.x, t); }
        else if (g_b) atomicAdd(g_b + k, t);
    }
}
int launch_periodic_features_bwd(const float* x, const float* gy, long long rows, int dim, const int* slot,
                                 const float* w, const float* scale, int n_periodic, float* gx, float* g_w, float* g_b,
                                 cudaStream_t st) {
    if (g_w) NFB_CUDA(cudaMemsetAsync(g_w, 0, (size_t)n_periodic * 2 * 4, st));
    if (g_b) NFB_CUDA(cudaMemsetAsync(g_b, 0, (size_t)n_periodic * 4, st));
    if (rows == 0 || dim == 0) return NFB_OK;
    const long long rpb = 4096;
    periodic_features_bwd_kernel<<<dim3((unsigned)((rows + rpb - 1) / rpb), (unsigned)dim), 256, 0, st>>>(
        x, gy, rows, rpb, dim, slot, w, scale, gx, g_w, g_b);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out = gate > 0 ? in : slope * in.  LeakyReLU (gate = in) and its adjoint (in = the output gradient, gate = the
// activation, whose sign is that of its argument for slope >= 0) of nets/mlp.py.  In place allowed.
__global__ void leaky_gate_kernel(const float* __restrict__ in, const float* __restrict__ gate, float slope, long long n,
                                  float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = gate[i] > 0.f ? in[i] : slope * in[i];
}
int launch_leaky_gate(const float* in, const float* gate, float slope, long long n, float* out, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    leaky_gate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, gate, slope, n, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[n] += sum_m G[m, n]
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ G, long long ld, long long M, int N,
                                                     long long rows_per_block, float* __restrict__ out) {
    __shared__ float red[8][32];
    const int c = blockIdx.y * 32 + (threadIdx.x & 31);
    const int rl = threadIdx.x >> 5;
    const long long r0 = (long long)blockIdx.x * rows_per_block;
    const long long r1 = r0 + rows_per_block < M ? r0 + rows_per_block : M;
    float s = 0.f;
    if (c < N)
        for (long long r = r0 + rl; r < r1; r += 8) s += G[r * ld + c];
    red[rl][threadIdx.x & 31] = s;
    __syncthreads();
    if (rl == 0 && c < N) {
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) t += red[j][threadIdx.x & 31];
        atomicAdd(out + c, t);
    }
}
int launch_colsum(const float* G, long long ld, long long M, int N, float* out, cudaStream_t st) {
    if (M == 0 || N == 0) return NFB_OK;
    const long long rpb = 1024;
    dim3 grid((unsigned)((M + rpb - 1) / rpb), (unsigned)((N + 31) / 32));
    colsum_kernel<<<grid, 256, 0, st>>>(G, ld, M, N, rpb, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// d log N(z; loc, exp(ls)) / dz = -(z - loc) / sigma^2, scaled by the upstream g_lq[row].
// t_loc / t_ls (optional, [rows x d]): per-element contributions to d/dloc and d/dlog_scale (column-summed by the caller).
__global__ void diag_gauss_bwd_kernel(const float* __restrict__ z, const float* __restrict__ loc,
                                      const float* __restrict__ ls, const float* __restrict__ g_lq, long long rows, int d,
                                      float* __restrict__ gz, float* __restrict__ t_loc, float* __restrict__ t_ls) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * d) return;
    const long long r = i / d;
    const int c = (int)(i - r * d);
    const float inv = __expf(-ls[c]);
    const float u = (z[i] - loc[c]) * inv;  // (z - loc) / sigma
    const float g = g_lq[r];
    gz[i] = -g * u * inv;
    if (t_loc) t_loc[i] = g * u * inv;
    if (t_ls) t_ls[i] = g * (u * u - 1.f);
}
int launch_diag_gauss_bwd(const float* z, const float* loc, const float* ls, const float* g_lq, long long rows, int d,
                          float* gz, float* t_loc, float* t_ls, cudaStream_t st) {
    const long long n = rows * d;
    if (n == 0) return NFB_OK;
    diag_gauss_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(z, loc, ls, g_lq, rows, d, gz, t_loc, t_ls);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// LULinearPermute parameters from dW (gradient of W = L U), flows/mixing.py:402-412 (L unit-lower from
// lower_entries, U = upper_entries + diag(softplus(unconstrained_upper_diag) + eps)) and :514-532
// (logabsdet = sum log diag; `g_logdet` = sum over rows of the upstream gradient on it).  One block, n <= 64.
// NEG: dW and g_logdet enter negated (the sampling direction's map W^-1 (y - b) and its log-det -logabsdet).
template <bool NEG>
__global__ void lu_param_bwd_kernel(const float* __restrict__ dW, const float* __restrict__ lower_e,
                                    const float* __restrict__ upper_e, const float* __restrict__ udiag, float eps, int n,
                                    const float* __restrict__ g_logdet, float* __restrict__ g_lower,
                                    float* __restrict__ g_upper, float* __restrict__ g_udiag) {
    extern __shared__ float shf[];
    float* L = shf;             // n*n
    float* U = shf + n * n;     // n*n
    float* G = shf + 2 * n * n; // n*n
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i % n;
        float l = 0.f, u = 0.f;
        if (c < r) l = lower_e[r * (r - 1) / 2 + c];
        if (c == r) {
            l = 1.f;
            const float d = udiag[r];
            u = (d > 20.f ? d : log1pf(expf(d))) + eps;
        }
        if (c > r) u = upper_e[r * n - r * (r + 1) / 2 + (c - r - 1)];
        L[i] = l; U[i] = u; G[i] = NEG ? -dW[i] : dW[i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i % n;
        if (c < r) {          // dL = dW U^T  (strictly lower part)
            float acc = 0.f;
            for (int k = c; k < n; ++k) acc = fmaf(G[r * n + k], U[c * n + k], acc);
            if (g_lower) g_lower[r * (r - 1) / 2 + c] = acc;
        } else {              // dU = L^T dW  (upper part incl. diagonal)
            float acc = 0.f;
            for (int k = r; k < n; ++k) acc = fmaf(L[k * n + r], G[k * n + c], acc);
            if (c > r) {
                if (g_upper) g_upper[r * n - r * (r + 1) / 2 + (c - r - 1)] = acc;
            } else if (g_udiag) {
                const float d = udiag[r];
                const float sg = d > 20.f ? 1.f : 1.f / (1.f + expf(-d));
                const float gld = g_logdet ? (NEG ? -*g_logdet : *g_logdet) : 0.f;
                g_udiag[r] = (acc + gld / U[r * n + r]) * sg;
            }
        }
    }
}
int launch_lu_param_bwd(const float* dW, const float* lower_e, const float* upper_e, const float* udiag, float eps,
                        int n, const float* g_logdet, float* g_lower, float* g_upper, float* g_udiag, cudaStream_t st,
                        int negate) {
    NFB_CHECK(n >= 1 && n <= 64, NFB_ERR_UNSUPPORTED, "LULinearPermute backward: features %d > 64", n);
    (negate ? lu_param_bwd_kernel<true> : lu_param_bwd_kernel<false>)<<<1, 256, (size_t)3 * n * n * sizeof(float), st>>>(
        dW, lower_e, upper_e, udiag, eps, n, g_logdet, g_lower, g_upper, g_udiag);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[r, idx[j]] (+)= in[r, j]    (scatter by columns: gradient of a column gather / permutation)
__global__ void scatter_cols_kernel(const float* __restrict__ in, float* __restrict__ out, const int* __restrict__ idx,
                                    long long rows, int n_in, int ld_out, int accumulate) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * n_in) return;
    const long long r = i / n_in;
    const int j = (int)(i - r * n_in);
    float* o = out + r * ld_out + idx[j];
    *o = accumulate ? *o + in[i] : in[i];
}
int launch_scatter_cols(const float* in, float* out, const int* idx, long long rows, int n_in, int ld_out, int accumulate,
                        cudaStream_t st) {
    const long long n = rows * n_in;
    if (n == 0) return NFB_OK;
    scatter_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, idx, rows, n_in, ld_out, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[r, j] = in[r * ld_in + idx[j]],  j < n_out   (column gather into a narrower matrix)
__global__ void gather_cols_ld_kernel(const float* __restrict__ in, int ld_in, float* __restrict__ out, int n_out,
                                      const int* __restrict__ idx, long long rows) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * n_out) return;
    const long long r = i / n_out;
    const int j = (int)(i - r * n_out);
    out[i] = in[r * ld_in + idx[j]];
}
int launch_gather_cols_ld(const float* in, int ld_in, float* out, int n_out, const int* idx, long long rows,
                          cudaStream_t st) {
    const long long n = rows * n_out;
    if (n == 0) return NFB_OK;
    gather_cols_ld_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, ld_in, out, n_out, idx, rows);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// y[i] = a * x[i] (+ y[i])
__global__ void axpy_kernel(const float* __restrict__ x, float a, float* __restrict__ y, long long n, int accumulate) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = accumulate ? fmaf(a, x[i], y[i]) : a * x[i];
}
int launch_axpy(const float* x, float a, float* y, long long n, int accumulate, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    axpy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, a, y, n, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// table [n][23] (w(8) | h(8) | d(7) interleaved per feature) -> separate [n x 8], [n x 8], [n x 7] gradient tensors
__global__ void split_table_kernel(const float* __restrict__ tab, int n, float* __restrict__ gw, float* __restrict__ gh,
                                   float* __restrict__ gd) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * kP) return;
    const int f = i / kP, k = i - f * kP;
    if (k < 8) { if (gw) gw[f * 8 + k] = tab[i]; }
    else if (k < 16) { if (gh) gh[f * 8 + k - 8] = tab[i]; }
    else if (gd) gd[f * 7 + k - 16] = tab[i];
}
int launch_split_table(const float* tab, int n, float* gw, float* gh, float* gd, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    split_table_kernel<<<(n * kP + 255) / 256, 256, 0, st>>>(tab, n, gw, gh, gd);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// One pass of the MAF density adjoint (nfb_maf_bwd.cuh), one thread per element: lam = g_y + g_in (g_in, the MADE data
// gradient of the previous pass, NULL on the first), pbar [rows, d, 2] in the MADE output layout, and g_x = lam / scale
// when g_x is given (the last pass).  g_y / g_ld NULL: zero.
__global__ void __launch_bounds__(256) maf_affine_adjoint_kernel(const float* __restrict__ x,
                                                                 const float* __restrict__ params,
                                                                 const float* __restrict__ gy, const float* __restrict__ gld,
                                                                 const float* __restrict__ gin, long long n, int d,
                                                                 float* __restrict__ pbar, float* __restrict__ gx) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float2 p = reinterpret_cast<const float2*>(params)[i];
    const float lam = (gy ? gy[i] : 0.f) + (gin ? gin[i] : 0.f);
    float gu, gs, g;
    maf_affine_adjoint<float>(x[i], p.x, p.y, lam, gld ? gld[i / d] : 0.f, gu, gs, g);
    reinterpret_cast<float2*>(pbar)[i] = make_float2(gu, gs);
    if (gx) gx[i] = g;
}
int launch_maf_affine_adjoint(const float* x, const float* params, const float* gy, const float* gld, const float* gin,
                              long long rows, int d, float* pbar, float* gx, cudaStream_t st) {
    const long long n = rows * d;
    if (n == 0) return NFB_OK;
    maf_affine_adjoint_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, params, gy, gld, gin, n, d, pbar, gx);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
