// nfb_mixture.cu -- the Gaussian-mixture base (reference distributions/base.py:573-659 GaussianMixture): its
// log-density and the adjoint, for any number of modes K >= 1 and any number of features D.
//
// Density: one launch, one thread per row, kMixRows rows per CTA.  Every CTA forms the per-mode constants from the
// parameters itself -- logsumexp(weight_scores), exp(-log_scale) -- so an optimizer step needs no repack and no host
// sync.  The parameters are staged in shared memory in tiles of kMixModes modes x kMixFeat features, next to the CTA's
// rows of z (transposed, so a thread reads its row without bank conflicts); a thread keeps the tile's kMixModes partial
// exponents in registers and folds each finished mode into a streaming (max-subtracted) log-sum-exp.  So K and D are
// bounded by nothing but the index types.
//
// Backward: two launches whatever the rows, K and D.
//   mixture_bwd_kernel   a fixed grid of at most kMixMaxParts CTAs walks the row blocks (block b on CTA b % grid, in
//                        order).  Per block: the rows' log p (pass 1), then per mode tile the responsibilities
//                        a_rk = g_r resp_rk into shared memory, g_z of the rows, and one thread per (mode, feature)
//                        element walking the block's rows in order into the CTA's partial sums of g_loc, g_log_scale;
//                        sum_r a_rk and sum_r g_r complete the partials.
//   mixture_bwd_sum_kernel  sums the CTAs' partials in CTA order (fp64) and forms g_ws = sum a - softmax(ws) sum g.
// No atomics: two calls give identical bits.  The workspace is grid x (2 K D + K + 1) floats, under kMixWsCap bytes
// unless a single partial is larger; it does not grow with the rows.
#include "nfb_kernels.h"
#include "nfb_mixture.cuh"

#include <algorithm>

namespace nfb {

namespace {

constexpr int kMixRows = 128;     // rows per CTA (one per thread)
constexpr int kMixModes = 16;     // modes per shared-memory tile
constexpr int kMixFeat = 32;      // features per shared-memory tile
constexpr int kMixMaxParts = 256;
constexpr long long kMixWsCap = 64ll << 20;

struct MixTile {
    float z[kMixFeat][kMixRows + 1];  // z[d][r]: row r of the CTA, feature d0 + d
    float4 p[kMixModes][kMixFeat];    // (loc, exp(-log_scale), log_scale, 0) of mode k0 + kk, feature d0 + d
};

// stage the CTA's rows and the parameters of modes [k0, k0 + nk) x features [d0, d0 + nd); modes past nk get
// (0, 1, 0) so the unrolled loops read defined values
__device__ __forceinline__ void mix_stage(MixTile& t, const float* __restrict__ z, long long row0, long long rows, int D,
                                          const float* __restrict__ loc, const float* __restrict__ log_scale, int k0,
                                          int nk, int d0, int nd) {
    __syncthreads();   // the previous tile is no longer read
    for (int i = threadIdx.x; i < kMixRows * nd; i += kMixRows) {
        const int r = i / nd, d = i - r * nd;
        const long long row = row0 + r;
        t.z[d][r] = row < rows ? z[row * D + d0 + d] : 0.f;
    }
    for (int i = threadIdx.x; i < kMixModes * nd; i += kMixRows) {
        const int kk = i / nd, d = i - kk * nd;
        float4 v = make_float4(0.f, 1.f, 0.f, 0.f);
        if (kk < nk) {
            const long long j = (long long)(k0 + kk) * D + d0 + d;
            const float ls = log_scale[j];
            v = make_float4(loc[j], expf(-ls), ls, 0.f);
        }
        t.p[kk][d] = v;
    }
    __syncthreads();
}

// quad[kk] = sum_d mix_quad_term over all D features of mode k0 + kk, for this thread's row
__device__ __forceinline__ void mix_tile_quads(MixTile& t, const float* __restrict__ z, long long row0, long long rows,
                                               int D, const float* __restrict__ loc,
                                               const float* __restrict__ log_scale, int k0, int nk,
                                               float (&quad)[kMixModes]) {
#pragma unroll
    for (int kk = 0; kk < kMixModes; ++kk) quad[kk] = 0.f;
    for (int d0 = 0; d0 < D; d0 += kMixFeat) {
        const int nd = min(kMixFeat, D - d0);
        mix_stage(t, z, row0, rows, D, loc, log_scale, k0, nk, d0, nd);
        for (int d = 0; d < nd; ++d) {
            const float zv = t.z[d][threadIdx.x];
#pragma unroll
            for (int kk = 0; kk < kMixModes; ++kk) {
                const float4 p = t.p[kk][d];
                quad[kk] += mix_quad_term(zv, p.x, p.y, p.z);
            }
        }
    }
}

// log p of this thread's row (pass over every mode)
__device__ __forceinline__ float mix_row_lse(MixTile& t, const float* __restrict__ z, long long row0, long long rows,
                                             int K, int D, const float* __restrict__ loc,
                                             const float* __restrict__ log_scale, const float* __restrict__ ws,
                                             float wl) {
    float m = -INFINITY, s = 0.f;
    for (int k0 = 0; k0 < K; k0 += kMixModes) {
        const int nk = min(kMixModes, K - k0);
        float quad[kMixModes];
        mix_tile_quads(t, z, row0, rows, D, loc, log_scale, k0, nk, quad);
#pragma unroll
        for (int kk = 0; kk < kMixModes; ++kk)
            if (kk < nk) mix_lse_push(m, s, mix_mode_exponent(__ldg(ws + k0 + kk), wl, D, quad[kk]));
    }
    return mix_lse_value(m, s);
}

__global__ void __launch_bounds__(kMixRows) mixture_log_prob_kernel(
    const float* __restrict__ z, const float* __restrict__ loc, const float* __restrict__ log_scale,
    const float* __restrict__ ws, float* __restrict__ log_q, long long rows, int K, int D, int accumulate) {
    __shared__ MixTile t;
    const float wl = mix_weight_lse(ws, K);
    const long long row0 = (long long)blockIdx.x * kMixRows, row = row0 + threadIdx.x;
    const float lp = mix_row_lse(t, z, row0, rows, K, D, loc, log_scale, ws, wl);
    if (row < rows) log_q[row] = accumulate ? log_q[row] + lp : lp;
}

__global__ void __launch_bounds__(kMixRows) mixture_bwd_kernel(
    const float* __restrict__ z, const float* __restrict__ loc, const float* __restrict__ log_scale,
    const float* __restrict__ ws, const float* __restrict__ g_lq, float* __restrict__ g_z, float* __restrict__ part,
    long long rows, int K, int D) {
    __shared__ MixTile t;
    __shared__ float a_s[kMixModes][kMixRows];
    __shared__ float g_s[kMixRows];
    const float wl = mix_weight_lse(ws, K);
    const long long KD = (long long)K * D;
    float* P = part + (long long)blockIdx.x * (2 * KD + K + 1);
    const long long n_blk = (rows + kMixRows - 1) / kMixRows;
    bool first = true;
    for (long long b = blockIdx.x; b < n_blk; b += gridDim.x, first = false) {
        const long long row0 = b * kMixRows, row = row0 + threadIdx.x;
        const bool valid = row < rows;
        const float g = valid ? g_lq[row] : 0.f;
        const float lp = mix_row_lse(t, z, row0, rows, K, D, loc, log_scale, ws, wl);
        for (int k0 = 0; k0 < K; k0 += kMixModes) {
            const int nk = min(kMixModes, K - k0);
            float quad[kMixModes];
            mix_tile_quads(t, z, row0, rows, D, loc, log_scale, k0, nk, quad);
#pragma unroll
            for (int kk = 0; kk < kMixModes; ++kk)
                a_s[kk][threadIdx.x] = (valid && kk < nk)
                    ? g * expf(mix_mode_exponent(__ldg(ws + k0 + kk), wl, D, quad[kk]) - lp) : 0.f;
            for (int d0 = 0; d0 < D; d0 += kMixFeat) {
                const int nd = min(kMixFeat, D - d0);
                mix_stage(t, z, row0, rows, D, loc, log_scale, k0, nk, d0, nd);   // (also publishes a_s)
                if (g_z && valid) {
                    for (int d = 0; d < nd; ++d) {
                        const float zv = t.z[d][threadIdx.x];
                        float acc = 0.f;
#pragma unroll
                        for (int kk = 0; kk < kMixModes; ++kk) {
                            const float4 p = t.p[kk][d];
                            acc += a_s[kk][threadIdx.x] * ((zv - p.x) * p.y) * p.y;
                        }
                        float* o = g_z + row * D + d0 + d;
                        *o = (k0 == 0 ? 0.f : *o) - acc;
                    }
                }
                for (int i = threadIdx.x; i < nk * nd; i += kMixRows) {
                    const int kk = i / nd, d = i - kk * nd;
                    const float4 p = t.p[kk][d];
                    float gl = 0.f, gs = 0.f;
                    for (int r = 0; r < kMixRows; ++r) {
                        const float a = a_s[kk][r];
                        const float tt = (t.z[d][r] - p.x) * p.y;
                        gl += a * tt * p.y;
                        gs += a * (tt * tt - 1.f);
                    }
                    const long long j = (long long)(k0 + kk) * D + d0 + d;
                    P[j] = first ? gl : P[j] + gl;
                    P[KD + j] = first ? gs : P[KD + j] + gs;
                }
            }
            if (threadIdx.x < nk) {
                float sa = 0.f;
                for (int r = 0; r < kMixRows; ++r) sa += a_s[threadIdx.x][r];
                float* o = P + 2 * KD + k0 + threadIdx.x;
                *o = first ? sa : *o + sa;
            }
        }
        g_s[threadIdx.x] = g;
        __syncthreads();
        if (threadIdx.x == 0) {
            float sg = 0.f;
            for (int r = 0; r < kMixRows; ++r) sg += g_s[r];
            P[2 * KD + K] = first ? sg : P[2 * KD + K] + sg;
        }
        // (g_s is rewritten only after the next block's first mix_stage barrier)
    }
}

__global__ void mixture_bwd_sum_kernel(const float* __restrict__ part, int n_parts, const float* __restrict__ ws,
                                       int K, int D, float* __restrict__ g_loc, float* __restrict__ g_log_scale,
                                       float* __restrict__ g_ws) {
    const long long KD = (long long)K * D, stride = 2 * KD + K + 1;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 2 * KD + K) return;
    double acc = 0.0;
    for (int c = 0; c < n_parts; ++c) acc += part[c * stride + idx];
    if (idx < KD) {
        if (g_loc) g_loc[idx] = (float)acc;
    } else if (idx < 2 * KD) {
        if (g_log_scale) g_log_scale[idx - KD] = (float)acc;
    } else if (g_ws) {
        double sg = 0.0;
        for (int c = 0; c < n_parts; ++c) sg += part[c * stride + 2 * KD + K];
        const int k = (int)(idx - 2 * KD);
        g_ws[k] = (float)(acc - (double)expf(ws[k] - mix_weight_lse(ws, K)) * sg);
    }
}

int mixture_parts(long long rows, int K, int D) {
    const long long n_blk = (rows + kMixRows - 1) / kMixRows;
    const long long per = (2ll * K * D + K + 1) * 4;
    const long long cap = std::max(1ll, std::min((long long)kMixMaxParts, kMixWsCap / per));
    return (int)std::min(n_blk, cap);
}

}  // namespace

int launch_mixture_log_prob(const float* z, const float* loc, const float* log_scale, const float* ws, float* log_q,
                            long long rows, int K, int D, int accumulate, cudaStream_t st) {
    NFB_CHECK(K >= 1 && D >= 1, NFB_ERR_ARG, "gaussian mixture: n_modes %d and dim %d must be >= 1", K, D);
    if (rows == 0) return NFB_OK;
    const long long blocks = (rows + kMixRows - 1) / kMixRows;
    NFB_CHECK(blocks < (1ll << 31), NFB_ERR_ARG, "gaussian mixture: %lld rows", rows);
    mixture_log_prob_kernel<<<(unsigned)blocks, kMixRows, 0, st>>>(z, loc, log_scale, ws, log_q, rows, K, D,
                                                                    accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

long long mixture_bwd_ws_bytes(long long rows, int K, int D) {
    return (long long)mixture_parts(rows, K, D) * (2ll * K * D + K + 1) * 4;
}

int launch_mixture_bwd(const float* z, const float* loc, const float* log_scale, const float* ws, const float* g_lq,
                       long long rows, int K, int D, void* wsp, long long ws_bytes, float* g_z, float* g_loc,
                       float* g_log_scale, float* g_ws, cudaStream_t st) {
    NFB_CHECK(K >= 1 && D >= 1, NFB_ERR_ARG, "gaussian mixture: n_modes %d and dim %d must be >= 1", K, D);
    const int n_parts = mixture_parts(rows, K, D);
    NFB_CHECK(ws_bytes >= mixture_bwd_ws_bytes(rows, K, D) && (n_parts == 0 || wsp), NFB_ERR_ARG,
              "gaussian mixture backward: workspace of %lld bytes, needs %lld", ws_bytes,
              mixture_bwd_ws_bytes(rows, K, D));
    float* part = static_cast<float*>(wsp);
    if (n_parts > 0)
        mixture_bwd_kernel<<<n_parts, kMixRows, 0, st>>>(z, loc, log_scale, ws, g_lq, g_z, part, rows, K, D);
    const long long n_out = 2ll * K * D + K;
    NFB_CHECK(n_out / 256 < (1ll << 31), NFB_ERR_ARG, "gaussian mixture: %d x %d parameters", K, D);
    mixture_bwd_sum_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, st>>>(part, n_parts, ws, K, D, g_loc,
                                                                             g_log_scale, g_ws);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
