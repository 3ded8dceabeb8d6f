// nfb_kernels.cu -- generic (any-shape) CUDA kernels of the coupling-stack hot path:
//   * rqs_rows_kernel      stand-alone RQ-spline, per-row parameters from HBM (HBM-bound)
//   * rqs_shared_kernel    RQ-spline with per-feature parameters shared over the batch
//                          (PiecewiseRationalQuadraticCDF, neural_spline/coupling.py:221-253)
//   * linear_kernel        Y = act(X[:,idx]) W^T + b (+R), fp32 FFMA tiles (conditioner nets of
//                          shapes the fused tensor-core kernel does not cover)
//   * pack / log-det / base-density / reduction helpers
// The flagship shapes run through nfb_fused_rqs.cu instead; these kernels are the same
// arithmetic in plain fp32 and serve every other shape.  Built for sm_90a.
#include "nfb_kernels.h"
#include "nfb_spline.cuh"

namespace nfb {

// -----------------------------------------------------------------------------------------
// stand-alone spline, per-row parameters.  One thread per (row, feature) element; the block's
// 256 x P parameter slab is contiguous in HBM, staged through shared memory with 16-byte
// coalesced loads and read back at stride P (odd for the 3K-1 layout -> conflict-free).
// Algorithmic HBM bytes per element: 4*(3K-1) params + 4 x + 4 y  (+ 8/feats for log_det).
// -----------------------------------------------------------------------------------------
constexpr int kSplineBlock = 256;

template <int KT, bool INVERSE>
__global__ void __launch_bounds__(kSplineBlock)
rqs_rows_kernel(const float* __restrict__ zin, const float* __restrict__ params,
                float* __restrict__ zout, float* __restrict__ logdet, long long rows, int feats,
                int ld, const int* __restrict__ fidx, int K, float tail, float wh_scale) {
    extern __shared__ __align__(16) float sp[];
    const int P = 3 * K - 1;
    const long long total = rows * (long long)feats;
    const long long e0 = (long long)blockIdx.x * kSplineBlock;
    const int n_el = (int)min((long long)kSplineBlock, total - e0);
    const float* src = params + e0 * P;
    const int n_f = n_el * P;
    if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(sp);
        const int n4 = n_f >> 2;
        for (int i = threadIdx.x; i < n4; i += kSplineBlock) d4[i] = __ldg(s4 + i);
        for (int i = (n4 << 2) + threadIdx.x; i < n_f; i += kSplineBlock) sp[i] = __ldg(src + i);
    } else {
        for (int i = threadIdx.x; i < n_f; i += kSplineBlock) sp[i] = __ldg(src + i);
    }
    __syncthreads();
    const int t = threadIdx.x;
    float lad = 0.f;
    long long row = -1;
    if (t < n_el) {
        const long long e = e0 + t;
        row = e / feats;
        const int f = (int)(e - row * feats);
        const int col = fidx ? fidx[f] : f;
        const float x = zin[row * ld + col];
        const float* p = sp + t * P;
        auto acc = [p](int i) { return p[i]; };
        float y;
        if (KT > 0)
            rqs_eval<(KT > 0 ? KT : 1), INVERSE>(x, acc, tail, wh_scale, y, lad);
        else
            rqs_eval_dyn<INVERSE>(K, x, acc, tail, wh_scale, y, lad);
        zout[row * ld + col] = y;
    }
    if (logdet) {
        // segmented warp reduction keyed by row; one atomic per (warp, row) segment
        const unsigned lane = threadIdx.x & 31;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_down_sync(0xffffffffu, lad, o);
            const long long r = __shfl_down_sync(0xffffffffu, row, o);
            if (lane + o < 32 && r == row) lad += v;
        }
        const long long rprev = __shfl_up_sync(0xffffffffu, row, 1);
        if (row >= 0 && (lane == 0 || rprev != row)) atomicAdd(logdet + row, lad);
    }
}

// spline with per-feature parameters shared across the batch: table[feats][P] in shared memory.
template <bool INVERSE>
__global__ void __launch_bounds__(256)
rqs_shared_kernel(const float* __restrict__ zin, const float* __restrict__ table,
                  float* __restrict__ zout, float* __restrict__ logdet, long long rows, int feats,
                  int ld, const int* __restrict__ fidx, int K, float tail) {
    extern __shared__ __align__(16) float sp[];
    const int P = 3 * K - 1;
    for (int i = threadIdx.x; i < feats * P; i += blockDim.x) sp[i] = table[i];
    __syncthreads();
    const long long total = rows * (long long)feats;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float lad = 0.f;
    long long row = -1;
    if (e < total) {
        row = e / feats;
        const int f = (int)(e - row * feats);
        const int col = fidx ? fidx[f] : f;
        const float x = zin[row * ld + col];
        const float* p = sp + f * P;
        auto acc = [p](int i) { return p[i]; };
        float y;
        rqs_eval_dyn<INVERSE>(K, x, acc, tail, 1.0f, y, lad);
        zout[row * ld + col] = y;
    }
    if (logdet) {
        const unsigned lane = threadIdx.x & 31;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_down_sync(0xffffffffu, lad, o);
            const long long r = __shfl_down_sync(0xffffffffu, row, o);
            if (lane + o < 32 && r == row) lad += v;
        }
        const long long rprev = __shfl_up_sync(0xffffffffu, row, 1);
        if (row >= 0 && (lane == 0 || rprev != row)) atomicAdd(logdet + row, lad);
    }
}

int launch_rqs_rows(const float* zin, const float* params, float* zout, float* logdet,
                    long long rows, int feats, int ld, const int* fidx, int K, float tail,
                    float wh_scale, int inverse, cudaStream_t st) {
    NFB_CHECK(K >= 1 && K <= 32, NFB_ERR_ARG, "rqs: num_bins %d out of range [1,32]", K);
    NFB_CHECK(kMinBinWidth * K <= 1.0f, NFB_ERR_ARG,
              "Minimal bin width too large for the number of bins");
    if (rows == 0 || feats == 0) return NFB_OK;
    const int P = 3 * K - 1;
    const long long total = rows * (long long)feats;
    const unsigned grid = (unsigned)((total + kSplineBlock - 1) / kSplineBlock);
    const size_t smem = (size_t)kSplineBlock * P * sizeof(float);
#define NFB_RQS_LAUNCH(KT, INV)                                                               \
    do {                                                                                      \
        NFB_CUDA(cudaFuncSetAttribute(rqs_rows_kernel<KT, INV>,                               \
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        rqs_rows_kernel<KT, INV><<<grid, kSplineBlock, smem, st>>>(                           \
            zin, params, zout, logdet, rows, feats, ld, fidx, K, tail, wh_scale);             \
    } while (0)
    if (K == 8) {
        if (inverse) NFB_RQS_LAUNCH(8, true); else NFB_RQS_LAUNCH(8, false);
    } else {
        if (inverse) NFB_RQS_LAUNCH(0, true); else NFB_RQS_LAUNCH(0, false);
    }
#undef NFB_RQS_LAUNCH
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// stand-alone spline with PER-FEATURE tails (circular NSF layers, flows/neural_spline/wrapper.py:88-183,247-311;
// utils/splines.py:42-57): nd derivative parameters per element (K + 1 for a tails list, K for all-circular),
// circ[f] != 0 = circular feature, tail[f] = that feature's bound.  One thread per element, parameters read in place
// (breadth path: the flagship shapes never come here).
// -----------------------------------------------------------------------------------------
template <bool INVERSE>
__global__ void __launch_bounds__(256)
rqs_rows_tails_kernel(const float* __restrict__ zin, const float* __restrict__ params, float* __restrict__ zout,
                      float* __restrict__ logdet, long long rows, int feats, int K, int nd,
                      const float* __restrict__ tail, const int* __restrict__ circ, float wh_scale) {
    const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long total = rows * (long long)feats;
    float lad = 0.f;
    long long row = -1;
    if (e < total) {
        row = e / feats;
        const int f = (int)(e - row * feats);
        const float* p = params + e * (long long)(2 * K + nd);
        auto acc = [p](int i) { return __ldg(p + i); };
        float y;
        rqs_eval_dyn<INVERSE>(K, zin[e], acc, __ldg(tail + f), wh_scale, y, lad, nd, __ldg(circ + f) != 0);
        zout[e] = y;
    }
    if (logdet) {
        const unsigned lane = threadIdx.x & 31;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const float v = __shfl_down_sync(0xffffffffu, lad, o);
            const long long r = __shfl_down_sync(0xffffffffu, row, o);
            if (lane + o < 32 && r == row) lad += v;
        }
        const long long prev = __shfl_up_sync(0xffffffffu, row, 1);
        if (row >= 0 && (lane == 0 || prev != row)) atomicAdd(logdet + row, lad);
    }
}
int launch_rqs_rows_tails(const float* zin, const float* params, float* zout, float* logdet, long long rows, int feats,
                          int K, int nd, const float* tail, const int* circ, float wh_scale, int inverse,
                          cudaStream_t st) {
    NFB_CHECK(K >= 1 && K <= 32, NFB_ERR_ARG, "rqs: num_bins %d out of range [1,32]", K);
    NFB_CHECK(nd == K || nd == K + 1, NFB_ERR_ARG, "rqs tails: %d derivative parameters for %d bins", nd, K);
    if (rows == 0 || feats == 0) return NFB_OK;
    const long long total = rows * (long long)feats;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (inverse) rqs_rows_tails_kernel<true><<<grid, 256, 0, st>>>(zin, params, zout, logdet, rows, feats, K, nd, tail, circ, wh_scale);
    else rqs_rows_tails_kernel<false><<<grid, 256, 0, st>>>(zin, params, zout, logdet, rows, feats, K, nd, tail, circ, wh_scale);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// PeriodicFeaturesElementwise (utils/nn.py:64-130): y[r, j] = w[j,0] sin(s[j] x) + w[j,1] cos(s[j] x) (+ b[j]) where
// kind[j] >= 0 is the feature's slot in the periodic parameter tables, y = x elsewhere.
__global__ void periodic_features_kernel(const float* __restrict__ x, float* __restrict__ y, long long rows, int dim,
                                         const int* __restrict__ slot, const float* __restrict__ w,
                                         const float* __restrict__ scale, const float* __restrict__ bias) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= rows * dim) return;
    const int j = (int)(e % dim);
    const int k = slot[j];
    float v = x[e];
    if (k >= 0) {
        const float a = scale[k] * v;
        v = w[2 * k] * sinf(a) + w[2 * k + 1] * cosf(a);
        if (bias) v += bias[k];
    }
    y[e] = v;
}
int launch_periodic_features(const float* x, float* y, long long rows, int dim, const int* slot, const float* w,
                             const float* scale, const float* bias, cudaStream_t st) {
    if (rows == 0 || dim == 0) return NFB_OK;
    const long long n = rows * dim;
    periodic_features_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, y, rows, dim, slot, w, scale, bias);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_rqs_shared(const float* zin, const float* table, float* zout, float* logdet,
                      long long rows, int feats, int ld, const int* fidx, int K, float tail,
                      int inverse, cudaStream_t st) {
    NFB_CHECK(K >= 1 && K <= 32, NFB_ERR_ARG, "rqs: num_bins %d out of range [1,32]", K);
    if (rows == 0 || feats == 0) return NFB_OK;
    const int P = 3 * K - 1;
    const size_t smem = (size_t)feats * P * sizeof(float);
    NFB_CHECK(smem <= 200 * 1024, NFB_ERR_UNSUPPORTED, "rqs_shared: table too large");
    const long long total = rows * (long long)feats;
    const unsigned grid = (unsigned)((total + 255) / 256);
    if (inverse) {
        NFB_CUDA(cudaFuncSetAttribute(rqs_shared_kernel<true>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rqs_shared_kernel<true><<<grid, 256, smem, st>>>(zin, table, zout, logdet, rows, feats, ld,
                                                         fidx, K, tail);
    } else {
        NFB_CUDA(cudaFuncSetAttribute(rqs_shared_kernel<false>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        rqs_shared_kernel<false><<<grid, 256, smem, st>>>(zin, table, zout, logdet, rows, feats, ld,
                                                          fidx, K, tail);
    }
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// Y[M,N] = act_in(X[:, idx])[M,K] * W[N,K]^T + b[N] (+ R[M,N]);  act_out applied last.
// act: 0 none, 1 relu, 2 leaky-relu(slope).  fp32 FFMA, 64x64 block tile, 4x4 per thread.
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    if (act == 1) return fmaxf(v, 0.f);
    if (act == 2) return v >= 0.f ? v : v * slope;
    return v;
}

__global__ void __launch_bounds__(256)
linear_kernel(const float* __restrict__ X, int ldx, const int* __restrict__ xidx,
              const float* __restrict__ W, const float* __restrict__ bias,
              const float* __restrict__ R, int ldr, float* __restrict__ Y, int ldy,
              long long M, int N, int K, int act_in, int act_out, float slope) {
    __shared__ float As[16][64 + 1];
    __shared__ float Bs[16][64 + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const long long m0 = (long long)blockIdx.x * 64;
    const int n0 = blockIdx.y * 64;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
        for (int i = threadIdx.x; i < 64 * 16; i += 256) {
            const int r = i >> 4, k = i & 15;
            const long long m = m0 + r;
            float a = 0.f, b = 0.f;
            if (k0 + k < K) {
                const int kk = xidx ? xidx[k0 + k] : (k0 + k);
                if (m < M) a = apply_act(X[m * ldx + kk], act_in, slope);
                if (n0 + r < N) b = W[(long long)(n0 + r) * K + k0 + k];
            }
            As[k][r] = a;
            Bs[k][r] = b;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                a[i] = As[k][ty * 4 + i];
                b[i] = Bs[k][tx * 4 + i];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long m = m0 + ty * 4 + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= N) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (R) v += R[m * ldr + n];
            Y[m * ldy + n] = apply_act(v, act_out, slope);
        }
    }
}

int launch_linear(const float* X, int ldx, const int* xidx, const float* W, const float* bias,
                  const float* R, int ldr, float* Y, int ldy, long long M, int N, int K, int act_in,
                  int act_out, float slope, cudaStream_t st) {
    if (M == 0 || N == 0) return NFB_OK;
    dim3 grid((unsigned)((M + 63) / 64), (unsigned)((N + 63) / 64));
    linear_kernel<<<grid, 256, 0, st>>>(X, ldx, xidx, W, bias, R, ldr, Y, ldy, M, N, K, act_in,
                                        act_out, slope);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// parameter packing helpers (run when parameters change, not per step)
// -----------------------------------------------------------------------------------------
// out[i] = w[i] * mask[i]   (nets/made.py:80-81 does this on every call)
__global__ void mask_mul_kernel(const float* __restrict__ w, const float* __restrict__ m,
                                float* __restrict__ out, long long n) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = m ? w[i] * m[i] : w[i];
}
int launch_mask_mul(const float* w, const float* m, float* out, long long n, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    mask_mul_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, m, out, n);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// _LULinear (flows/mixing.py:402-412,:514-532): builds W = L U  [n,n] (row-major, y = x W^T + b),
// Winv = (L U)^-1 (for the sampling direction, :436-473), and logabsdet = sum log(softplus(d)+eps).
// One block; n <= 64.  Triangular entries are packed row-major (np.tril_indices / np.triu_indices).
__device__ __forceinline__ void lu_pack_block(const float* __restrict__ lower_e, const float* __restrict__ upper_e,
                                              const float* __restrict__ udiag, float eps, int n,
                                              float* __restrict__ Wout, float* __restrict__ Winv,
                                              float* __restrict__ logabsdet) {
    extern __shared__ double sh[];
    double* L = sh;               // n*n
    double* U = sh + n * n;       // n*n
    double* Li = sh + 2 * n * n;  // n*n  (L^-1)
    double* Ui = sh + 3 * n * n;  // n*n  (U^-1)
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i % n;
        double l = 0.0, u = 0.0;
        if (c < r) l = lower_e[r * (r - 1) / 2 + c];
        if (c == r) l = 1.0;
        if (c > r) u = upper_e[r * n - r * (r + 1) / 2 + (c - r - 1)];
        if (c == r) {
            const float d = udiag[r];
            const float sp = d > 20.f ? d : log1pf(expf(d));
            u = (double)(sp + eps);
        }
        L[i] = l;
        U[i] = u;
        Li[i] = 0.0;
        Ui[i] = 0.0;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int r = 0; r < n; ++r) s += logf((float)U[r * n + r]);
        *logabsdet = s;
    }
    // W = L U in the reference's fp32 arithmetic class (F.linear twice); we form it once.
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i % n;
        float acc = 0.f;
        for (int k = 0; k <= min(r, c); ++k) acc = fmaf((float)L[r * n + k], (float)U[k * n + c], acc);
        Wout[i] = acc;
    }
    // inverses by substitution, one column per thread (fp64; n <= 64)
    for (int c = threadIdx.x; c < n; c += blockDim.x) {
        for (int r = 0; r < n; ++r) {  // L^-1 column c (unit lower)
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = c; k < r; ++k) v -= L[r * n + k] * Li[k * n + c];
            Li[r * n + c] = (r < c) ? 0.0 : v;
        }
        for (int r = n - 1; r >= 0; --r) {  // U^-1 column c (upper)
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = r + 1; k <= c; ++k) v -= U[r * n + k] * Ui[k * n + c];
            Ui[r * n + c] = (r > c) ? 0.0 : v / U[r * n + r];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int r = i / n, c = i % n;
        double acc = 0.0;  // (LU)^-1 = U^-1 L^-1
        for (int k = max(r, c); k < n; ++k) acc += Ui[r * n + k] * Li[k * n + c];
        Winv[i] = (float)acc;
    }
}
__global__ void lu_pack_kernel(const float* __restrict__ lower_e, const float* __restrict__ upper_e,
                               const float* __restrict__ udiag, float eps, int n, float* __restrict__ Wout,
                               float* __restrict__ Winv, float* __restrict__ logabsdet) {
    lu_pack_block(lower_e, upper_e, udiag, eps, n, Wout, Winv, logabsdet);
}
// every LU layer of a flow in ONE launch, one block per layer (32 serialised single-block launches dominated the
// packing phase of a 32-layer stack)
__global__ void lu_pack_batched_kernel(const LuPackArgs* __restrict__ args) {
    const LuPackArgs a = args[blockIdx.x];
    lu_pack_block(a.lower_e, a.upper_e, a.udiag, a.eps, a.n, a.W, a.Winv, a.logabsdet);
}
int launch_lu_pack_batched(const LuPackArgs* args_dev, int count, int n_max, cudaStream_t st) {
    if (count == 0) return NFB_OK;
    NFB_CHECK(n_max >= 1 && n_max <= 64, NFB_ERR_UNSUPPORTED, "LULinearPermute: features %d > 64", n_max);
    const size_t smem = (size_t)4 * n_max * n_max * sizeof(double);
    NFB_CUDA(cudaFuncSetAttribute(lu_pack_batched_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lu_pack_batched_kernel<<<count, 256, smem, st>>>(args_dev);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
int launch_lu_pack(const float* lower_e, const float* upper_e, const float* udiag, float eps, int n,
                   float* W, float* Winv, float* logabsdet, cudaStream_t st) {
    NFB_CHECK(n >= 1 && n <= 64, NFB_ERR_UNSUPPORTED, "LULinearPermute: features %d > 64", n);
    const size_t smem = (size_t)4 * n * n * sizeof(double);
    NFB_CUDA(cudaFuncSetAttribute(lu_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    lu_pack_kernel<<<1, 256, smem, st>>>(lower_e, upper_e, udiag, eps, n, W, Winv, logabsdet);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// small elementwise pieces of the driver loop (core.py:96-102)
// -----------------------------------------------------------------------------------------
__global__ void add_scalar_kernel(float* __restrict__ v, long long n, const float* __restrict__ c,
                                  float sign) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] += sign * (*c);
}
int launch_add_scalar(float* v, long long n, const float* c, float sign, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    add_scalar_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(v, n, c, sign);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

__global__ void fill_kernel(float* __restrict__ v, long long n, float c) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) v[i] = c;
}
int launch_fill(float* v, long long n, float c, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(v, n, c);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[r, j] = in[r, idx[j]]   (flows/mixing.py:239 index_select; Permute :31-54)
__global__ void gather_cols_kernel(const float* __restrict__ in, float* __restrict__ out,
                                   const int* __restrict__ idx, long long rows, int d, long long inner) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long per = (long long)d * inner;
    if (i >= rows * per) return;
    const long long r = i / per;
    const long long rem = i - r * per;
    const int j = (int)(rem / inner);
    const long long in_off = rem - (long long)j * inner;
    out[i] = in[r * per + (long long)idx[j] * inner + in_off];
}
int launch_gather_cols(const float* in, float* out, const int* idx, long long rows, int d,
                       long long inner, cudaStream_t st) {
    const long long n = rows * d * inner;
    if (n == 0) return NFB_OK;
    gather_cols_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, idx, rows, d, inner);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// DiagGaussian.log_prob (distributions/base.py:94-103), accumulated into log_q:
//   log_q[r] += -d/2 log(2 pi) - sum_j (ls_j + 0.5 ((z_rj - loc_j) / exp(ls_j))^2)
// One warp per row.
__global__ void __launch_bounds__(256)
diag_gauss_kernel(const float* __restrict__ z, const float* __restrict__ loc,
                  const float* __restrict__ log_scale, float* __restrict__ logq, long long rows,
                  int d, int accumulate) {
    const long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float s = 0.f;
    for (int j = lane; j < d; j += 32) {
        const float ls = log_scale[j];
        const float t = (z[row * d + j] - loc[j]) / expf(ls);
        s += ls + 0.5f * t * t;
    }
    s = warp_sum(s);
    if (lane == 0) {
        const float lp = -0.5f * (float)d * 1.8378770664093453f - s;
        logq[row] = accumulate ? logq[row] + lp : lp;
    }
}
int launch_diag_gauss(const float* z, const float* loc, const float* log_scale, float* logq,
                      long long rows, int d, int accumulate, cudaStream_t st) {
    if (rows == 0) return NFB_OK;
    const long long threads = rows * 32;
    diag_gauss_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(z, loc, log_scale, logq,
                                                                         rows, d, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Deterministic sum of v[0..n) -> out[0] = scale * sum (two-stage, fixed tree order).
__global__ void __launch_bounds__(256)
sum_stage1_kernel(const float* __restrict__ v, long long n, double* __restrict__ partial) {
    __shared__ double sh[8];
    double s = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        s += (double)v[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 8; ++i) t += sh[i];
        partial[blockIdx.x] = t;
    }
}
__global__ void sum_stage2_kernel(const double* __restrict__ partial, int np, double scale, long long n,
                                  float* __restrict__ out, double* __restrict__ out_sum) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < np; ++i) t += partial[i];
        if (out_sum) { out_sum[0] = t; out_sum[1] = (double)n; }  // [sum, count]: the all-reduce operand
        if (out) *out = (float)(t * scale);
    }
}
int launch_sum(const float* v, long long n, double scale, double* scratch /*>=1024*/, float* out,
               double* out_sum, cudaStream_t st) {
    int nb = (int)min((long long)592, (n + 255) / 256);
    if (nb < 1) nb = 1;
    sum_stage1_kernel<<<nb, 256, 0, st>>>(v, n, scratch);
    sum_stage2_kernel<<<1, 32, 0, st>>>(scratch, nb, scale, n, out, out_sum);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// Masked affine autoregressive flow, element-wise part (flows/affine/autoregressive.py:96-128):
//   params [rows, D, 2] = (unconstrained_scale, shift) per feature; scale = sigmoid(u + 2) + 1e-3
//   forward: y = scale x + shift, log_det += sum log scale;   inverse: y = (x - shift) / scale, log_det -= sum log scale
// One warp per row (lanes stride the features), shuffle reduction of the log-det.  HBM-bound: 16 B per element.
// -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) maf_affine_kernel(const float* __restrict__ x, const float* __restrict__ params,
                                                         float* __restrict__ y, float* __restrict__ logdet,
                                                         long long rows, int d, int inverse, int accumulate) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float acc = 0.f;
    for (int j = lane; j < d; j += 32) {
        const float2 p = reinterpret_cast<const float2*>(params + row * 2 * d)[j];
        const float scale = 1.f / (1.f + expf(-(p.x + 2.f))) + 1e-3f;
        const float ls = logf(scale);
        const float v = x[row * d + j];
        y[row * d + j] = inverse ? (v - p.y) / scale : fmaf(scale, v, p.y);
        acc += inverse ? -ls : ls;
    }
    acc = warp_sum(acc);
    if (lane == 0 && logdet) logdet[row] = accumulate ? logdet[row] + acc : acc;
}
int launch_maf_affine(const float* x, const float* params, float* y, float* logdet, long long rows, int d, int inverse,
                      int accumulate, cudaStream_t st) {
    if (rows == 0 || d == 0) return NFB_OK;
    maf_affine_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(x, params, y, logdet, rows, d, inverse, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb

