// nfb_residual.cu -- element-wise kernels of the invertible residual block (flows/residual.py:12-251 `Residual` /
// `iResBlock`) with a Lipschitz MLP (nets/lipschitz.py:14-67: [Swish, InducedNormLinear] x n).
//
// The Linear layers of g(x), of its Jacobian-vector products (forward mode: the exact 2 x 2 Jacobian of the 2-D eval
// path, residual.py:148-161) and of its vector-Jacobian products (reverse mode: the Hutchinson power series,
// :355-379) are tensor-core GEMMs (csrc/nfb_gemm_tc.cu); what is left is element-wise and HBM-bound:
//   swish        a = x sigmoid(b x) / 1.1,  da = d a / d x          (nets/lipschitz.py:642-648, b = softplus(beta))
//   mul_rows     T[t, i] *= m[i]                                     (tangents / cotangents through the activation)
//   logdet2      log |det(I + J)| for [B, 2, 2] Jacobians given as two tangent outputs
//   rowdot       out[r] (+)= c * sum_j a[r, j] b[r, j]              (trace estimate v^T J^k eps per sample)
// and those of the training pass (nfb_lipschitz_mlp_dual_backward, nfb_api.cu): swish_dual / swish_dual_adjoint (the
// activation of the network pushed forward with its tangents, and its adjoint) and logdet2_backward.
#include "nfb_kernels.h"

#include <algorithm>

namespace nfb {

__global__ void swish_kernel(const float* __restrict__ x, float b, long long n, float* __restrict__ a,
                             float* __restrict__ da) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = x[i];
    const float s = 1.f / (1.f + __expf(-b * v));
    a[i] = v * s * (1.f / 1.1f);
    if (da) da[i] = (s + b * v * s * (1.f - s)) * (1.f / 1.1f);
}
int launch_swish(const float* x, float b, long long n, float* a, float* da, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    swish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, b, n, a, da);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// T[t * n + i] = S[t * n + i] * m[i]  for t < nt  (in place allowed)
__global__ void mul_rows_kernel(const float* __restrict__ S, const float* __restrict__ m, long long n, int nt,
                                float* __restrict__ T) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float w = m[i];
    for (int t = 0; t < nt; ++t) T[(long long)t * n + i] = S[(long long)t * n + i] * w;
}
int launch_mul_rows(const float* S, const float* m, long long n, int nt, float* T, cudaStream_t st) {
    if (n == 0 || nt == 0) return NFB_OK;
    mul_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(S, m, n, nt, T);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// jt: [2, B, 2] -- jt[t, r, :] = J(x_r) e_t (column t of the Jacobian of g at sample r).  out[r] = log |det(I + J)|.
__global__ void logdet2_kernel(const float* __restrict__ jt, long long B, float* __restrict__ out) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    const float2 c0 = reinterpret_cast<const float2*>(jt)[r];        // (J00, J10)
    const float2 c1 = reinterpret_cast<const float2*>(jt)[B + r];    // (J01, J11)
    out[r] = logf(fabsf((c0.x + 1.f) * (c1.y + 1.f) - c1.x * c0.y));
}
int launch_logdet2(const float* jt, long long B, float* out, cudaStream_t st) {
    if (B == 0) return NFB_OK;
    logdet2_kernel<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(jt, B, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out = h + t * sigmoid(c): the GLU gate of a context-conditioned residual block (nets/resnet.py:48-50,
// nets/made.py:212-214: F.glu(cat(temps, context_layer(context))) + inputs)
__global__ void glu_residual_kernel(const float* __restrict__ h, const float* __restrict__ t, const float* __restrict__ c,
                                    long long n, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = fmaf(t[i], 1.f / (1.f + __expf(-c[i])), h[i]);
}
int launch_glu_residual(const float* h, const float* t, const float* c, long long n, float* out, cudaStream_t st) {
    if (n == 0) return NFB_OK;
    glu_residual_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(h, t, c, n, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Adjoint of the GLU gate out = h + t sigmoid(c): gh = g (optional copy), gt = g sigmoid(c), gc = g t sigmoid'(c).
// gt / gc may alias g.
__global__ void glu_residual_bwd_kernel(const float* __restrict__ g, const float* __restrict__ t,
                                        const float* __restrict__ c, long long n, float* gh, float* gt, float* gc) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float gi = g[i], sg = 1.f / (1.f + __expf(-c[i]));
    if (gh) gh[i] = gi;
    if (gc) gc[i] = gi * t[i] * sg * (1.f - sg);
    if (gt) gt[i] = gi * sg;
}
int launch_glu_residual_bwd(const float* g, const float* t, const float* c, long long n, float* gh, float* gt, float* gc,
                            cudaStream_t st) {
    if (n == 0) return NFB_OK;
    glu_residual_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, t, c, n, gh, gt, gc);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[r] = (accumulate ? out[r] : 0) + c * sum_j a[r, j] * b[r, j]   (one warp per row)
__global__ void __launch_bounds__(256) rowdot_kernel(const float* __restrict__ a, const float* __restrict__ b, long long rows,
                                                     int d, float c, int accumulate, float* __restrict__ out) {
    const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float s = 0.f;
    for (int j = lane; j < d; j += 32) s = fmaf(a[row * d + j], b[row * d + j], s);
    s = warp_sum(s);
    if (lane == 0) out[row] = (accumulate ? out[row] : 0.f) + c * s;
}
int launch_rowdot(const float* a, const float* b, long long rows, int d, float c, int accumulate, float* out,
                  cudaStream_t st) {
    if (rows == 0) return NFB_OK;
    rowdot_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(a, b, rows, d, c, accumulate, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// ---- training pass: the Lipschitz MLP pushed forward together with nt tangents (the "dual" network) ----
// Stacked layout of every [(1 + nt) B x w] tensor: rows [0, B) are the primal, rows [(t + 1) B, (t + 2) B) tangent t.
// H holds a layer's pre-activation WITHOUT its bias (the stacked forward GEMM has no epilogue, because the bias belongs
// to the primal rows only); the kernels add bias[j] to the primal rows while they read them.
//
// With s = sigmoid(b h), s1 = s (1 - s), u = b h:
//   sigma    = h s / 1.1                       d sigma / d b  = h^2 s1 / 1.1
//   sigma'   = (s + u s1) / 1.1                d sigma' / d b = h s1 (2 + u (1 - 2 s)) / 1.1
//   sigma''  = b s1 (2 + u (1 - 2 s)) / 1.1
struct SwishTerms { float d1, d2, db0, db1; float a; };
__device__ __forceinline__ SwishTerms swish_terms(float h, float b) {
    const float s = 1.f / (1.f + __expf(-b * h));
    const float s1 = s * (1.f - s);
    const float u = b * h;
    const float q = s1 * (2.f + u * (1.f - 2.f * s)) * (1.f / 1.1f);
    SwishTerms r;
    r.a = h * s * (1.f / 1.1f);
    r.d1 = (s + u * s1) * (1.f / 1.1f);
    r.d2 = b * q;
    r.db0 = h * h * s1 * (1.f / 1.1f);
    r.db1 = h * q;
    return r;
}

// A = [sigma(h); sigma'(h) t_1; ...; sigma'(h) t_nt]  from H = [h - bias; t_1; ...]   (one thread per primal element)
__global__ void swish_dual_kernel(const float* __restrict__ H, const float* __restrict__ bias, float b, long long B, int w,
                                  int nt, float* __restrict__ A) {
    const long long n = B * w;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float h = H[i] + (bias ? bias[i % w] : 0.f);
    const float s = 1.f / (1.f + __expf(-b * h));
    A[i] = h * s * (1.f / 1.1f);
    const float d1 = (s + b * h * s * (1.f - s)) * (1.f / 1.1f);
    for (int t = 1; t <= nt; ++t) A[t * n + i] = d1 * H[t * n + i];
}
int launch_swish_dual(const float* H, const float* bias, float b, long long B, int w, int nt, float* A, cudaStream_t st) {
    const long long n = B * w;
    if (n == 0) return NFB_OK;
    swish_dual_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(H, bias, b, B, w, nt, A);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Adjoint of swish_dual.  Abar = [abar; tabar_1; ...] (cotangents of A), H as above:
//   hbar  = sigma'(h) abar + sigma''(h) sum_t t_t tabar_t          -> out_primal [B x w]
//   tbar_t = sigma'(h) tabar_t                                      -> out_tangent [nt B x w] (NULL: not written)
//   d/db  = sum over elements of abar dsigma/db + sum_t tabar_t t_t dsigma'/db   -> partials[blockIdx.x] (fp64)
// out_primal / out_tangent may alias Abar (every thread reads its own elements before writing them).
// A grid of at most kSwishPartials CTAs, grid-stride: the per-CTA partials are in a fixed order for a given shape.
constexpr int kSwishPartials = 1024;
__global__ void __launch_bounds__(256) swish_dual_adjoint_kernel(const float* __restrict__ H, const float* __restrict__ bias,
                                                                 float b, long long B, int w, int nt, const float* Abar,
                                                                 float* out_primal, float* out_tangent,
                                                                 double* __restrict__ partials) {
    const long long n = B * w;
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float h = H[i] + (bias ? bias[i % w] : 0.f);
        const SwishTerms k = swish_terms(h, b);
        const float ab = Abar[i];
        float mix = 0.f, dbt = 0.f;
        for (int t = 1; t <= nt; ++t) {
            const float tt = H[t * n + i], tb = Abar[t * n + i];
            mix = fmaf(tt, tb, mix);
            if (out_tangent) out_tangent[(t - 1) * n + i] = k.d1 * tb;
        }
        dbt = fmaf(ab, k.db0, mix * k.db1);
        if (out_primal) out_primal[i] = fmaf(k.d1, ab, k.d2 * mix);
        acc += (double)dbt;
    }
    __shared__ double red[256];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) partials[blockIdx.x] = red[0];
}
// second stage: *out = sum of `count` partials, in a fixed order (deterministic)
__global__ void __launch_bounds__(256) sum_partials_kernel(const double* __restrict__ partials, int count,
                                                           float* __restrict__ out) {
    __shared__ double red[256];
    double acc = 0.0;
    for (int i = threadIdx.x; i < count; i += 256) acc += partials[i];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) *out = (float)red[0];
}
int launch_swish_dual_adjoint(const float* H, const float* bias, float b, long long B, int w, int nt, const float* Abar,
                              float* out_primal, float* out_tangent, double* partials, float* g_b, cudaStream_t st) {
    const long long n = B * w;
    int grid = (int)std::min<long long>((n + 255) / 256, kSwishPartials);
    if (grid < 1) grid = 1;   // no rows: one CTA writes a zero partial, so g_b is still defined
    swish_dual_adjoint_kernel<<<grid, 256, 0, st>>>(H, bias, b, B, w, nt, Abar, out_primal, out_tangent, partials);
    NFB_LAUNCH_CHECK();
    if (g_b) {
        sum_partials_kernel<<<1, 256, 0, st>>>(partials, grid, g_b);
        NFB_LAUNCH_CHECK();
    }
    return NFB_OK;
}

// Tangent seeds of the exact 2 x 2 log-det (the adjoint of logdet2): with M = I + J_r and g = g_ld[r],
// d log|det M| / dM = M^-T, so the cotangent of column t of J (jt[t, r, :]) is g times column t of M^-T.
__global__ void logdet2_backward_kernel(const float* __restrict__ jt, const float* __restrict__ g_ld, long long B,
                                        float* __restrict__ seeds) {
    const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B) return;
    const float2 c0 = reinterpret_cast<const float2*>(jt)[r];        // (J00, J10)
    const float2 c1 = reinterpret_cast<const float2*>(jt)[B + r];    // (J01, J11)
    const float m00 = c0.x + 1.f, m10 = c0.y, m01 = c1.x, m11 = c1.y + 1.f;
    const float g = g_ld[r] / (m00 * m11 - m01 * m10);
    reinterpret_cast<float2*>(seeds)[r] = make_float2(g * m11, -g * m01);
    reinterpret_cast<float2*>(seeds)[B + r] = make_float2(-g * m10, g * m00);
}
int launch_logdet2_backward(const float* jt, const float* g_ld, long long B, float* seeds, cudaStream_t st) {
    if (B == 0) return NFB_OK;
    logdet2_backward_kernel<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(jt, g_ld, B, seeds);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
