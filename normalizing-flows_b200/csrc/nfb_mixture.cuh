// nfb_mixture.cuh -- element math of the Gaussian-mixture base (reference distributions/base.py:573-659
// GaussianMixture), shared by the kernels of nfb_mixture.cu and, compiled for the host, by
// tests/native/mixture_adjoint_host_check.cu.  Templated on the scalar type.
//
// One row z [D], K modes with loc mu [K, D], log_scale ls [K, D] and weight_scores ws [K]:
//   e_k    = log_softmax(ws)_k - D/2 log 2pi - sum_d (ls_kd + t_kd^2 / 2),   t_kd = (z_d - mu_kd) exp(-ls_kd)
//   log p  = logsumexp_k e_k          (streaming, max-subtracted: no bound on K, no underflow for e_k near -5e5)
// log_softmax is ws_k - logsumexp(ws), not log(softmax): a weight that underflows in the reference's softmax gives a
// finite, negligible e_k here (and finite gradients) instead of -inf.
// Row cotangent g, responsibilities resp_k = exp(e_k - log p), a_k = g resp_k:
//   g_z_d   = -sum_k a_k t_kd exp(-ls_kd)
//   g_mu_kd =  a_k t_kd exp(-ls_kd)          (summed over rows)
//   g_ls_kd =  a_k (t_kd^2 - 1)              (summed over rows)
//   g_ws_k  =  a_k - softmax(ws)_k g         (summed over rows)
// The differences z - mu are formed directly; no moment expansion (sum a z^2 ...), which would cancel when |mu| >> sigma.
#pragma once
#include <cmath>

namespace nfb {

__host__ __device__ __forceinline__ float mx_exp(float v) { return expf(v); }
__host__ __device__ __forceinline__ double mx_exp(double v) { return exp(v); }
__host__ __device__ __forceinline__ float mx_log(float v) { return logf(v); }
__host__ __device__ __forceinline__ double mx_log(double v) { return log(v); }

constexpr double kHalfLog2Pi = 0.91893853320467274178;

// streaming log-sum-exp: state (m, s) stands for m + log s; starts at (-inf, 0).  A NaN term makes the result NaN; a
// -inf term adds nothing (all terms -inf: the result is -inf).
template <typename T>
__host__ __device__ __forceinline__ void mix_lse_push(T& m, T& s, T x) {
    if (x > m) {
        s = s * mx_exp(m - x) + (T)1;
        m = x;
    } else if (!(x == -(T)INFINITY)) {
        s += mx_exp(x - m);
    }
}

template <typename T>
__host__ __device__ __forceinline__ T mix_lse_value(T m, T s) { return m + mx_log(s); }

// logsumexp(ws) over the K weight scores, in index order
template <typename T>
__host__ __device__ inline T mix_weight_lse(const T* ws, int K) {
    T m = -(T)INFINITY, s = (T)0;
    for (int k = 0; k < K; ++k) mix_lse_push(m, s, ws[k]);
    return mix_lse_value(m, s);
}

// one feature's share of -e_k (without the weight and the 2 pi constant): ls + t^2 / 2, inv = exp(-ls)
template <typename T>
__host__ __device__ __forceinline__ T mix_quad_term(T z, T mu, T inv, T ls) {
    const T t = (z - mu) * inv;
    return ls + (T)0.5 * t * t;
}

// e_k from its weight score, the weight normaliser and the feature sum of mix_quad_term
template <typename T>
__host__ __device__ __forceinline__ T mix_mode_exponent(T ws_k, T ws_lse, int D, T quad) {
    return (ws_k - ws_lse) - (T)D * (T)kHalfLog2Pi - quad;
}

// log p of one row (the kernels' arithmetic, one thread per row)
template <typename T>
__host__ __device__ inline T mixture_row_log_prob(const T* z, const T* mu, const T* ls, const T* ws, int K, int D) {
    const T wl = mix_weight_lse(ws, K);
    T m = -(T)INFINITY, s = (T)0;
    for (int k = 0; k < K; ++k) {
        T q = (T)0;
        for (int d = 0; d < D; ++d) q += mix_quad_term(z[d], mu[k * D + d], mx_exp(-ls[k * D + d]), ls[k * D + d]);
        mix_lse_push(m, s, mix_mode_exponent(ws[k], wl, D, q));
    }
    return mix_lse_value(m, s);
}

// the adjoint of one row with cotangent g: g_z [D] overwritten, g_mu / g_ls [K, D] and g_ws [K] accumulated
template <typename T>
__host__ __device__ inline void mixture_row_adjoint(const T* z, const T* mu, const T* ls, const T* ws, int K, int D,
                                                    T g, T* g_z, T* g_mu, T* g_ls, T* g_ws) {
    const T wl = mix_weight_lse(ws, K);
    const T lp = mixture_row_log_prob(z, mu, ls, ws, K, D);
    for (int d = 0; d < D; ++d) g_z[d] = (T)0;
    for (int k = 0; k < K; ++k) {
        T q = (T)0;
        for (int d = 0; d < D; ++d) q += mix_quad_term(z[d], mu[k * D + d], mx_exp(-ls[k * D + d]), ls[k * D + d]);
        const T a = g * mx_exp(mix_mode_exponent(ws[k], wl, D, q) - lp);
        for (int d = 0; d < D; ++d) {
            const T inv = mx_exp(-ls[k * D + d]);
            const T t = (z[d] - mu[k * D + d]) * inv;
            g_z[d] -= a * t * inv;
            g_mu[k * D + d] += a * t * inv;
            g_ls[k * D + d] += a * (t * t - (T)1);
        }
        g_ws[k] += a - mx_exp(ws[k] - wl) * g;
    }
}

// log p of one row of at most DMAX features and, when grad is not null, c * grad_z log p added to grad [D]:
// grad_d -= c resp_k t_kd exp(-ls_kd), the g_z of mixture_row_adjoint with cotangent c.  The feature loops unroll
// over DMAX, so a caller's z / grad arrays stay in registers (the HMC / MH kernels of nfb_stochastic.cu, one row per
// thread); the mode loop streams, so K is unbounded.  Two passes over the modes: the log-sum-exp, then the
// responsibilities.
template <int DMAX, typename T>
__host__ __device__ __forceinline__ T mixture_row_log_prob_grad(const T* z, int D, const T* mu, const T* ls,
                                                                const T* ws, int K, T c, T* grad) {
    const T wl = mix_weight_lse(ws, K);
    T m = -(T)INFINITY, s = (T)0;
    for (int k = 0; k < K; ++k) {
        T q = (T)0;
#pragma unroll
        for (int d = 0; d < DMAX; ++d)
            if (d < D) q += mix_quad_term(z[d], mu[k * D + d], mx_exp(-ls[k * D + d]), ls[k * D + d]);
        mix_lse_push(m, s, mix_mode_exponent(ws[k], wl, D, q));
    }
    const T lp = mix_lse_value(m, s);
    if (grad) {
        for (int k = 0; k < K; ++k) {
            T q = (T)0;
#pragma unroll
            for (int d = 0; d < DMAX; ++d)
                if (d < D) q += mix_quad_term(z[d], mu[k * D + d], mx_exp(-ls[k * D + d]), ls[k * D + d]);
            const T a = c * mx_exp(mix_mode_exponent(ws[k], wl, D, q) - lp);
#pragma unroll
            for (int d = 0; d < DMAX; ++d) {
                if (d < D) {
                    const T inv = mx_exp(-ls[k * D + d]);
                    const T t = (z[d] - mu[k * D + d]) * inv;
                    grad[d] -= a * t * inv;
                }
            }
        }
    }
    return lp;
}

}  // namespace nfb
