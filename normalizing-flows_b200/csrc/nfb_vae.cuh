// nfb_vae.cuh -- element math of the flow-VAE encoders and decoders (reference distributions/encoder.py
// ConstDiagGaussian / NNDiagGaussian, distributions/decoder.py NNDiagGaussianDecoder / NNBernoulliDecoder), shared by
// the kernels of nfb_vae.cu and, compiled for the host, by tests/native/vae_host_check.cu.  Templated on the scalar type.
//
// Diagonal Gaussian with mean m and a scale column p, read as (kind):
//   NFB_VAE_LOGVAR  p = log variance (NNDiagGaussian, NNDiagGaussianDecoder):  sd = exp(p / 2), log sd = p / 2
//   NFB_VAE_SCALE   p = standard deviation (ConstDiagGaussian):                sd = p,          log sd = log p
// (a negative scale gives NaN, as in the reference).
//   reparameterised draw   z = m + sd eps,   log q = -D/2 log 2pi - sum (log sd + eps^2 / 2)
//   density                log p(v) = -N/2 log 2pi - sum (log sd + u^2 / 2),  u = (v - m) / sd
// (N is the reference's normalising count: the latent size for NNDiagGaussianDecoder.log_prob, D otherwise).
// Adjoints per element, with cotangents gz of z and g of the row's log q / log p:
//   draw     g_m = gz,          g_sd = gz eps - g / sd
//   density  g_m = g u / sd,    g_sd = g (u^2 - 1) / sd,   g_v = -g u / sd
// and g_p = g_sd dsd/dp with dsd/dp = sd / 2 (log variance) or 1 (scale), applied after the sums over rows.
//
// Bernoulli decoder with score s (the net's output) and data x:
//   log p = sum x log_sig(s) + (1 - x) log_sig(-s),   log_sig(a) = -relu(-a) - log(1 + exp(-|a|))
//   g_s = g (x - sigmoid(s)), except at s == 0 exactly, where it is 0: the reference differentiates relu and |.|
//         with derivative 0 at 0 (torch), so both halves vanish there
//   g_x = g s   (log_sig(s) - log_sig(-s) = s)
// log1p replaces log(1 + .): the same value up to rounding, exact for the saturated tails (|s| >> 1).
#pragma once
#include <cmath>

#define NFB_VAE_LOGVAR 0
#define NFB_VAE_SCALE 1

namespace nfb {

__host__ __device__ __forceinline__ float vae_exp(float v) { return expf(v); }
__host__ __device__ __forceinline__ double vae_exp(double v) { return exp(v); }
__host__ __device__ __forceinline__ float vae_log(float v) { return logf(v); }
__host__ __device__ __forceinline__ double vae_log(double v) { return log(v); }
__host__ __device__ __forceinline__ float vae_log1p(float v) { return log1pf(v); }
__host__ __device__ __forceinline__ double vae_log1p(double v) { return log1p(v); }

constexpr double kVaeHalfLog2Pi = 0.91893853320467274178;

// sd and log sd from the scale column
template <typename T>
__host__ __device__ __forceinline__ void vae_std(T p, int kind, T& sd, T& log_sd) {
    if (kind == NFB_VAE_LOGVAR) {
        log_sd = (T)0.5 * p;
        sd = vae_exp(log_sd);
    } else {
        sd = p;
        log_sd = vae_log(p);
    }
}

// dsd/dp
template <typename T>
__host__ __device__ __forceinline__ T vae_dstd(T sd, int kind) { return kind == NFB_VAE_LOGVAR ? (T)0.5 * sd : (T)1; }

// the draw: z (returned) and the element's share of -log q (without the 2 pi constant)
template <typename T>
__host__ __device__ __forceinline__ T vae_draw(T m, T sd, T log_sd, T eps, T& nlq) {
    nlq = log_sd + (T)0.5 * eps * eps;
    return m + sd * eps;
}

template <typename T>
__host__ __device__ __forceinline__ void vae_draw_adjoint(T sd, T eps, T gz, T g, T& g_m, T& g_sd) {
    g_m = gz;
    g_sd = gz * eps - g / sd;
}

// the element's share of -log p(v) (without the 2 pi constant)
template <typename T>
__host__ __device__ __forceinline__ T vae_density_term(T v, T m, T sd, T log_sd) {
    const T u = (v - m) / sd;
    return log_sd + (T)0.5 * u * u;
}

template <typename T>
__host__ __device__ __forceinline__ void vae_density_adjoint(T v, T m, T sd, T g, T& g_v, T& g_m, T& g_sd) {
    const T u = (v - m) / sd;
    g_m = g * u / sd;
    g_v = -g_m;
    g_sd = g * (u * u - (T)1) / sd;
}

template <typename T>
__host__ __device__ __forceinline__ T vae_log_sig(T a) {
    return -(a < (T)0 ? -a : (T)0) - vae_log1p(vae_exp(-(a < (T)0 ? -a : a)));
}

template <typename T>
__host__ __device__ __forceinline__ T vae_sigmoid(T s) {
    if (s >= (T)0) return (T)1 / ((T)1 + vae_exp(-s));
    const T e = vae_exp(s);
    return e / ((T)1 + e);
}

template <typename T>
__host__ __device__ __forceinline__ T vae_bernoulli_term(T s, T x) {
    return x * vae_log_sig(s) + ((T)1 - x) * vae_log_sig(-s);
}

// d term / d s
template <typename T>
__host__ __device__ __forceinline__ T vae_bernoulli_dscore(T s, T x) {
    return s == (T)0 ? (T)0 : x - vae_sigmoid(s);
}

}  // namespace nfb
