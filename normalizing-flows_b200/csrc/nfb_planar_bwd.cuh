// nfb_planar_bwd.cuh -- per-layer constants and element adjoints of the planar and radial flows (Rezende & Mohamed
// 2015; reference flows/planar.py:51-81, flows/radial.py:37-46), shared by the kernels of nfb_planar.cu and, compiled
// for the host, by tests/native/planar_adjoint_host_check.cu.  Templated on the scalar type.
//
// Planar, sampling direction, one row:  lin = w.z + b,  x = z + u_hat h(lin),  ld = log|1 + psi h'(lin)|
//   with inner = w.u, m = log(1 + exp(inner)) - 1 - inner, q = |w|^2, k = m / q, u_hat = u + k w, psi = w.u_hat.
//   Row cotangents g (of x) and gam (of ld), A = 1 + psi h'(lin):
//     c = (g.u_hat) hd(lin) + gam psi h''(lin) / A     (cotangent of lin)      g_z = g + c w
//     e = gam h'(lin) / A                               (cotangent of psi)
//     rows' contributions: g_w += c z, g_b += c, g_u_hat += h(lin) g, g_psi += e
//   hd is the derivative autograd takes of h(lin) itself, h' the reference's closed form inside the log-det:
//     tanh:  h' = 1 / cosh^2 (as the reference writes it), hd = 1 - tanh^2, h'' = -2 tanh h'.  Where cosh overflows
//            h' = 0 and h'' = 0: the finite limit, where autograd of 1 / cosh^2 gives NaN.
//     leaky: h' = (lin < 0)(slope - 1) + 1 (1 at lin = 0, planar.py:60), hd = 1 if lin > 0 else slope (torch's
//            leaky_relu_backward: slope at 0), h'' = 0.
//   Parameter chain (planar_param_chain): g_u_hat = Sg + Se w, then through u_hat(u, w):
//     g_u = G + (G.w) m' / q w,   g_w = Sz + Se u_hat + k G + (G.w)(m' u / q - 2 m w / q^2),   g_b = Sc
//   with m' = exp(inner) / (1 + exp(inner)) - 1, the reference's expression differentiated as autograd does.
//
// Radial, sampling direction:  dz = z - z0, r = |dz|, s = alpha_hat + r, h = beta_hat / s, h_ = -beta_hat r / s^2,
//   x = z + h dz,  ld = (d - 1) log(1 + h) + log(1 + h + h_),  alpha_hat = |alpha|, beta_hat = log(1 + exp(beta)) - |alpha|
//     g_h = g.dz + gam ((d - 1) / (1 + h) + 1 / (1 + h + h_)),  g_h_ = gam / (1 + h + h_)
//     g_r = -g_h beta_hat / s^2 + g_h_ (2 beta_hat r / s^3 - beta_hat / s^2)
//     g_dz = h g + (g_r / r) dz  (0 / r taken as 0 at r = 0: vector_norm's backward),  g_z = g + g_dz,  g_z0 -= g_dz
//     row contributions to beta_hat: g_h / s - g_h_ r / s^2;  to alpha_hat: -g_h beta_hat / s^2 + 2 g_h_ beta_hat r / s^3
//   Parameter chain: g_beta = S_bh exp(beta) / (1 + exp(beta)),  g_alpha = sign(alpha)(S_ah - S_bh) (0 at alpha = 0).
#pragma once
#include <cmath>

namespace nfb {

__host__ __device__ __forceinline__ float pl_exp(float v) { return expf(v); }
__host__ __device__ __forceinline__ double pl_exp(double v) { return exp(v); }
__host__ __device__ __forceinline__ float pl_log(float v) { return logf(v); }
__host__ __device__ __forceinline__ double pl_log(double v) { return log(v); }
__host__ __device__ __forceinline__ float pl_tanh(float v) { return tanhf(v); }
__host__ __device__ __forceinline__ double pl_tanh(double v) { return tanh(v); }
__host__ __device__ __forceinline__ float pl_cosh(float v) { return coshf(v); }
__host__ __device__ __forceinline__ double pl_cosh(double v) { return cosh(v); }
__host__ __device__ __forceinline__ float pl_sqrt(float v) { return sqrtf(v); }
__host__ __device__ __forceinline__ double pl_sqrt(double v) { return sqrt(v); }

enum { kPlanarTanh = 0, kPlanarLeaky = 1, kRadial = 2 };

// inner = w.u, q = |w|^2 and m = log(1 + exp(inner)) - 1 - inner, summed in index order
template <typename T>
__host__ __device__ inline void planar_inner(const T* u, const T* w, int d, T& inner, T& q, T& m) {
    inner = (T)0; q = (T)0;
    for (int j = 0; j < d; ++j) { inner += w[j] * u[j]; q += w[j] * w[j]; }
    m = pl_log((T)1 + pl_exp(inner)) - (T)1 - inner;   // the reference's expression, not a stabilised softplus
}

// the per-layer constants of the sampling and density directions: k (u_hat = u + k w) and psi = w.u_hat
template <typename T>
__host__ __device__ inline void planar_consts(const T* u, const T* w, int d, T& k, T& psi) {
    T inner, q, m;
    planar_inner(u, w, d, inner, q, m);
    k = m / q;
    psi = (T)0;
    for (int j = 0; j < d; ++j) psi += w[j] * (u[j] + k * w[j]);
}

template <typename T>
__host__ __device__ inline void radial_consts(T alpha, T beta, T& alpha_hat, T& beta_hat) {
    alpha_hat = alpha < (T)0 ? -alpha : alpha;
    beta_hat = pl_log((T)1 + pl_exp(beta)) - alpha_hat;
}

// h(lin), h'(lin) of the log-det, and (backward only) hd = d h / d lin as autograd takes it and h''(lin)
template <typename T>
__host__ __device__ inline void planar_act(int act, T slope, T lin, T& h, T& hp, T& hd, T& hpp) {
    if (act == kPlanarTanh) {
        h = pl_tanh(lin);
        const T c = pl_cosh(lin);
        hp = (T)1 / (c * c);
        hd = (T)1 - h * h;
        hpp = (T)-2 * h * hp;
    } else {
        h = lin > (T)0 ? lin : lin * slope;
        hp = lin < (T)0 ? (slope - (T)1) + (T)1 : (T)1;
        hd = lin > (T)0 ? (T)1 : slope;
        hpp = (T)0;
    }
}

// planar row adjoint: gu = g.u_hat; returns c (cotangent of lin), hv = h(lin), e (cotangent of psi)
template <typename T>
__host__ __device__ inline void planar_row_adjoint(int act, T slope, T lin, T psi, T gu, T gam, T& c, T& hv, T& e) {
    T hp, hd, hpp;
    planar_act(act, slope, lin, hv, hp, hd, hpp);
    const T A = (T)1 + psi * hp;
    c = gu * hd + (hpp != (T)0 ? gam * psi * hpp / A : (T)0);
    e = gam * hp / A;
}

// radial row adjoint: gdot = g.dz, dm1 = d - 1; returns h, the coefficient cr of dz in g_dz (g_dz = h g + cr dz) and
// the row's contributions to beta_hat and alpha_hat
template <typename T>
__host__ __device__ inline void radial_row_adjoint(T r, T alpha_hat, T beta_hat, T dm1, T gdot, T gam, T& h, T& cr,
                                                   T& gbh, T& gah) {
    const T s = alpha_hat + r;
    const T s2 = s * s;
    h = beta_hat / s;
    const T h_ = -beta_hat * r / s2;
    const T g_h = gdot + gam * (dm1 / ((T)1 + h) + (T)1 / ((T)1 + h + h_));
    const T g_h_ = gam / ((T)1 + h + h_);
    const T g_r = -g_h * beta_hat / s2 + g_h_ * ((T)2 * beta_hat * r / (s2 * s) - beta_hat / s2);
    cr = r > (T)0 ? g_r / r : (T)0;
    gbh = g_h / s - g_h_ * r / s2;
    gah = -g_h * beta_hat / s2 + (T)2 * g_h_ * beta_hat * r / (s2 * s);
}

// planar parameter chain.  sums: Sz[d], Sc, Sg[d], (unused), Se -- the rows' reduced contributions; writes g_u[d],
// g_w[d], g_b[1] (each may be null)
template <typename T>
__host__ __device__ inline void planar_param_chain(const T* u, const T* w, int d, const T* Sz, T Sc, const T* Sg, T Se,
                                                   T* gu, T* gw, T* gb) {
    T inner, q, m;
    planar_inner(u, w, d, inner, q, m);
    const T k = m / q;
    const T ei = pl_exp(inner);
    const T mp = ei / ((T)1 + ei) - (T)1;
    T Gw = (T)0;
    for (int j = 0; j < d; ++j) Gw += (Sg[j] + Se * w[j]) * w[j];
    for (int j = 0; j < d; ++j) {
        const T G = Sg[j] + Se * w[j];
        if (gu) gu[j] = G + Gw * mp / q * w[j];
        if (gw) gw[j] = Sz[j] + Se * (u[j] + k * w[j]) + k * G + Gw * (mp * u[j] / q - (T)2 * m * w[j] / (q * q));
    }
    if (gb) *gb = Sc;
}

// radial parameter chain: S_bh, S_ah the reduced contributions to beta_hat and alpha_hat
template <typename T>
__host__ __device__ inline void radial_param_chain(T alpha, T beta, T S_bh, T S_ah, T& g_beta, T& g_alpha) {
    const T eb = pl_exp(beta);
    g_beta = S_bh * (eb / ((T)1 + eb));
    const T sg = alpha > (T)0 ? (T)1 : (alpha < (T)0 ? (T)-1 : (T)0);
    g_alpha = sg * (S_ah - S_bh);
}

}  // namespace nfb
