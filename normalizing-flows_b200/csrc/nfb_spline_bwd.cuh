// nfb_spline_bwd.cuh -- analytic backward of the monotone rational-quadratic spline element
// (utils/splines.py:100-219, forward branch :200-219; tails :28-57).  Host/device and templated on the scalar type so
// that tests/native can check it in double precision against finite differences and against gradients minted from the
// reference's autograd (tests/test_spline_host.py, tests/test_conditional_training.py).  Kernels: nfb_backward.cu.
//
// Same formulation as rqs_core (nfb_spline.cuh): logits in the log2 domain, knots on the unit interval
// (knot j = a * prefix_{j-1} + 1e-3 j, a = (1 - 1e-3 K) / sum), bin by search on the width knots, softplus on the
// two selected derivative logits only.  Given the upstream gradients (gy, glad) of one element it returns the
// gradients w.r.t. x, the K + K log2-domain logits and the K - 1 derivative logits.  Only the two knots of the
// selected bin and the two selected derivatives receive gradient directly; the softmax couples all K logits.
#pragma once
#include "nfb_common.cuh"
#include "nfb_spline.cuh"

namespace nfb {

template <typename T> __host__ __device__ __forceinline__ T t_exp2(T x);
template <> __host__ __device__ __forceinline__ float t_exp2<float>(float x) { return fast_ex2(x); }
template <> __host__ __device__ __forceinline__ double t_exp2<double>(double x) { return exp2(x); }
template <typename T> __host__ __device__ __forceinline__ T t_log(T x);
template <> __host__ __device__ __forceinline__ float t_log<float>(float x) { return kLn2 * fast_lg2(x); }
template <> __host__ __device__ __forceinline__ double t_log<double>(double x) { return log(x); }
template <typename T> __host__ __device__ __forceinline__ T t_exp(T x);
template <> __host__ __device__ __forceinline__ float t_exp<float>(float x) { return fast_ex2(x * kLog2e); }
template <> __host__ __device__ __forceinline__ double t_exp<double>(double x) { return exp(x); }

template <typename T> __host__ __device__ __forceinline__ T t_rcp(T x);
template <> __host__ __device__ __forceinline__ float t_rcp<float>(float x) { return rcp_nr(x); }
template <> __host__ __device__ __forceinline__ double t_rcp<double>(double x) { return 1.0 / x; }
template <typename T> __host__ __device__ __forceinline__ T t_sqrt(T x);
template <> __host__ __device__ __forceinline__ float t_sqrt<float>(float x) { return sqrtf(x); }
template <> __host__ __device__ __forceinline__ double t_sqrt<double>(double x) { return sqrt(x); }

// Forward (y, lad) and backward in one pass (the backward needs every forward intermediate), for K <= KMAX bins
// given at run time (KMAX == K on the templated fast path, where every loop unrolls).  udk[0..K] are the raw
// derivative logits of all K + 1 knots, boundary knots included; gudk[0..K] receives their gradients.  Outside
// [-tail, tail] (and for NaN) the element is the identity, or, with `zero_outside` (the tails-list branch of
// utils/splines.py:48-57, which never copies outside inputs), the constant 0: gx = 0 there.
//
// INV: the inverse spline (utils/splines.py:172-198), x = g(z), ld = -log f'(x), given z (the `x` argument) and the
// cotangents (gy, glad) of (x, ld).  The bin is searched on the HEIGHT knots at z with the real-domain running sums of
// rqs_eval_dyn's inverse branch, and theta is solved in that bin (never re-searched on x, so a z on an interior knot
// keeps its bin).  With c = g_x - g_ld d_x log f'(x):  g_z = c / f'(x)  and  g_theta = -(c / f') d_theta f
// - g_ld d_theta log f', which is the forward adjoint at x with the cotangents (-c / f', -g_ld): the backward of the
// local rational function below is shared, its x gradient is replaced by g_z.  `y` / `lad` return x and ld.
template <int KMAX, bool INV, typename T>
__host__ __device__ inline void rqs_adjoint_impl(int K, T x, const T* lw, const T* lh, const T* udk, T tail, T gy,
                                                 T glad, bool zero_outside, T& y, T& lad, T& gx, T* glw, T* glh,
                                                 T* gudk) {
    const T m = (T)1e-3, md = (T)1e-3, cfac = (T)1 - m * (T)K, ln2 = (T)0.6931471805599453;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) if (i < K) { glw[i] = (T)0; glh[i] = (T)0; gudk[i] = (T)0; }
    gudk[K] = (T)0;
    if (!(x >= -tail && x <= tail)) {  // outside the interval, and NaN  (:28,:40-41)
        y = zero_outside ? (T)0 : x; lad = (T)0; gx = zero_outside ? (T)0 : gy;
        return;
    }
    // ---- forward ----
    T mw = lw[0], mh = lh[0];
#pragma unroll
    for (int i = 1; i < KMAX; ++i) if (i < K) { mw = lw[i] > mw ? lw[i] : mw; mh = lh[i] > mh ? lh[i] : mh; }
    T ew[KMAX], eh[KMAX], cw[KMAX], ch[KMAX];
    T sw = (T)0, sh = (T)0;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) {
        if (i < K) {
            ew[i] = t_exp2<T>(lw[i] - mw); eh[i] = t_exp2<T>(lh[i] - mh);
            sw += ew[i]; sh += eh[i];
            cw[i] = sw; ch[i] = sh;
        }
    }
    const T aw = cfac / sw, ah = cfac / sh;
    T kw[KMAX + 1], kh[KMAX + 1];
    kw[0] = (T)0; kh[0] = (T)0; kw[K] = (T)1; kh[K] = (T)1;
#pragma unroll
    for (int i = 0; i < KMAX - 1; ++i)
        if (i < K - 1) { kw[i + 1] = aw * cw[i] + m * (T)(i + 1); kh[i + 1] = ah * ch[i] + m * (T)(i + 1); }
    const T two_b = (T)2 * tail;
    const T xu = x / two_b + (T)0.5;
    int b = 0;
    if (INV) {   // rqs_eval_dyn<true>: bottom of bin i = 2B cumh_i - B, compared with z in the real domain
        const T khs = cfac * t_rcp<T>(sh);
        T cum = (T)0, bottom = -tail;
#pragma unroll
        for (int i = 0; i < KMAX; ++i)
            if (i < K) {
                cum += m + khs * eh[i];
                const T top = (i == K - 1) ? tail : (two_b * cum - tail);
                if (x >= bottom) b = i;
                bottom = top;
            }
    } else {
#pragma unroll
        for (int i = 1; i < KMAX; ++i) if (i < K) b += (xu >= kw[i]) ? 1 : 0;  // knots increase: count = bin index
    }
    const T l_w = kw[b], r_w = kw[b + 1], l_h = kh[b], r_h = kh[b + 1];
    const T u0 = udk[b], u1 = udk[b + 1];
    auto softplus = [](T u) { return u > (T)20 ? u : (u < (T)-30 ? t_exp<T>(u) : t_log<T>((T)1 + t_exp<T>(u))); };
    auto sigmoid = [](T u) { return (T)1 / ((T)1 + t_exp<T>(-u)); };
    const T d0 = md + softplus(u0), d1 = md + softplus(u1);
    const T w = r_w - l_w, h = r_h - l_h;
    const T delta = h / w;
    const T s = d0 + d1 - (T)2 * delta;
    T theta;
    if (INV) {   // root of the quadratic (:184-193)
        const T t = xu - l_h;
        const T qa = t * s + h * (delta - d0), qb = h * d0 - t * s, qc = -delta * t;
        const T disc = qb * qb - (T)4 * qa * qc;
        theta = ((T)2 * qc) / (-qb - t_sqrt<T>(disc > (T)0 ? disc : (T)0));
    } else {
        theta = (xu - l_w) / w;
    }
    const T omt = (T)1 - theta;
    const T A = theta * theta, Bq = theta * omt, C = omt * omt;
    const T den = delta + s * Bq;
    const T P = delta * A + d0 * Bq;
    const T num = h * P;
    const T Q = d1 * A + (T)2 * delta * Bq + d0 * C;
    const T dnum = delta * delta * Q;
    T gyf = gy, gladf = glad, gz = (T)0;
    if (INV) {
        y = (l_w + theta * w) * two_b - tail;
        lad = (T)2 * t_log<T>(den) - t_log<T>(dnum);
        // d_theta log f' at x, then c = g_x - g_ld d_x log f';  f' = dnum / den^2
        const T dl = ((T)2 * (d1 * theta + delta * ((T)1 - (T)2 * theta) - d0 * omt)) / Q -
                     (T)2 * s * ((T)1 - (T)2 * theta) / den;
        const T c = gy - glad * dl / (w * two_b);
        gz = c * den * den / dnum;
        gyf = -gz; gladf = -glad;
    } else {
        const T outu = l_h + num / den;
        y = outu * two_b - tail;
        lad = t_log<T>(dnum) - (T)2 * t_log<T>(den);
    }
    // ---- backward of the local rational function ----
    const T g_out = gyf * two_b;
    const T g_num = g_out / den;
    const T g_den = -g_out * num / (den * den) - (T)2 * gladf / den;
    const T g_dnum = gladf / dnum;
    T g_delta = g_dnum * ((T)2 * delta * Q + delta * delta * (T)2 * Bq);
    const T g_Q = g_dnum * delta * delta;
    T g_d1 = g_Q * A, g_d0 = g_Q * C;
    T g_A = g_Q * d1, g_B = g_Q * (T)2 * delta;
    const T g_C = g_Q * d0;
    T g_h = g_num * P;
    const T g_P = g_num * h;
    g_delta += g_P * A; g_A += g_P * delta; g_d0 += g_P * Bq; g_B += g_P * d0;
    g_delta += g_den;
    const T g_s = g_den * Bq;
    g_B += g_den * s;
    g_d0 += g_s; g_d1 += g_s; g_delta -= (T)2 * g_s;
    const T g_theta = (T)2 * theta * g_A + ((T)1 - (T)2 * theta) * g_B - (T)2 * omt * g_C;
    const T g_xu = g_theta / w;
    T g_lw = -g_theta / w;
    T g_w = -g_theta * theta / w;
    g_h += g_delta / w;
    g_w -= g_delta * delta / w;
    const T g_rw = g_w;
    g_lw -= g_w;
    const T g_rh = g_h;
    const T g_lh = g_out - g_h;
    gx = INV ? gz : g_xu / two_b;
    gudk[b] += g_d0 * (u0 > (T)20 ? (T)1 : sigmoid(u0));
    gudk[b + 1] += g_d1 * (u1 > (T)20 ? (T)1 : sigmoid(u1));
    // ---- knots -> softmax logits.  knot j = cfac * prefix_{j-1} / sum + m j  (1 <= j <= K-1) ----
    //   d knot_j / d e_t = cfac * ([t <= j-1] - prefix_{j-1} / sum) / sum ;  d e_t / d logit_t = ln2 * e_t
    auto knots_bwd = [&](const T* e, const T* c, T sum, T g_left, T g_right, T* g) {
        const T gk[2] = {b >= 1 ? g_left : (T)0, b + 1 <= K - 1 ? g_right : (T)0};
        const int jj[2] = {b, b + 1};
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            if (gk[q] == (T)0) continue;
            const int j = jj[q];
            const T frac = c[j - 1] / sum, base = gk[q] * cfac / sum;
#pragma unroll
            for (int t = 0; t < KMAX; ++t)
                if (t < K) g[t] += base * ((t <= j - 1 ? (T)1 : (T)0) - frac) * ln2 * e[t];
        }
    };
    knots_bwd(ew, cw, sw, g_lw, g_rw, glw);
    knots_bwd(eh, ch, sh, g_lh, g_rh, glh);
}

template <int KMAX, typename T>
__host__ __device__ inline void rqs_adjoint(int K, T x, const T* lw, const T* lh, const T* udk, T tail, T gy, T glad,
                                            bool zero_outside, T& y, T& lad, T& gx, T* glw, T* glh, T* gudk) {
    rqs_adjoint_impl<KMAX, false, T>(K, x, lw, lh, udk, tail, gy, glad, zero_outside, y, lad, gx, glw, glh, gudk);
}
// The inverse element: z in, (x, ld) = (y, lad) out, gx = g_z (see rqs_adjoint_impl).
template <int KMAX, typename T>
__host__ __device__ inline void rqs_inverse_adjoint(int K, T z, const T* lw, const T* lh, const T* udk, T tail, T gx_out,
                                                    T gld, bool zero_outside, T& x, T& ld, T& gz, T* glw, T* glh,
                                                    T* gudk) {
    rqs_adjoint_impl<KMAX, true, T>(K, z, lw, lh, udk, tail, gx_out, gld, zero_outside, x, ld, gz, glw, glh, gudk);
}

// Linear tails, K - 1 interior derivative logits (the fused blocks' layout): boundary knots pinned to the constant.
template <int K, typename T>
__host__ __device__ inline void rqs_fwd_bwd(T x, const T (&lw)[K], const T (&lh)[K], const T (&ud)[K - 1], T tail,
                                            T gy, T glad, T& y, T& lad, T& gx, T (&glw)[K], T (&glh)[K],
                                            T (&gud)[K - 1]) {
    T udk[K + 1], gudk[K + 1];
    udk[0] = (T)NFB_BOUNDARY_UD; udk[K] = (T)NFB_BOUNDARY_UD;
#pragma unroll
    for (int i = 0; i < K - 1; ++i) udk[i + 1] = ud[i];
    rqs_adjoint<K, T>(K, x, lw, lh, udk, tail, gy, glad, false, y, lad, gx, glw, glh, gudk);
#pragma unroll
    for (int i = 0; i < K - 1; ++i) gud[i] = gudk[i + 1];
}

// The same layout, inverse element: z in, (x, ld) out, gz = g_z given the cotangents (gx_out, gld) of (x, ld).
template <int K, typename T>
__host__ __device__ inline void rqs_inv_fwd_bwd(T z, const T (&lw)[K], const T (&lh)[K], const T (&ud)[K - 1], T tail,
                                                T gx_out, T gld, T& x, T& ld, T& gz, T (&glw)[K], T (&glh)[K],
                                                T (&gud)[K - 1]) {
    T udk[K + 1], gudk[K + 1];
    udk[0] = (T)NFB_BOUNDARY_UD; udk[K] = (T)NFB_BOUNDARY_UD;
#pragma unroll
    for (int i = 0; i < K - 1; ++i) udk[i + 1] = ud[i];
    rqs_inverse_adjoint<K, T>(K, z, lw, lh, udk, tail, gx_out, gld, false, x, ld, gz, glw, glh, gudk);
#pragma unroll
    for (int i = 0; i < K - 1; ++i) gud[i] = gudk[i + 1];
}

// One element of the stand-alone splines (nfb_rqs_spline / nfb_rqs_spline_tails), on its raw parameter record
// p[2K + nd] = [widths(K) | heights(K) | derivatives(nd)], with the knot layout of rqs_eval_dyn (nfb_spline.cuh):
//   nd = K - 1: linear tails, boundary knots pinned to the constant of utils/splines.py:35-38;
//   nd = K:     tails="circular" (:42-47), knot K repeats knot 0, identity outside;
//   nd = K + 1: tails list (:48-57), every knot has a parameter; a linear feature (circular = false) pins both ends
//               (their parameters get no gradient), a circular one copies knot 0 into knot K; outside inputs give 0.
// A circular feature's derivative 0 is used twice, so both gradients land on parameter 2K; parameter 3K gets 0.
// wh_scale multiplies the width / height logits.  gp[2K + nd] is overwritten.
template <int KMAX, bool INV, typename T>
__host__ __device__ inline void rqs_adjoint_params_impl(int K, int nd, bool circular, T x, const T* p, T wh_scale, T tail,
                                                        T gy, T glad, T& y, T& lad, T& gx, T* gp) {
    const T s2 = wh_scale * (T)1.4426950408889634;
    T lw[KMAX], lh[KMAX], udk[KMAX + 1], gudk[KMAX + 1];
#pragma unroll
    for (int i = 0; i < KMAX; ++i) if (i < K) { lw[i] = p[i] * s2; lh[i] = p[K + i] * s2; }
    const int dshift = nd == K - 1 ? 1 : 0;
    const bool learned_ends = nd != K - 1 && circular;
    udk[0] = learned_ends ? p[2 * K] : (T)NFB_BOUNDARY_UD;
    udk[K] = udk[0];
#pragma unroll
    for (int i = 1; i < KMAX; ++i) if (i < K) udk[i] = p[2 * K + i - dshift];
    rqs_adjoint_impl<KMAX, INV, T>(K, x, lw, lh, udk, tail, gy, glad, nd == K + 1, y, lad, gx, gp, gp + K, gudk);
#pragma unroll
    for (int i = 0; i < KMAX; ++i) if (i < K) { gp[i] *= s2; gp[K + i] *= s2; }
    for (int i = 0; i < nd; ++i) gp[2 * K + i] = (T)0;
#pragma unroll
    for (int i = 1; i < KMAX; ++i) if (i < K) gp[2 * K + i - dshift] = gudk[i];
    if (learned_ends) gp[2 * K] = gudk[0] + gudk[K];
}

template <int KMAX, typename T>
__host__ __device__ inline void rqs_adjoint_params(int K, int nd, bool circular, T x, const T* p, T wh_scale, T tail,
                                                   T gy, T glad, T& y, T& lad, T& gx, T* gp) {
    rqs_adjoint_params_impl<KMAX, false, T>(K, nd, circular, x, p, wh_scale, tail, gy, glad, y, lad, gx, gp);
}
// The inverse spline x = g(z; p), ld = -log f'(x; p) on the same record layout (nfb_rqs_spline(_tails) with
// inverse = 1): given z and the cotangents (g_x, g_ld) it returns x, ld, g_z and g_p (same tails modes and circular
// parameter sharing as rqs_adjoint_params; tails-list inputs outside the interval give x = 0 and zero gradients).
template <int KMAX, typename T>
__host__ __device__ inline void rqs_inverse_adjoint_params(int K, int nd, bool circular, T z, const T* p, T wh_scale,
                                                           T tail, T g_x, T g_ld, T& x, T& ld, T& gz, T* gp) {
    rqs_adjoint_params_impl<KMAX, true, T>(K, nd, circular, z, p, wh_scale, tail, g_x, g_ld, x, ld, gz, gp);
}

}  // namespace nfb
