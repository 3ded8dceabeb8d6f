// nfb_spline.cuh -- monotone rational-quadratic spline, one element per call (rqs_core_lanes: N independent ones).
//
// Mask-free restatement of normflows/utils/splines.py:16-219 (`unconstrained_rational_
// quadratic_spline` with tails="linear" -> `rational_quadratic_spline`):
//   * outside [-B,B] (or NaN): identity, logabsdet 0                       (:28,:40-41)
//   * widths/heights: softmax -> min size 1e-3 -> cumsum -> scale to [-B,B],
//     end knots pinned exactly, bin sizes re-derived as knot differences    (:126-152)
//   * bin = (#knots <= x) - 1 with +1e-6 on the last knot only, so x == +B is
//     inside the last bin and an interior-knot hit goes to the right bin    (:11-13,:154-157)
//   * derivatives 1e-3 + softplus(.), boundary derivative from the constant
//     log(exp(1-1e-3)-1)                                                    (:35-38,:138)
//   * forward: :200-219   inverse (quadratic root 2c/(-b-sqrt(b^2-4ac))): :172-198
// Differences that are deliberate (and covered by the stated fp32 tolerance):
//   softplus is evaluated only for the two selected knot derivatives instead of all K+1;
//   the scan keeps running knots instead of materialising [K+1] arrays and gathering.
#pragma once
#include "nfb_common.cuh"

namespace nfb {

// MUFU approximations on the device.  The __host__ bodies exist only so that tests/native can
// compile this header for the CPU and check the arithmetic against the golden vectors without a
// GPU; no product code calls them on the host.
__host__ __device__ __forceinline__ float fast_ex2(float x) {
#ifdef __CUDA_ARCH__
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return exp2f(x);
#endif
}
__host__ __device__ __forceinline__ float fast_lg2(float x) {
#ifdef __CUDA_ARCH__
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return log2f(x);
#endif
}
__host__ __device__ __forceinline__ float fast_rcp(float x) {
#ifdef __CUDA_ARCH__
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
#else
    return 1.0f / x;
#endif
}

// Reciprocal to ~0.5 ulp: MUFU.RCP (1 ulp) plus one Newton step (2 FMAs).  The spline's knot scale, bin width,
// theta and output all hang on reciprocals; on the ill-conditioned rows of a deep stack the 1-ulp approximations
// alone moved log_prob by 1e-4 relative (offline error-injection study, DESIGN.md "Numerics"), the refined ones do not.
__host__ __device__ __forceinline__ float rcp_nr(float x) {
#ifdef __CUDA_ARCH__
    const float r = fast_rcp(x);
    return fmaf(r, fmaf(-x, r, 1.f), r);
#else
    return 1.0f / x;
#endif
}

// F.softplus(beta=1, threshold=20).  log1p(e) by series for small e: 1+e would round away
// up to 6e-8 absolute, which matters when the derivative sits at its 1e-3 floor.
// Branch-free (selects only) so that two independent spline evaluations inlined back to back stay in
// one basic block and ptxas can interleave them.
__host__ __device__ __forceinline__ float softplus_f(float u) {
    const float e = fast_ex2(fminf(u, 20.f) * kLog2e);
    const float series = e * (1.f - e * (0.5f - e * (0.33333334f - 0.25f * e)));
    const float lg = kLn2 * fast_lg2(1.f + e);
    const float sp = e < 0.03f ? series : lg;
    return u > 20.f ? u : sp;
}

// Root in [0, 1] of a theta^2 + b theta + c = 0 for the inverse spline (:172-198).  The reference's form 2c / (-b - sqrt(disc))
// is free of cancellation for b >= 0 (and is kept there bit for bit); for b < 0 its denominator cancels.  That happens
// where the bin is nearly flat at one end and steep at the other (large derivative parameters).  There the fp32 root can
// land outside [0, 1], so den = delta + s theta (1 - theta) goes negative and the log-det becomes NaN.  The same root as
// (-b + sqrt(disc)) / 2a has no cancellation for b < 0 (a >= |b| > 0 whenever that root lies in [0, 1]).  The clamp
// keeps the last ulps inside the bin.
__host__ __device__ __forceinline__ float rqs_inverse_root(float a, float b, float c) {
    const float sq = sqrtf(fmaxf(b * b - 4.f * a * c, 0.f));
    const float theta = b >= 0.f ? (2.f * c) / (-b - sq) : (sq - b) / (2.f * a);
    return fminf(fmaxf(theta, 0.f), 1.f);
}

// The unnormalised boundary derivative, as the reference computes it in fp32 (:36).
#define NFB_BOUNDARY_UD 0.5397424f /* float32(log(exp(1 - 1e-3) - 1)) = 0.5397424172... */

// Core evaluator.  lw / lh are the width / height logits already multiplied by log2(e) (and by the
// layer's 1/sqrt(hidden) where it has one); D(i) returns the i-th of the K-1 raw interior derivative
// parameters.  Everything between the softmax and the rational function is done on the unit interval
// u = (x + B) / 2B: knot i+1 is  a * prefix_i + 1e-3 (i+1)  with a = (1 - 1e-3 K) / sum -- one FMA per
// knot on a running sum that the softmax needs anyway (theta, delta and the derivative terms are scale
// free; only the output is mapped back with one FMA).  The knot positions differ from the reference's
// cumsum-then-scale order by a few ulp of B, far inside the tolerance; which side an x within that
// distance of a knot falls on is immaterial because the spline and its derivative are continuous there.
// K = 8 (the reference default) locates the bin by bisection on the 9 knots: 3 compares + 30 selects
// carrying {left, right} of both axes and the two derivative logits, instead of a 7-step scan.
// ud_first / ud_last: raw derivative parameters of the two boundary knots.  Linear tails pin both to the constant that
// makes the derivative exactly 1 (:35-38); circular tails (:42-45, :48-57) pass learned values (last = first).
//
// N independent evaluations in one call (lane n: input x[n], parameters w(n, i), h(n, i), d(n, i)), one stage after the
// other for all lanes: each stage is a dependent chain of MUFU ops and FMAs, and the lanes' chains interleave where one
// thread has nothing else to issue.  A lane's arithmetic is that of a single evaluation, expression for expression, so
// its results do not depend on N.  Branch-free up to the inverse root's division, so the lanes stay in one basic block.
template <int N, int K, bool INVERSE, typename PW, typename PH, typename PD>
__host__ __device__ __forceinline__ void rqs_core_lanes(const float (&x)[N], PW pw, PH ph, PD pd, float tail,
                                                        float (&y)[N], float (&lad)[N],
                                                        float ud_first = NFB_BOUNDARY_UD,
                                                        float ud_last = NFB_BOUNDARY_UD) {
    // softmax of the width and height logits -> knots on the unit interval, with the raw derivative parameters
    float kw[N][K + 1], kh[N][K + 1], ud[N][K + 1];
#pragma unroll
    for (int n = 0; n < N; ++n) {
        float mw = pw(n, 0), mh = ph(n, 0);
#pragma unroll
        for (int i = 1; i < K; ++i) {
            mw = fmaxf(mw, pw(n, i));
            mh = fmaxf(mh, ph(n, i));
        }
        float cw[K], ch[K];
        float sw = 0.f, sh = 0.f;
#pragma unroll
        for (int i = 0; i < K; ++i) {
            sw += fast_ex2(pw(n, i) - mw);
            sh += fast_ex2(ph(n, i) - mh);
            cw[i] = sw;
            ch[i] = sh;
        }
        const float aw = (1.f - kMinBinWidth * K) * rcp_nr(sw);
        const float ah = (1.f - kMinBinHeight * K) * rcp_nr(sh);
        kw[n][0] = 0.f; kh[n][0] = 0.f; kw[n][K] = 1.f; kh[n][K] = 1.f;
        ud[n][0] = ud_first; ud[n][K] = ud_last;
#pragma unroll
        for (int i = 0; i < K - 1; ++i) {
            kw[n][i + 1] = fmaf(aw, cw[i], kMinBinWidth * (float)(i + 1));
            kh[n][i + 1] = fmaf(ah, ch[i], kMinBinHeight * (float)(i + 1));
            ud[n][i + 1] = pd(n, i);
        }
    }
    // the bin of x, its derivatives and slope
    const float two_b = 2.f * tail;
    float xu[N], l_w[N], l_h[N], in_w[N], in_h[N], d0[N], d1[N], rw[N], delta[N], s[N];
#pragma unroll
    for (int n = 0; n < N; ++n) {
        xu[n] = fmaf(x[n], rcp_nr(two_b), 0.5f);
        float r_w, r_h, ud0, ud1;
        if (K == 8) {
            const float* ks = INVERSE ? kh[n] : kw[n];
            const bool c1 = xu[n] >= ks[4];
            float a_w[5], a_h[5], a_d[5];
#pragma unroll
            for (int j = 0; j < 5; ++j) {
                a_w[j] = c1 ? kw[n][4 + j] : kw[n][j];
                a_h[j] = c1 ? kh[n][4 + j] : kh[n][j];
                a_d[j] = c1 ? ud[n][4 + j] : ud[n][j];
            }
            const bool c2 = xu[n] >= (INVERSE ? a_h[2] : a_w[2]);
            float b_w[3], b_h[3], b_d[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                b_w[j] = c2 ? a_w[2 + j] : a_w[j];
                b_h[j] = c2 ? a_h[2 + j] : a_h[j];
                b_d[j] = c2 ? a_d[2 + j] : a_d[j];
            }
            const bool c3 = xu[n] >= (INVERSE ? b_h[1] : b_w[1]);
            l_w[n] = c3 ? b_w[1] : b_w[0]; r_w = c3 ? b_w[2] : b_w[1];
            l_h[n] = c3 ? b_h[1] : b_h[0]; r_h = c3 ? b_h[2] : b_h[1];
            ud0 = c3 ? b_d[1] : b_d[0]; ud1 = c3 ? b_d[2] : b_d[1];
        } else {
            l_w[n] = kw[n][0]; r_w = kw[n][1]; l_h[n] = kh[n][0]; r_h = kh[n][1]; ud0 = ud[n][0]; ud1 = ud[n][1];
#pragma unroll
            for (int i = 1; i < K; ++i) {
                if (xu[n] >= (INVERSE ? kh[n][i] : kw[n][i])) {  // knot i <= x
                    l_w[n] = kw[n][i]; r_w = kw[n][i + 1]; l_h[n] = kh[n][i]; r_h = kh[n][i + 1];
                    ud0 = ud[n][i]; ud1 = ud[n][i + 1];
                }
            }
        }
        in_w[n] = r_w - l_w[n];
        in_h[n] = r_h - l_h[n];
        d0[n] = kMinDerivative + softplus_f(ud0);
        d1[n] = kMinDerivative + softplus_f(ud1);
        rw[n] = rcp_nr(in_w[n]);
        delta[n] = in_h[n] * rw[n];
        s[n] = d0[n] + d1[n] - 2.f * delta[n];
    }
    // the rational function and its log-derivative
#pragma unroll
    for (int n = 0; n < N; ++n) {
        const bool inside = (x[n] >= -tail) && (x[n] <= tail);
        float outu, theta, tomt, den;
        if (INVERSE) {
            const float t = xu[n] - l_h[n];
            const float a = t * s[n] + in_h[n] * (delta[n] - d0[n]);
            const float b = in_h[n] * d0[n] - t * s[n];
            const float c = -delta[n] * t;
            theta = rqs_inverse_root(a, b, c);
            outu = theta * in_w[n] + l_w[n];
            tomt = theta * (1.f - theta);
            den = delta[n] + s[n] * tomt;
        } else {
            theta = (xu[n] - l_w[n]) * rw[n];
            tomt = theta * (1.f - theta);
            den = delta[n] + s[n] * tomt;
            const float num = in_h[n] * (delta[n] * theta * theta + d0[n] * tomt);
            outu = l_h[n] + num * rcp_nr(den);
        }
        const float omt = 1.f - theta;
        const float dnum = delta[n] * delta[n] * (d1[n] * theta * theta + 2.f * delta[n] * tomt + d0[n] * omt * omt);
        float l = kLn2 * (fast_lg2(dnum) - 2.f * fast_lg2(den));
        if (INVERSE) l = -l;
        y[n] = inside ? fmaf(outu, two_b, -tail) : x[n];
        lad[n] = inside ? l : 0.f;
    }
}

// one evaluation: lw / lh the logits, pd(i) the interior derivative parameters
template <int K, bool INVERSE, typename PD>
__host__ __device__ __forceinline__ void rqs_core(float x, const float (&lw)[K], const float (&lh)[K], PD pd,
                                                  float tail, float& y, float& lad,
                                                  float ud_first = NFB_BOUNDARY_UD, float ud_last = NFB_BOUNDARY_UD) {
    const float xs[1] = {x};
    float ys[1], ls[1];
    rqs_core_lanes<1, K, INVERSE>(xs, [&lw](int, int i) { return lw[i]; }, [&lh](int, int i) { return lh[i]; },
                                  [&pd](int, int i) { return pd(i); }, tail, ys, ls, ud_first, ud_last);
    y = ys[0];
    lad = ls[0];
}

// Param accessor: P(i) returns the i-th of the 3K-1 raw parameters [w(K) | h(K) | d(K-1)] of this
// element.  `wh_scale` multiplies the w and h logits (1/sqrt(hidden) in the coupling layer,
// neural_spline/coupling.py:334-336; 1 in the autoregressive layer and the unconditional CDF).
template <int K, bool INVERSE, typename P>
__host__ __device__ __forceinline__ void rqs_eval(float x, P p, float tail, float wh_scale, float& y,
                                         float& lad) {
    const float s2 = wh_scale * kLog2e;
    float lw[K], lh[K];
#pragma unroll
    for (int i = 0; i < K; ++i) {
        lw[i] = p(i) * s2;
        lh[i] = p(K + i) * s2;
    }
    rqs_core<K, INVERSE>(x, lw, lh, [&p](int i) { return p(2 * K + i); }, tail, y, lad);
}

// Runtime-K version (K <= 32) reading parameters through the accessor twice; used by the
// generic kernels for bin counts other than 8.
// nd = number of derivative parameters per element: K - 1 (linear tails; boundaries pinned), K (circular: parameter
// i is knot i, knot K repeats knot 0) or K + 1 (per-feature tails list: parameters 0..K are the knots; `circular`
// says whether this feature copies knot 0 into knot K or pins both ends, utils/splines.py:48-57).
template <bool INVERSE, typename P>
__host__ __device__ __forceinline__ void rqs_eval_dyn(int K, float x, P p, float tail, float wh_scale,
                                             float& y, float& lad, int nd = -1, bool circular = false) {
    if (nd < 0) nd = K - 1;
    const int dshift = nd == K - 1 ? 1 : 0;                      // parameter index of knot i is i - dshift
    const float ud_first = (nd == K - 1 || !circular) ? NFB_BOUNDARY_UD : p(2 * K);
    const float ud_last = ud_first;
    const bool inside = (x >= -tail) && (x <= tail);
    const float s2 = wh_scale * kLog2e;
    float mw = -3.0e38f, mh = -3.0e38f;
    for (int i = 0; i < K; ++i) {
        mw = fmaxf(mw, p(i) * s2);
        mh = fmaxf(mh, p(K + i) * s2);
    }
    float sw = 0.f, sh = 0.f;
    for (int i = 0; i < K; ++i) {
        sw += fast_ex2(p(i) * s2 - mw);
        sh += fast_ex2(p(K + i) * s2 - mh);
    }
    const float kw = (1.f - kMinBinWidth * K) * rcp_nr(sw);
    const float kh = (1.f - kMinBinHeight * K) * rcp_nr(sh);
    const float two_b = 2.f * tail;
    float cumw = 0.f, cumh = 0.f, left = -tail, bottom = -tail;
    float in_cw = -tail, in_w = 1.f, in_ch = -tail, in_h = 1.f;
    float ud0 = ud_first, ud1 = ud_last;
    for (int i = 0; i < K; ++i) {
        cumw += kMinBinWidth + kw * fast_ex2(p(i) * s2 - mw);
        cumh += kMinBinHeight + kh * fast_ex2(p(K + i) * s2 - mh);
        const float right = (i == K - 1) ? tail : (two_b * cumw - tail);
        const float top = (i == K - 1) ? tail : (two_b * cumh - tail);
        const bool ge = INVERSE ? (x >= bottom) : (x >= left);
        if (ge) {
            in_cw = left;
            in_w = right - left;
            in_ch = bottom;
            in_h = top - bottom;
            ud0 = (i == 0) ? ud_first : p(2 * K + i - dshift);
            ud1 = (i == K - 1) ? ud_last : p(2 * K + i + 1 - dshift);
        }
        left = right;
        bottom = top;
    }
    const float d0 = kMinDerivative + softplus_f(ud0);
    const float d1 = kMinDerivative + softplus_f(ud1);
    const float rw = rcp_nr(in_w);
    const float delta = in_h * rw;
    const float s = d0 + d1 - 2.f * delta;
    float out, theta, tomt, den;
    if (INVERSE) {
        const float t = x - in_ch;
        const float a = t * s + in_h * (delta - d0);
        const float b = in_h * d0 - t * s;
        const float c = -delta * t;
        theta = rqs_inverse_root(a, b, c);
        out = theta * in_w + in_cw;
        tomt = theta * (1.f - theta);
        den = delta + s * tomt;
    } else {
        theta = (x - in_cw) * rw;
        tomt = theta * (1.f - theta);
        den = delta + s * tomt;
        const float num = in_h * (delta * theta * theta + d0 * tomt);
        out = in_ch + num * rcp_nr(den);
    }
    const float omt = 1.f - theta;
    const float dnum = delta * delta * (d1 * theta * theta + 2.f * delta * tomt + d0 * omt * omt);
    float l = kLn2 * (fast_lg2(dnum) - 2.f * fast_lg2(den));
    if (INVERSE) l = -l;
    // (tails given as a LIST, nd = K + 1: the reference leaves out-of-interval outputs at their zero initialisation,
    //  utils/splines.py:31,48-57 -- no identity copy in that branch; restated as is)
    y = inside ? out : (nd == K + 1 ? 0.f : x);
    lad = inside ? l : 0.f;
}

}  // namespace nfb
