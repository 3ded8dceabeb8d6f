// nfb_affine_bwd.cuh -- element adjoints of the affine family's sampling direction (affine_stack_kernel with
// direction = 1, nfb_affine.cu), with row cotangents g of the op's output and gam of the log-det:
//   MaskedAffineFlow     x = zm + (1-b)(z e^s + t), ld += sum (1-b) s, zm = b z, s = S(zm), t = T(zm)
//                          s_hat = (1-b)(g z e^s + gam),  t_hat = (1-b) g,
//                          g_z = (b + (1-b) e^s) g + b (J_S^T s_hat + J_T^T t_hat)   (the MLP part is added by the caller)
//                        an entry of s or t that is not finite was replaced by NaN in the forward: it passes no gradient
//                        into its MLP (the reference's torch.where)
//   AffineConstFlow      x = z e^s + t:  g_z = g e^s,  per-row contributions g z e^s + gam to g_s and g to g_t
//   AffineCouplingBlock  x2 = z2 e^sc + shift (exp), z2 / sig(sc+2) + shift (sigmoid), z2 sig(sc+2) + shift (sigmoid_inv),
//                        x2 = z2 + param without scale; z1 passes through (its J_P^T part is added by the caller)
// Host/device and templated on the scalar type, so that tests/native can check them in double precision against
// autograd and central differences (tests/test_affine_rkl_training.py, tests/test_affine_fkl_training.py).  Kernels:
// affine_bwd_rows_kernel (nfb_affine.cu).  The density direction's adjoints follow the sampling direction's below.
#pragma once
#include <cmath>

namespace nfb {

__host__ __device__ __forceinline__ float aff_exp(float v) { return expf(v); }
__host__ __device__ __forceinline__ double aff_exp(double v) { return exp(v); }
__host__ __device__ __forceinline__ bool aff_finite(float v) { return isfinite(v); }
__host__ __device__ __forceinline__ bool aff_finite(double v) { return isfinite(v); }

// s, t: the nets' raw outputs (before the NaN substitution); s_hat / t_hat: cotangents of those outputs; g_z: the direct
// part of the input cotangent
template <typename T>
__host__ __device__ inline void masked_affine_adjoint(T z, T b, T s, T t, T g, T gam, T& s_hat, T& t_hat, T& g_z) {
    const bool fs = aff_finite(s), ft = aff_finite(t);
    const T sj = fs ? s : (T)NAN;
    const T e = aff_exp(sj);
    const T ob = (T)1 - b;
    s_hat = fs ? ob * (g * z * e + gam) : (T)0;
    t_hat = ft ? ob * g : (T)0;
    g_z = (b + ob * e) * g;
}

// per-row contributions cs (to g_s) and ct (to g_t)
template <typename T>
__host__ __device__ inline void affine_const_adjoint(T z, T s, T g, T gam, T& g_z, T& cs, T& ct) {
    const T e = aff_exp(s);
    g_z = g * e;
    cs = g * z * e + gam;
    ct = g;
}

// one transformed element v of z2; smap: 0 exp, 1 sigmoid, 2 sigmoid_inv; scale = 0: x2 = v + shift (sc unused)
template <typename T>
__host__ __device__ inline void coupling_adjoint(int scale, int smap, T v, T sc, T g, T gam, T& g_v, T& g_shift,
                                                 T& g_sc) {
    g_shift = g;
    if (!scale) { g_v = g; g_sc = (T)0; return; }
    if (smap == 0) {
        const T e = aff_exp(sc);
        g_v = g * e;
        g_sc = g * v * e + gam;
        return;
    }
    const T sg = (T)1 / ((T)1 + aff_exp(-(sc + (T)2)));
    const T omsg = (T)1 / ((T)1 + aff_exp(sc + (T)2));   // 1 - sg, exact 0 / 1 at the saturations
    if (smap == 1) {   // x2 = v / sg, ld -= log sg
        g_v = g / sg;
        g_sc = -(g * v * omsg / sg + gam * omsg);
    } else {           // x2 = v sg, ld += log sg
        g_v = g * sg;
        g_sc = g * v * sg * omsg + gam * omsg;
    }
}

// ---- density direction (affine_stack_kernel with direction = 0), same conventions: z / v is the op's input ----------
//   MaskedAffineFlow     x = zm + (1-b)(z - t) e^-s, ld -= sum (1-b) s
//                          s_hat = -(1-b)(g (z-t) e^-s + gam),  t_hat = -(1-b) g e^-s,  g_z = (b + (1-b) e^-s) g
//                          (+ b (J_S^T s_hat + J_T^T t_hat), added by the caller); a non-finite s or t passes no gradient
//   AffineConstFlow      x = (z - t) e^-s:  g_z = g e^-s,  per-row contributions -(g (z-t) e^-s + gam) to g_s, -g e^-s to g_t
//   AffineCouplingBlock  x2 = (v - shift) e^-sc (exp), (v - shift) sg (sigmoid), (v - shift) / sg (sigmoid_inv),
//                        sg = sig(sc + 2); x2 = v - param without scale
// Kernel: affine_density_bwd_rows_kernel (nfb_affine.cu).
template <typename T>
__host__ __device__ inline void masked_affine_density_adjoint(T z, T b, T s, T t, T g, T gam, T& s_hat, T& t_hat,
                                                              T& g_z) {
    const bool fs = aff_finite(s), ft = aff_finite(t);
    const T sj = fs ? s : (T)NAN, tj = ft ? t : (T)NAN;
    const T e = aff_exp(-sj);
    const T ob = (T)1 - b;
    s_hat = fs ? -ob * (g * (z - tj) * e + gam) : (T)0;
    t_hat = ft ? -ob * g * e : (T)0;
    g_z = (b + ob * e) * g;
}

template <typename T>
__host__ __device__ inline void affine_const_density_adjoint(T z, T s, T t, T g, T gam, T& g_z, T& cs, T& ct) {
    const T e = aff_exp(-s);
    g_z = g * e;
    cs = -(g * (z - t) * e + gam);
    ct = -g_z;
}

// without scale, `shift` is the whole param entry (x2 = v - param) and sc is unused
template <typename T>
__host__ __device__ inline void coupling_density_adjoint(int scale, int smap, T v, T shift, T sc, T g, T gam, T& g_v,
                                                         T& g_shift, T& g_sc) {
    if (!scale) { g_v = g; g_shift = -g; g_sc = (T)0; return; }
    const T u = v - shift;
    if (smap == 0) {
        const T e = aff_exp(-sc);
        g_v = g * e;
        g_shift = -g_v;
        g_sc = -(g * u * e + gam);
        return;
    }
    const T sg = (T)1 / ((T)1 + aff_exp(-(sc + (T)2)));
    const T omsg = (T)1 / ((T)1 + aff_exp(sc + (T)2));   // 1 - sg, exact 0 / 1 at the saturations
    if (smap == 1) {   // x2 = (v - shift) sg, ld += log sg
        g_v = g * sg;
        g_sc = g * u * sg * omsg + gam * omsg;
    } else {           // x2 = (v - shift) / sg, ld -= log sg
        g_v = g / sg;
        g_sc = -(g * u * omsg / sg + gam * omsg);
    }
    g_shift = -g_v;
}

}  // namespace nfb
