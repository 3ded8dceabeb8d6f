// nfb_maf_bwd.cuh -- adjoint of one element of MaskedAffineAutoregressive's density pass
// (flows/affine/autoregressive.py:96-128, inverse branch):
//   scale = sigmoid(u + 2) + 1e-3,   y = (x - shift) / scale,   log_det = -sum_j log scale_j
// with (u, shift) the interleaved pair of the conditioner output.  Host/device and templated on the scalar type so that
// tests/native can check it in double precision against autograd and finite differences (tests/test_maf_training.py).
// Kernel: maf_affine_adjoint_kernel (nfb_backward.cu).
//
// Given the cotangent lam of y (g_y plus the conditioner's data gradient of the previous fixed-point pass) and g_ld of
// log_det, it returns the cotangents of the conditioner outputs and of x:
//   pbar_shift = -lam / scale,   pbar_u = -(sig (1 - sig) / scale) (lam y + g_ld),   g_x = lam / scale.
// y is recomputed from x and (u, shift) with the forward's own expression, so no saved y is read.  1 - sig is formed as
// 1 / (1 + 1 / e), e = exp(-(u + 2)), which stays accurate where sig rounds to 1 and gives exactly 0 at either
// saturation (e = 0 or e = inf) instead of inf * 0.
#pragma once
#include <cmath>

namespace nfb {

__host__ __device__ __forceinline__ float maf_exp(float v) { return expf(v); }
__host__ __device__ __forceinline__ double maf_exp(double v) { return exp(v); }

template <typename T>
__host__ __device__ inline void maf_affine_adjoint(T x, T u, T shift, T lam, T g_ld, T& pbar_u, T& pbar_shift, T& g_x) {
    const T e = maf_exp(-(u + (T)2));
    const T sig = (T)1 / ((T)1 + e);
    const T scale = sig + (T)1e-3;
    const T y = (x - shift) / scale;
    const T dsig = sig * ((T)1 / ((T)1 + (T)1 / e));   // sig (1 - sig)
    g_x = lam / scale;
    pbar_shift = -g_x;
    pbar_u = -(dsig / scale) * (lam * y + g_ld);
}

}  // namespace nfb
