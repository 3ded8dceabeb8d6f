// nfb_affine_wide.cuh -- element formulas of the affine family's wide path (nfb_affine_wide.cu): one feature of one row,
// the op's output and its log-det term, in either direction (dir 1: sampling, 0: density).  They are the float32
// expressions of affine_stack_kernel (nfb_affine.cu), written once here so that the wide kernels and a host-compiled
// check (tests/native/affine_wide_host_check.cu) share them:
//   MaskedAffineFlow     x = b z + (1-b)(z e^s + t), ld (1-b) s;  inverse b z + (1-b)(z - t) e^-s, ld -(1-b) s
//                        (s / t = the nets' outputs; a non-finite entry becomes NaN, flows/affine/coupling.py:209-229)
//   AffineConstFlow      x = z e^s + t, ld s;  inverse (z - t) e^-s, ld -s
//   AffineCouplingBlock  one transformed element v of z2, smap 0 exp, 1 sigmoid (sg = sig(sc + 2), x = v / sg + shift),
//                        2 sigmoid_inv (x = v sg + shift); scale = 0: x = v + shift
// The adjoints are those of nfb_affine_bwd.cuh.  Templated on the scalar type for the double-precision host check.
#pragma once
#include "nfb_affine_bwd.cuh"

namespace nfb {

// AffineCouplingBlock's torch.chunk(2) of the features (flows/affine/coupling.py): z1 = features [o1, o1 + n1) feed the
// net, z2 = [o2, o2 + n2) are transformed; channel_inv swaps the halves.  n1 = ceil(d / 2) for `channel`.
struct CouplingSplit {
    int o1, n1, o2, n2;
    __host__ __device__ CouplingSplit(int d, bool inv_split) {
        const int h = (d + 1) / 2;
        o1 = inv_split ? h : 0; n1 = inv_split ? d - h : h;
        o2 = inv_split ? 0 : h; n2 = d - n1;
    }
};

__host__ __device__ __forceinline__ float aff_log(float v) { return logf(v); }
__host__ __device__ __forceinline__ double aff_log(double v) { return log(v); }

template <typename T>
__host__ __device__ inline void masked_affine_elem(int dir, T z, T b, T s, T t, T& x, T& ld) {
    const T zm = b * z;
    const T sj = aff_finite(s) ? s : (T)NAN;
    const T tj = aff_finite(t) ? t : (T)NAN;
    if (dir) {
        x = zm + ((T)1 - b) * (z * aff_exp(sj) + tj);
        ld = ((T)1 - b) * sj;
    } else {
        x = zm + ((T)1 - b) * (z - tj) * aff_exp(-sj);
        ld = -(((T)1 - b) * sj);
    }
}

template <typename T>
__host__ __device__ inline void affine_const_elem(int dir, T z, T s, T t, T& x, T& ld) {
    x = dir ? z * aff_exp(s) + t : (z - t) * aff_exp(-s);
    ld = dir ? s : -s;
}

template <typename T>
__host__ __device__ inline void coupling_elem(int dir, int scale, int smap, T v, T shift, T sc, T& x, T& ld) {
    ld = (T)0;
    if (!scale) { x = dir ? v + shift : v + -shift; return; }
    if (smap == 0) {
        if (dir) { x = v * aff_exp(sc) + shift; ld = sc; }
        else { x = (v - shift) * aff_exp(-sc); ld = -sc; }
        return;
    }
    const T sg = (T)1 / ((T)1 + aff_exp(-(sc + (T)2)));
    const T lsg = aff_log(sg);
    const bool div = (smap == 1) == (dir != 0);
    if (dir) x = div ? v / sg + shift : v * sg + shift;
    else x = div ? (v - shift) / sg : (v - shift) * sg;
    ld = div ? -lsg : lsg;
}

}  // namespace nfb
