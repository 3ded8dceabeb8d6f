// nfb_glow.cu -- image-shaped (NCHW) pieces of the Glow block, density direction:
//   GlowBlock.inverse = ActNorm.inverse -> Invertible1x1Conv.inverse -> AffineCouplingBlock.inverse
//   (flows/affine/glow.py:79-84; normalization.py:31-39; mixing.py:123-133; coupling.py:149-171,262-267)
// ActNorm and the 1x1 convolution are both per-pixel affine maps over channels, so they are folded into ONE
// 1x1 convolution W' = (P L U) diag(exp(-s)), b' = -W' t at pack time (`glow_fold_kernel`) and run through
// the same implicit-GEMM kernel as the ConvNet2d conditioner (nets/cnn.py:33-61: 3x3 -> 1x1 -> 3x3 with
// LeakyReLU).  The coupling epilogue applies shift/scale (interleaved channels, coupling.py:152-160) and
// reduces log|det| per sample.  Conditioner-sized convolutions run on the wgmma implicit GEMM (nfb_conv_tc.cu);
// the small maps stay on the plain fp32 FFMA tiles below.
#include <cstdlib>
#include "nfb_kernels.h"

namespace nfb {

// y[b,n,h,w] = act( sum_{c,kh,kw} w[n,c,kh,kw] * x[b, c0+c, h+kh-p, w+kw-p] + bias[n] ),  stride 1, pad k/2.
// Implicit GEMM: M = B*H*W pixels, N = Cout, K = Cin*k*k; 64x64 tile, 4x4 per thread.
__global__ void __launch_bounds__(256)
conv2d_kernel(const float* __restrict__ x, int ctot, int c0, const float* __restrict__ w,
              const float* __restrict__ bias, float* __restrict__ y, long long B, int cin, int H, int W,
              int cout, int ks, float leaky, const float* __restrict__ mask, float mslope, int accumulate) {
    __shared__ float As[16][64 + 1];
    __shared__ float Bs[16][64 + 1];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const long long M = B * H * W;
    const int K = cin * ks * ks, pad = ks >> 1, HW = H * W, kk2 = ks * ks;
    const long long m0 = (long long)blockIdx.x * 64;
    const int n0 = blockIdx.y * 64;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += 16) {
        for (int i = threadIdx.x; i < 64 * 16; i += 256) {
            const int r = i & 63, k = i >> 6;  // r fastest: consecutive threads -> consecutive pixels
            const long long m = m0 + r;
            const int kk = k0 + k;
            float a = 0.f, b = 0.f;
            if (kk < K) {
                if (m < M) {
                    const int c = kk / kk2, rem = kk - c * kk2, kh = rem / ks, kw = rem - kh * ks;
                    const long long bi = m / HW;
                    const int pix = (int)(m - bi * HW), h = pix / W, ww = pix - h * W;
                    const int hh = h + kh - pad, w2 = ww + kw - pad;
                    if (hh >= 0 && hh < H && w2 >= 0 && w2 < W)
                        a = x[((bi * ctot + c0 + c) * H + hh) * W + w2];
                }
                if (n0 + r < cout) b = w[(long long)(n0 + r) * K + kk];
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
        const long long bi = m / HW;
        const int pix = (int)(m - bi * HW);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= cout) continue;
            float v = acc[i][j] + (bias ? bias[n] : 0.f);
            if (leaky >= 0.f) v = v >= 0.f ? v : v * leaky;
            const long long yo = (bi * cout + n) * HW + pix;
            if (mask) v *= mask[yo] > 0.f ? 1.f : mslope;
            if (accumulate) v += y[yo];
            y[yo] = v;
        }
    }
}

// 1x1 convolution with few channels (the folded ActNorm + Invertible1x1Conv of a Glow block, C <= 64): one
// thread per pixel keeps its cin inputs in registers, the [cout x cin] matrix sits in shared memory and is read
// as warp-wide broadcasts.  HBM-bound: 4 (cin + cout) bytes per pixel, no tile padding to 64 channels.
template <int CMAX>
__global__ void __launch_bounds__(256)
conv1x1_small_kernel(const float* __restrict__ x, int ctot, int c0, const float* __restrict__ w,
                     const float* __restrict__ bias, float* __restrict__ y, long long M, int cin, int HW, int cout,
                     float leaky, const float* __restrict__ mask, float mslope, int accumulate) {
    __shared__ float ws[CMAX * CMAX];
    __shared__ float bs[CMAX];
    for (int i = threadIdx.x; i < cout * cin; i += 256) ws[i] = w[i];
    for (int i = threadIdx.x; i < cout; i += 256) bs[i] = bias ? bias[i] : 0.f;
    __syncthreads();
    const long long m = (long long)blockIdx.x * 256 + threadIdx.x;
    if (m >= M) return;
    const long long bi = m / HW;
    const int pix = (int)(m - bi * HW);
    const float* xp = x + (bi * ctot + c0) * (long long)HW + pix;
    float v[CMAX];
#pragma unroll
    for (int c = 0; c < CMAX; ++c) v[c] = c < cin ? xp[(long long)c * HW] : 0.f;
    float* yp = y + bi * (long long)cout * HW + pix;
    for (int n = 0; n < cout; ++n) {
        const float* wr = ws + n * cin;
        float acc = bs[n];
#pragma unroll
        for (int c = 0; c < CMAX; ++c)
            if (c < cin) acc = fmaf(wr[c], v[c], acc);
        if (leaky >= 0.f) acc = acc >= 0.f ? acc : acc * leaky;
        const long long yo = (bi * cout + n) * (long long)HW + pix;
        if (mask) acc *= mask[yo] > 0.f ? 1.f : mslope;
        if (accumulate) acc += yp[(long long)n * HW];
        yp[(long long)n * HW] = acc;
    }
}

int launch_conv2d(const float* x, int ctot, int c0, const float* w, const float* bias, float* y, long long B,
                  int cin, int H, int W, int cout, int ks, float leaky, cudaStream_t st, const float* mask,
                  float mask_slope, int accumulate) {
    NFB_CHECK(ks == 1 || ks == 3 || ks == 5, NFB_ERR_UNSUPPORTED, "conv2d: kernel size %d", ks);
    NFB_CHECK(c0 >= 0 && c0 + cin <= ctot, NFB_ERR_ARG, "conv2d: channel slice out of range");
    const long long M = B * H * W;
    if (M == 0 || cout == 0) return NFB_OK;
    // conditioner-sized convolutions run on the tensor core (sm_90 only; NFB_CONV_FP32=1 forces this kernel)
    static const bool tc = [] {
        int dev = 0, major = 0;
        if (getenv("NFB_CONV_FP32")) return false;
        if (cudaGetDevice(&dev) != cudaSuccess) return false;
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
        return major == 9;
    }();
    if (ks == 1 && cin <= 64 && cout <= 64) {
        const unsigned g = (unsigned)((M + 255) / 256);
        if (cin <= 16 && cout <= 16)
            conv1x1_small_kernel<16><<<g, 256, 0, st>>>(x, ctot, c0, w, bias, y, M, cin, H * W, cout, leaky, mask,
                                                          mask_slope, accumulate);
        else if (cin <= 32 && cout <= 32)
            conv1x1_small_kernel<32><<<g, 256, 0, st>>>(x, ctot, c0, w, bias, y, M, cin, H * W, cout, leaky, mask,
                                                          mask_slope, accumulate);
        else
            conv1x1_small_kernel<64><<<g, 256, 0, st>>>(x, ctot, c0, w, bias, y, M, cin, H * W, cout, leaky, mask,
                                                          mask_slope, accumulate);
        NFB_LAUNCH_CHECK();
        return NFB_OK;
    }
    if (tc && conv_tc_supported(cin, cout, ks))
        return launch_conv2d_tc(x, ctot, c0, w, bias, y, B, cin, H, W, cout, ks, leaky, kAccStepGain, nullptr, st, mask,
                                mask_slope, accumulate);
    dim3 grid((unsigned)((M + 63) / 64), (unsigned)((cout + 63) / 64));
    conv2d_kernel<<<grid, 256, 0, st>>>(x, ctot, c0, w, bias, y, B, cin, H, W, cout, ks, leaky, mask, mask_slope,
                                        accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// W = P (tril(L,-1)+I) (triu(U,1) + diag(sign_S exp(log_S)))      (mixing.py:88-104, density direction)
// w_out[o,c] = W[o,c] exp(-s[c]);  b_out[o] = -sum_c w_out[o,c] t[c]   (ActNorm.inverse folded in)
// logdet = HW * (sum log_S - sum s)                                  (mixing.py:125,132; coupling.py:47-54)
__global__ void glow_fold_kernel(const float* __restrict__ P, const float* __restrict__ L,
                                 const float* __restrict__ U, const float* __restrict__ sign_S,
                                 const float* __restrict__ log_S, const float* __restrict__ s,
                                 const float* __restrict__ t, int C, int HW, float* __restrict__ w_out,
                                 float* __restrict__ b_out, float* __restrict__ logdet) {
    extern __shared__ float sh[];
    float* LU = sh;          // C*C : L' U'
    float* Wm = sh + C * C;  // C*C : P L' U'
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
        const int r = i / C, c = i % C;
        float acc = 0.f;
        for (int k = 0; k < C; ++k) {
            const float l = (k < r) ? L[r * C + k] : (k == r ? 1.f : 0.f);
            const float u = (c > k) ? U[k * C + c] : (c == k ? sign_S[k] * expf(log_S[k]) : 0.f);
            acc = fmaf(l, u, acc);
        }
        LU[i] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
        const int r = i / C, c = i % C;
        float acc = 0.f;
        for (int k = 0; k < C; ++k) acc = fmaf(P[r * C + k], LU[k * C + c], acc);
        Wm[i] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) w_out[i] = Wm[i] * expf(-s[i % C]);
    for (int o = threadIdx.x; o < C; o += blockDim.x) {
        float acc = 0.f;
        for (int c = 0; c < C; ++c) acc = fmaf(Wm[o * C + c] * expf(-s[c]), t[c], acc);
        b_out[o] = -acc;
    }
    if (threadIdx.x == 0) {
        float a = 0.f;
        for (int c = 0; c < C; ++c) a += log_S[c] - s[c];
        *logdet = a * (float)HW;
    }
}
int launch_glow_fold(const float* P, const float* L, const float* U, const float* sign_S, const float* log_S,
                     const float* s, const float* t, int C, int HW, float* w_out, float* b_out, float* logdet,
                     cudaStream_t st) {
    NFB_CHECK(C >= 1 && C <= 128, NFB_ERR_UNSUPPORTED, "Invertible1x1Conv: channels %d > 128", C);
    const size_t smem = (size_t)2 * C * C * sizeof(float);
    NFB_CUDA(cudaFuncSetAttribute(glow_fold_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    glow_fold_kernel<<<1, 256, smem, st>>>(P, L, U, sign_S, log_S, s, t, C, HW, w_out, b_out, logdet);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Sampling direction: Invertible1x1Conv.forward (mixing.py:106-121, LU branch :94-101: the reference forms
// W^-1 = U'^-1 L'^-1 P^T in DOUBLE precision) followed by ActNorm.forward (coupling.py:38-45), folded:
// w_out[o,c] = exp(s[o]) Winv[o,c];  b_out[o] = t[o];  logdet = HW * (sum s - sum log_S).
// One block, fp64 triangular inverses by substitution (one column per thread), C <= 64.
__global__ void glow_fold_fwd_kernel(const float* __restrict__ P, const float* __restrict__ L,
                                     const float* __restrict__ U, const float* __restrict__ sign_S,
                                     const float* __restrict__ log_S, const float* __restrict__ s,
                                     const float* __restrict__ t, int C, int HW, float* __restrict__ w_out,
                                     float* __restrict__ b_out, float* __restrict__ logdet) {
    extern __shared__ double shd[];
    double* Lm = shd;              // C*C unit lower
    double* Um = shd + C * C;      // C*C upper incl. diagonal
    double* Li = shd + 2 * C * C;  // L^-1
    double* Ui = shd + 3 * C * C;  // U^-1
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
        const int r = i / C, c = i % C;
        Lm[i] = c < r ? (double)L[i] : (c == r ? 1.0 : 0.0);
        Um[i] = c > r ? (double)U[i] : (c == r ? (double)sign_S[r] * exp((double)log_S[r]) : 0.0);
        Li[i] = 0.0;
        Ui[i] = 0.0;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        for (int r = 0; r < C; ++r) {  // column c of L^-1
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = c; k < r; ++k) v -= Lm[r * C + k] * Li[k * C + c];
            Li[r * C + c] = (r < c) ? 0.0 : v;
        }
        for (int r = C - 1; r >= 0; --r) {  // column c of U^-1
            double v = (r == c) ? 1.0 : 0.0;
            for (int k = r + 1; k <= c; ++k) v -= Um[r * C + k] * Ui[k * C + c];
            Ui[r * C + c] = (r > c) ? 0.0 : v / Um[r * C + r];
        }
    }
    __syncthreads();
    // T = U^-1 L^-1 (reuse Lm), then Winv = T P^T: Winv[o,c] = sum_k T[o,k] P[c,k]
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
        const int r = i / C, c = i % C;
        double acc = 0.0;
        for (int k = (r > c ? r : c); k < C; ++k) acc += Ui[r * C + k] * Li[k * C + c];
        Um[i] = acc;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C * C; i += blockDim.x) {
        const int o = i / C, c = i % C;
        double acc = 0.0;
        for (int k = 0; k < C; ++k) acc += Um[o * C + k] * (double)P[c * C + k];
        w_out[i] = (float)(acc * exp((double)s[o]));
    }
    for (int o = threadIdx.x; o < C; o += blockDim.x) b_out[o] = t[o];
    if (threadIdx.x == 0) {
        double a = 0.0;
        for (int c = 0; c < C; ++c) a += (double)s[c] - (double)log_S[c];
        *logdet = (float)(a * HW);
    }
}
int launch_glow_fold_fwd(const float* P, const float* L, const float* U, const float* sign_S, const float* log_S,
                         const float* s, const float* t, int C, int HW, float* w_out, float* b_out, float* logdet,
                         cudaStream_t st) {
    NFB_CHECK(C >= 1 && C <= 64, NFB_ERR_UNSUPPORTED, "Invertible1x1Conv sampling direction: channels %d > 64", C);
    const size_t smem = (size_t)4 * C * C * sizeof(double);
    NFB_CUDA(cudaFuncSetAttribute(glow_fold_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    glow_fold_fwd_kernel<<<1, 256, smem, st>>>(P, L, U, sign_S, log_S, s, t, C, HW, w_out, b_out, logdet);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// AffineCoupling on images, in place on the z2 channels of z [B,C,H,W]; param [B, (scale?2:1)*n2, H, W].
// One block per sample; log_det[b] (+)= sum log-scale terms + *logdet_const.
__global__ void __launch_bounds__(256)
coupling_image_kernel(float* __restrict__ z, const float* __restrict__ param, float* __restrict__ logdet,
                      const float* __restrict__ logdet_const, int C, int HW, int scale, int smap, int inv_split,
                      int direction, int accumulate) {
    const long long b = blockIdx.x;
    const int h = (C + 1) / 2;
    const int o2 = inv_split ? 0 : h, n2 = inv_split ? h : C - h;  // channel_inv: z2 is the FIRST chunk
    const int np = scale ? 2 : 1;
    float ld = 0.f;
    for (int i = threadIdx.x; i < n2 * HW; i += 256) {
        const int c = i / HW, pix = i - c * HW;
        float& v = z[(b * C + o2 + c) * HW + pix];
        if (!scale) {
            const float pm = param[(b * n2 + c) * HW + pix];
            v = direction ? v + pm : v - pm;
            continue;
        }
        const float shift = param[(b * np * n2 + 2 * c) * HW + pix];
        const float sc = param[(b * np * n2 + 2 * c + 1) * HW + pix];
        if (smap == 0) {
            if (direction) { v = v * expf(sc) + shift; ld += sc; }
            else { v = (v - shift) * expf(-sc); ld -= sc; }
        } else {
            const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
            const float lsg = logf(sg);
            const bool div = (smap == 1) == (direction != 0);
            if (direction) v = div ? v / sg + shift : v * sg + shift;
            else v = div ? (v - shift) / sg : (v - shift) * sg;
            ld += div ? -lsg : lsg;
        }
    }
    __shared__ float red[8];
    ld = warp_sum(ld);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ld;
    __syncthreads();
    if (threadIdx.x == 0 && logdet) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        if (logdet_const) t += *logdet_const;
        logdet[b] = accumulate ? logdet[b] + t : t;
    }
}
int launch_coupling_image(float* z, const float* param, float* logdet, const float* logdet_const, long long B,
                          int C, int HW, int scale, int smap, int inv_split, int direction, int accumulate,
                          cudaStream_t st) {
    if (B == 0) return NFB_OK;
    coupling_image_kernel<<<(unsigned)B, 256, 0, st>>>(z, param, logdet, logdet_const, C, HW, scale, smap,
                                                       inv_split, direction, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// The same coupling with its parameters still in "tap" form: the last 3x3 convolution of the conditioner leaves nine
// stacked 1x1 products Y [B, 9 * cout, H, W] (csrc/nfb_glow_fused.cu; cout = np * n2), and param[b, n, y, x] = bias[n] +
// sum_t Y[b, t * cout + n, y + kh - 1, x + kw - 1].  One block per sample stages that sample's Y (<= 200 KB) in shared
// memory with coalesced 16-byte loads and forms the two parameters of every element on the fly: the summed parameter
// tensor is never written, and the nine-fold read happens once, from shared memory (round 2a: tap_shift_add_kernel 55 us +
// coupling_image_kernel 9 us per GlowBlock at C3's first level).
__global__ void __launch_bounds__(256)
coupling_taps_kernel(float* __restrict__ z, const float* __restrict__ Y, const float* __restrict__ bias,
                     float* __restrict__ logdet, const float* __restrict__ logdet_const, int C, int H, int W, int scale,
                     int smap, int inv_split, int direction, int accumulate) {
    extern __shared__ __align__(16) float sy[];
    const long long b = blockIdx.x;
    const int HW = H * W;
    const int h = (C + 1) / 2;
    const int o2 = inv_split ? 0 : h, n2 = inv_split ? h : C - h;
    const int np = scale ? 2 : 1, cout = np * n2;
    const long long per = 9LL * cout * HW;
    const float* src = Y + b * per;
    if ((per & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(sy);
        for (int i = threadIdx.x; i < (int)(per >> 2); i += 256) d4[i] = __ldg(s4 + i);
    } else {
        for (int i = threadIdx.x; i < (int)per; i += 256) sy[i] = __ldg(src + i);
    }
    __syncthreads();
    auto param = [&](int n, int y, int x) {
        float acc = bias ? __ldg(bias + n) : 0.f;
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
            const int yy = y + kh - 1;
            if (yy < 0 || yy >= H) continue;
#pragma unroll
            for (int kw = 0; kw < 3; ++kw) {
                const int xx = x + kw - 1;
                if (xx < 0 || xx >= W) continue;
                acc += sy[((kh * 3 + kw) * cout + n) * HW + yy * W + xx];
            }
        }
        return acc;
    };
    float ld = 0.f;
    for (int i = threadIdx.x; i < n2 * HW; i += 256) {
        const int c = i / HW, pix = i - c * HW;
        const int y = pix / W, x = pix - y * W;
        float& v = z[(b * C + o2 + c) * HW + pix];
        if (!scale) {
            const float pm = param(c, y, x);
            v = direction ? v + pm : v - pm;
            continue;
        }
        const float shift = param(2 * c, y, x);
        const float sc = param(2 * c + 1, y, x);
        if (smap == 0) {
            if (direction) { v = v * expf(sc) + shift; ld += sc; }
            else { v = (v - shift) * expf(-sc); ld -= sc; }
        } else {
            const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
            const float lsg = logf(sg);
            const bool div = (smap == 1) == (direction != 0);
            if (direction) v = div ? v / sg + shift : v * sg + shift;
            else v = div ? (v - shift) / sg : (v - shift) * sg;
            ld += div ? -lsg : lsg;
        }
    }
    __shared__ float red[8];
    ld = warp_sum(ld);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ld;
    __syncthreads();
    if (threadIdx.x == 0 && logdet) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        if (logdet_const) t += *logdet_const;
        logdet[b] = accumulate ? logdet[b] + t : t;
    }
}
bool coupling_taps_supported(int C, int H, int W, int scale) {
    const int h = (C + 1) / 2;
    const long long worst = 9LL * (scale ? 2 : 1) * h * H * W * 4;   // the larger of the two possible z2 chunks
    return worst <= 200 * 1024;
}
int launch_coupling_taps(float* z, const float* Y, const float* bias, float* logdet, const float* logdet_const, long long B,
                         int C, int H, int W, int scale, int smap, int inv_split, int direction, int accumulate,
                         cudaStream_t st) {
    if (B == 0) return NFB_OK;
    NFB_CHECK(coupling_taps_supported(C, H, W, scale), NFB_ERR_UNSUPPORTED, "coupling_taps: sample too large for shared memory");
    const int h = (C + 1) / 2;
    const int n2 = inv_split ? h : C - h;
    const size_t smem = (size_t)9 * (scale ? 2 : 1) * n2 * H * W * 4;
    static PerDevice per_dev;
    if (per_dev.ensure([] {
            return cudaFuncSetAttribute(coupling_taps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        }) < 0)
        return NFB_ERR_CUDA;
    coupling_taps_kernel<<<(unsigned)B, 256, smem, st>>>(z, Y, bias, logdet, logdet_const, C, H, W, scale, smap, inv_split,
                                                         direction, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Squeeze (flows/reshape.py:114-128).  direction 0 = inverse: [B,C,H,W] -> [B,4C,H/2,W/2]; 1 = forward.
__global__ void squeeze_kernel(const float* __restrict__ in, float* __restrict__ out, long long B, int C, int H,
                               int W, int direction) {
    // (C,H,W) always describe the LARGE-resolution side: big[b,c,2h2+i,2w2+j] <-> small[b,4c+2i+j,h2,w2]
    const long long n = B * C * H * W;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    const int w = (int)(idx % W), h = (int)((idx / W) % H), c = (int)((idx / ((long long)W * H)) % C);
    const long long b = idx / ((long long)W * H * C);
    const int h2 = h >> 1, i = h & 1, w2 = w >> 1, j = w & 1;
    const long long sidx = ((b * (4 * C) + 4 * c + 2 * i + j) * (H / 2) + h2) * (W / 2) + w2;
    if (direction == 0) out[sidx] = in[idx];
    else out[idx] = in[sidx];
}
int launch_squeeze(const float* in, float* out, long long B, int C, int H, int W, int direction, cudaStream_t st) {
    NFB_CHECK(H % 2 == 0 && W % 2 == 0, NFB_ERR_ARG, "squeeze: H and W must be even");
    const long long n = B * C * H * W;
    if (n == 0) return NFB_OK;
    squeeze_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, B, C, H, W, direction);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[b, j, :] = in[b, c0 + j, :]   (channel chunk of an NCHW tensor made contiguous; Split/Merge, reshape.py:27-31)
__global__ void copy_channels_kernel(const float* __restrict__ in, float* __restrict__ out, long long B, int C,
                                     int c0, int n, int HW) {
    const long long total = B * n * HW;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const long long b = idx / ((long long)n * HW);
    const long long rem = idx - b * n * HW;
    out[idx] = in[(b * C + c0) * HW + rem];
}
int launch_copy_channels(const float* in, float* out, long long B, int C, int c0, int n, int HW, cudaStream_t st) {
    NFB_CHECK(c0 >= 0 && n >= 0 && c0 + n <= C, NFB_ERR_ARG, "copy_channels: slice out of range");
    const long long total = B * n * HW;
    if (total == 0) return NFB_OK;
    copy_channels_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, B, C, c0, n, HW);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// out[b, c0 + j, :] = in[b, j, :]   (Merge.forward on images, reshape.py:68-74: the inverse of copy_channels)
__global__ void paste_channels_kernel(const float* __restrict__ in, float* __restrict__ out, long long B, int C,
                                      int c0, int n, int HW) {
    const long long total = B * n * HW;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const long long b = idx / ((long long)n * HW);
    const long long rem = idx - b * n * HW;
    out[(b * C + c0) * HW + rem] = in[idx];
}
int launch_paste_channels(const float* in, float* out, long long B, int C, int c0, int n, int HW, cudaStream_t st) {
    NFB_CHECK(c0 >= 0 && n >= 0 && c0 + n <= C, NFB_ERR_ARG, "paste_channels: slice out of range");
    const long long total = B * n * HW;
    if (total == 0) return NFB_OK;
    paste_channels_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, out, B, C, c0, n, HW);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// ClassCondDiagGaussian.log_prob (distributions/base.py:327-344): loc/log_scale [dim, num_classes], y[b] int64.
__global__ void __launch_bounds__(256)
class_cond_gauss_kernel(const float* __restrict__ z, const long long* __restrict__ y,
                        const float* __restrict__ loc, const float* __restrict__ log_scale,
                        float* __restrict__ logq, int dim, int ncls, int accumulate) {
    const long long b = blockIdx.x;
    const int cls = (int)y[b];
    float s = 0.f;
    for (int i = threadIdx.x; i < dim; i += 256) {
        const float ls = log_scale[(long long)i * ncls + cls];
        const float t = (z[b * dim + i] - loc[(long long)i * ncls + cls]) / expf(ls);
        s += ls + 0.5f * t * t;
    }
    __shared__ float red[8];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < 8; ++i) t += red[i];
        const float lp = -0.5f * (float)dim * 1.8378770664093453f - t;
        logq[b] = accumulate ? logq[b] + lp : lp;
    }
}
int launch_class_cond_gauss(const float* z, const long long* y, const float* loc, const float* log_scale,
                            float* logq, long long B, int dim, int ncls, int accumulate, cudaStream_t st) {
    if (B == 0) return NFB_OK;
    class_cond_gauss_kernel<<<(unsigned)B, 256, 0, st>>>(z, y, loc, log_scale, logq, dim, ncls, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// Input pre-transforms of MultiscaleFlow (normflows/transforms.py): Logit (:8-47) and Shift (:50-75).
// One block per sample: element-wise map + block reduction of the per-sample log-det.  HBM-bound (8 B/element).
//   direction NFB_INVERSE (density pass, Logit.inverse): y = log(u) - log(1-u), u = alpha + beta x,
//       log_det = log(beta) n - sum(log u + log(1-u))
//   direction NFB_FORWARD (sampling, Logit.forward):     y = (sigmoid(x) - alpha) / beta,
//       log_det = -log(beta) n + sum(logsigmoid(x) + logsigmoid(-x))
// -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) logit_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                    float* __restrict__ logdet, long long inner, float alpha,
                                                    int direction, int accumulate) {
    const long long b = blockIdx.x;
    const float beta = 1.f - 2.f * alpha;
    const float* src = in + b * inner;
    float* dst = out + b * inner;
    float acc = 0.f;
    for (long long i = threadIdx.x; i < inner; i += 256) {
        const float x = src[i];
        if (direction == 0) {
            const float u = alpha + beta * x;
            const float lu = logf(u), l1 = logf(1.f - u);
            dst[i] = lu - l1;
            acc -= lu + l1;
        } else {
            // logsigmoid(x) = -softplus(-x); stable for both signs
            const float ax = fabsf(x);
            const float sp = log1pf(expf(-ax));           // softplus(-|x|)
            const float ls_pos = -sp - fmaxf(-x, 0.f);    // logsigmoid(x)
            const float ls_neg = -sp - fmaxf(x, 0.f);     // logsigmoid(-x)
            dst[i] = (1.f / (1.f + expf(-x)) - alpha) / beta;
            acc += ls_pos + ls_neg;
        }
    }
    __shared__ float red[8];
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0 && logdet) {
        float s = 0.f;
        for (int j = 0; j < 8; ++j) s += red[j];
        const float c = logf(beta) * (float)inner;
        const float v = direction == 0 ? c + s : -c + s;
        logdet[b] = accumulate ? logdet[b] + v : v;
    }
}
int launch_logit(const float* in, float* out, float* logdet, long long B, long long inner, float alpha, int direction,
                 int accumulate, cudaStream_t st) {
    if (B == 0 || inner == 0) return NFB_OK;
    logit_kernel<<<(unsigned)B, 256, 0, st>>>(in, out, logdet, inner, alpha, direction, accumulate);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// Last convolution of the Glow conditioner (nets/cnn.py:50-57: k x k, 256 -> few channels) as k*k 1x1 products + a
// shifted sum.  An im2col GEMM spends its time gathering K = 256 k^2 values per pixel for a handful of outputs
// (measured: 456 us, tensor pipe 5 % active); instead ONE 1x1 convolution with the taps stacked along the output
// channels, Y[b, tap*cout + n] = sum_c W[n, c, tap] h[b, c] (K = 256, N = k^2 cout: the tensor-core kernel at a
// 1x1 conv's cost), followed by this HBM-bound pass:
//   out[b, n, y, x] = bias[n] + sum_{kh, kw} Y[b, (kh k + kw) cout + n, y + kh - p, x + kw - p]    (zero outside)
// -----------------------------------------------------------------------------------------
__global__ void tap_shift_add_kernel(const float* __restrict__ Y, const float* __restrict__ bias, float* __restrict__ out,
                                     long long B, int cout, int H, int W, int ks) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long HW = (long long)H * W;
    if (i >= B * cout * HW) return;
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int n = (int)((i / HW) % cout);
    const long long b = i / (HW * cout);
    const int p = ks >> 1;
    float acc = bias ? bias[n] : 0.f;
    const float* yb = Y + b * (long long)(ks * ks * cout) * HW;
    for (int kh = 0; kh < ks; ++kh) {
        const int yy = y + kh - p;
        if (yy < 0 || yy >= H) continue;
        for (int kw = 0; kw < ks; ++kw) {
            const int xx = x + kw - p;
            if (xx < 0 || xx >= W) continue;
            acc += yb[((long long)((kh * ks + kw) * cout + n)) * HW + (long long)yy * W + xx];
        }
    }
    out[i] = acc;
}
int launch_tap_shift_add(const float* Y, const float* bias, float* out, long long B, int cout, int H, int W, int ks,
                         cudaStream_t st) {
    const long long n = B * cout * H * W;
    if (n == 0) return NFB_OK;
    tap_shift_add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(Y, bias, out, B, cout, H, W, ks);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// Training pass of the image path (density direction): adjoints of the operators above.
// -----------------------------------------------------------------------------------------

// Data gradient of a stride-1 "same" k x k convolution: gx = conv(gy, w') with w'[c, n, kh, kw] = w[n, c, k-1-kh, k-1-kw]
// (in/out swapped, taps rotated by 180 degrees), i.e. the forward convolution kernels with the epilogue options
// mask (LeakyReLU' of the layer input's stored activation) and accumulate.
__global__ void conv_rot180_kernel(const float* __restrict__ w, float* __restrict__ wr, int cout, int cin, int ks) {
    const int T = ks * ks;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)cout * cin * T) return;
    const int tap = (int)(i % T), c = (int)((i / T) % cin), n = (int)(i / ((long long)T * cin));
    wr[((long long)c * cout + n) * T + (T - 1 - tap)] = w[i];
}
int launch_conv2d_dgrad(const float* gy, const float* w, float* gx, long long B, int cin, int H, int W, int cout, int ks,
                        const float* mask, float mask_slope, int accumulate, cudaStream_t st) {
    NFB_CHECK(ks == 1 || ks == 3 || ks == 5, NFB_ERR_UNSUPPORTED, "conv2d_dgrad: kernel size %d", ks);
    if (B * H * W == 0 || cin == 0) return NFB_OK;
    const long long n = (long long)cout * cin * ks * ks;
    void* wr = nullptr;
    NFB_CUDA(cudaMallocAsync(&wr, (size_t)n * sizeof(float), st));
    conv_rot180_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(w, static_cast<float*>(wr), cout, cin, ks);
    const int rc = launch_conv2d(gy, cout, 0, static_cast<const float*>(wr), nullptr, gx, B, cout, H, W, cin, ks, -1.f, st,
                                 mask, mask_slope, accumulate);
    cudaFreeAsync(wr, st);
    return rc;
}

// Adjoint of coupling_image_kernel in the density direction (direction 0; coupling.py:149-171), one block per sample.
// z: the coupling's input [B, C, HW]; param [B, np*n2, HW] (shift 0::2, scale 1::2); g_out [B, C, HW]; g_ld [B] or NULL.
// Writes the z2 channels of g_z (the z1 channels are the caller's: they pass through and feed the conditioner) and g_param.
__global__ void __launch_bounds__(256)
coupling_image_bwd_kernel(const float* __restrict__ z, const float* __restrict__ param, const float* __restrict__ g_out,
                          const float* __restrict__ g_ld, float* __restrict__ g_z, float* __restrict__ g_param, int C,
                          int HW, int scale, int smap, int inv_split) {
    const long long b = blockIdx.x;
    const int h = (C + 1) / 2;
    const int o2 = inv_split ? 0 : h, n2 = inv_split ? h : C - h;
    const int np = scale ? 2 : 1;
    const float gl = g_ld ? g_ld[b] : 0.f;
    for (int i = threadIdx.x; i < n2 * HW; i += 256) {
        const int c = i / HW, pix = i - c * HW;
        const long long zi = (b * C + o2 + c) * HW + pix;
        const float go = g_out[zi];
        if (!scale) {
            g_z[zi] = go;
            g_param[(b * n2 + c) * HW + pix] = -go;
            continue;
        }
        const long long ps = (b * np * n2 + 2 * c) * HW + pix, pc = ps + HW;
        const float d = z[zi] - param[ps], sc = param[pc];
        float f, gsc;   // out = d * f;  d out / d sc and d ld / d sc folded into gsc
        if (smap == 0) {
            f = expf(-sc);
            gsc = -go * d * f - gl;
        } else {
            const float sg = 1.f / (1.f + expf(-(sc + 2.f)));
            if (smap == 1) {   // out = d sg, ld += log sg
                f = sg;
                gsc = (go * d * sg + gl) * (1.f - sg);
            } else {           // out = d / sg, ld -= log sg
                f = 1.f / sg;
                gsc = -(go * d * f + gl) * (1.f - sg);
            }
        }
        g_z[zi] = go * f;
        g_param[ps] = -go * f;
        g_param[pc] = gsc;
    }
}
int launch_coupling_image_bwd(const float* z, const float* param, const float* g_out, const float* g_ld, float* g_z,
                              float* g_param, long long B, int C, int HW, int scale, int smap, int inv_split,
                              cudaStream_t st) {
    if (B == 0) return NFB_OK;
    coupling_image_bwd_kernel<<<(unsigned)B, 256, 0, st>>>(z, param, g_out, g_ld, g_z, g_param, C, HW, scale, smap,
                                                           inv_split);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Adjoint of the diagonal-Gaussian densities of the image bases (DiagGaussian, ClassCondDiagGaussian, GlowBase):
//   log_q[b] = -d/2 log 2pi - sum_i ( ls[e(i), y_b] + (z[b, i] - loc[e(i), y_b])^2 / (2 exp(2 ls)) ),  e(i) = i / group,
// tables [dim / group, ncls] (ncls = 1 and y = NULL: one table).  g_z[b, i] = -g[b] t / sigma (t = (z - loc) / sigma);
// the table gradients are deterministic: per-(sample, entry) partial sums, then a fixed-order sum over the batch per
// (entry, class) -- no float atomics.
__global__ void gauss_table_bwd_rows_kernel(const float* __restrict__ z, const long long* __restrict__ y,
                                            const float* __restrict__ loc, const float* __restrict__ log_scale,
                                            const float* __restrict__ g_lq, float* __restrict__ g_z,
                                            float* __restrict__ part, long long B, int dim, int group, int ncls) {
    const int E = dim / group;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * E) return;
    const long long b = idx / E;
    const int e = (int)(idx - b * E);
    const int cls = y ? (int)y[b] : 0;
    const float mu = loc[(long long)e * ncls + cls], ls = log_scale[(long long)e * ncls + cls];
    const float inv = expf(-ls), g = g_lq[b];
    float pl = 0.f, ps = 0.f;
    for (int j = 0; j < group; ++j) {
        const long long i = b * dim + (long long)e * group + j;
        const float t = (z[i] - mu) * inv;
        if (g_z) g_z[i] = -g * t * inv;
        pl += t * inv;
        ps += t * t - 1.f;
    }
    part[idx] = g * pl;
    part[B * E + idx] = g * ps;
}
__global__ void gauss_table_bwd_sum_kernel(const float* __restrict__ part, const long long* __restrict__ y,
                                           float* __restrict__ g_loc, float* __restrict__ g_log_scale, long long B,
                                           int E, int ncls) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= E * ncls) return;
    const int e = idx / ncls, k = idx - e * ncls;
    double sl = 0.0, ss = 0.0;
    for (long long b = 0; b < B; ++b) {
        if (y && (int)y[b] != k) continue;
        sl += part[b * E + e];
        ss += part[B * E + b * E + e];
    }
    if (g_loc) g_loc[idx] = (float)sl;
    if (g_log_scale) g_log_scale[idx] = (float)ss;
}
int launch_gauss_table_bwd(const float* z, const long long* y, const float* loc, const float* log_scale,
                           const float* g_lq, float* g_z, float* g_loc, float* g_log_scale, long long B, int dim,
                           int group, int ncls, cudaStream_t st) {
    NFB_CHECK(group >= 1 && dim % group == 0 && ncls >= 1, NFB_ERR_ARG, "gauss_table_bwd: bad table shape");
    const int E = dim / group;
    if (B == 0) {
        if (g_loc) NFB_CUDA(cudaMemsetAsync(g_loc, 0, (size_t)E * ncls * sizeof(float), st));
        if (g_log_scale) NFB_CUDA(cudaMemsetAsync(g_log_scale, 0, (size_t)E * ncls * sizeof(float), st));
        return NFB_OK;
    }
    void* part = nullptr;
    NFB_CUDA(cudaMallocAsync(&part, (size_t)2 * B * E * sizeof(float), st));
    gauss_table_bwd_rows_kernel<<<(unsigned)((B * E + 255) / 256), 256, 0, st>>>(
        z, y, loc, log_scale, g_lq, g_z, static_cast<float*>(part), B, dim, group, ncls);
    gauss_table_bwd_sum_kernel<<<(unsigned)((E * ncls + 255) / 256), 256, 0, st>>>(
        static_cast<const float*>(part), y, g_loc, g_log_scale, B, E, ncls);
    const cudaError_t e = cudaGetLastError();
    cudaFreeAsync(part, st);
    if (e != cudaSuccess) {
        nfb_set_error("gauss_table_bwd launch: %s", cudaGetErrorString(e));
        return NFB_ERR_CUDA;
    }
    return NFB_OK;
}

// Adjoint of Logit.inverse (logit_kernel, direction NFB_INVERSE): u = alpha + beta x, y = log u - log(1 - u),
// log_det = n log beta - sum(log u + log(1 - u)):
//   g_x = beta / (u (1 - u)) * (g_y - g_ld (1 - 2 u))
__global__ void logit_bwd_kernel(const float* __restrict__ in, const float* __restrict__ g_out,
                                 const float* __restrict__ g_ld, float* __restrict__ g_in, long long B, long long inner,
                                 float alpha) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * inner) return;
    const float beta = 1.f - 2.f * alpha;
    const float u = alpha + beta * in[i];
    const float gl = g_ld ? g_ld[i / inner] : 0.f;
    const float go = g_out ? g_out[i] : 0.f;
    g_in[i] = beta / (u * (1.f - u)) * (go - gl * (1.f - 2.f * u));
}
int launch_logit_bwd(const float* in, const float* g_out, const float* g_ld, float* g_in, long long B, long long inner,
                     float alpha, cudaStream_t st) {
    const long long n = B * inner;
    if (n == 0) return NFB_OK;
    logit_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, g_out, g_ld, g_in, B, inner, alpha);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb

