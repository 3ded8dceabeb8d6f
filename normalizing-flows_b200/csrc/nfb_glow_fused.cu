// nfb_glow_fused.cu -- the whole Glow conditioner (nets/cnn.py:33-61 ConvNet2d with kernel sizes (3, 1, 3), the
// parameter map of a GlowBlock's affine coupling, flows/affine/glow.py:48-62) as ONE wgmma kernel per call:
//
//   h1 = act(conv3x3(x[:, c0:c0+cin]) + b1)      [pixels x H]      GEMM 1: im2col A (K = 9 cin <= 256), N = H
//   h2 = act(conv1x1(h1) + b2)                   [pixels x H]      GEMM 2: K = H, N = H
//   Y  = h2 W3'^T                                [pixels x 9 cout] GEMM 3: the last 3x3 convolution as nine stacked
//                                                                  1x1 products (summed with shifts by tap_shift_add_kernel)
//
// Per 64-pixel tile the two hidden tensors never leave the SM: each GEMM is computed in 64-column output slices whose
// accumulators live in the registers of one warpgroup; the epilogue converts a slice (bias, LeakyReLU, bf16 hi/lo
// split) straight into the other of two swizzled A-operand buffers in shared memory, which the next GEMM reads.
//
// Numerics: split-bf16 (a w ~= a_hi w_hi + a_lo w_hi + a_hi w_lo), fp32 accumulation, weights packed with the
// accumulate-truncation gain (nfb_kernels.h kAccStepGain), like csrc/nfb_conv_tc.cu.
//
// Structure (160 threads, persistent: CTA b takes tiles b, b + grid, ...):
//   warps 0-3  one warpgroup: im2col builder of GEMM 1, wgmma issue and every epilogue
//   warp 4     weight producer: bulk TMA of pre-swizzled [64 x 64] hi | lo records (one output slice x one K-chunk)
//              into a 4 x 16 KB ring
#include "nfb_kernels.h"

namespace nfb {

namespace {
constexpr int kGfRows = 64;
constexpr int kGfCons = 128;
constexpr int kGfThreads = kGfCons + 32;
constexpr uint32_t kGfTileA = 8192;             // [64 x 64] bf16
constexpr uint32_t kGfBufA = 8 * kGfTileA;      // hi K-chunks 0..3 | lo K-chunks 0..3
constexpr uint32_t kGfRec = 16384;              // one record: [64 x 64] hi | lo
constexpr uint32_t kGfSlots = 4;
constexpr uint32_t kGfOffW = 2 * kGfBufA;       // 131072
constexpr uint32_t kGfOffBars = kGfOffW + kGfSlots * kGfRec;  // 196608
constexpr uint32_t kGfSmem = kGfOffBars + 8 * 8;

__device__ __forceinline__ uint32_t gf_chunk_off(int r, int c8) {
    return (r >> 3) * 1024 + (r & 7) * 128 + ((c8 ^ (r & 7)) << 4);
}
__device__ __forceinline__ void gf_st_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void gf_st_b32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void gf_split_store8(const float* v, uint32_t t_hi, uint32_t t_lo, uint32_t off) {
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float a = v[2 * i], b = v[2 * i + 1];
        hi[i] = pack_bf16x2(a, b);
        lo[i] = pack_bf16x2(a - __uint_as_float(hi[i] << 16), b - __uint_as_float(hi[i] & 0xffff0000u));
    }
    gf_st_v4(t_hi + off, hi[0], hi[1], hi[2], hi[3]);
    gf_st_v4(t_lo + off, lo[0], lo[1], lo[2], lo[3]);
}
__device__ __forceinline__ void gf_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kGfCons) : "memory"); }
}  // namespace

struct GlowCondParams {
    const float* x; float* y;            // x: [B, ctot, H, W]; y: [B, n3_real, H, W]
    const float* b1; const float* b2;    // [hidden]
    const uint8_t* wstream;              // records: GEMM 1 (hid/64 slices x k1c), GEMM 2 (hid/64 x hid/64), GEMM 3 (n3/64 x hid/64)
    long long M;                         // B * H * W pixels
    int ctot, c0, cin, H, W, hid, k1c, n3, n3_real;
    float leaky;
    int* err;
};

__global__ void __launch_bounds__(kGfThreads, 1) glow_cond_kernel(const GlowCondParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t bars = sbase + kGfOffBars;   // [0, 4) full, [4, 8) empty
    auto bar = [bars](int i) { return bars + 8u * i; };
    if (threadIdx.x == 0) {
        for (int i = 0; i < (int)kGfSlots; ++i) { mbar_init(bar(i), 1); mbar_init(bar(4 + i), 1); }
        fence_mbar_init();
    }
    __syncthreads();
    const long long n_tiles = (p.M + kGfRows - 1) / kGfRows;
    const int kch = p.hid >> 6;                       // K chunks (and output slices) of the hidden GEMMs
    const int n_rec = kch * p.k1c + kch * kch + (p.n3 >> 6) * kch;

    if (warp == kGfCons / 32) {
        // ------------------------------ weight producer -----------------------------------
        uint32_t slot = 0, par = 0;
        for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
            for (int i = 0; i < n_rec; ++i) {
                mbar_wait(bar(4 + slot), par ^ 1, p.err, 900 + slot);
                if (elect_one_sync()) {
                    mbar_expect_tx(bar(slot), kGfRec);
                    bulk_g2s(sbase + kGfOffW + slot * kGfRec, p.wstream + (size_t)i * kGfRec, kGfRec, bar(slot));
                }
                __syncwarp();
                if (++slot == kGfSlots) { slot = 0; par ^= 1; }
            }
        }
        return;
    }

    // ------------------------------ consumer warpgroup ------------------------------------
    const int et = threadIdx.x;
    const int ra = 16 * warp + (lane >> 2), rb = ra + 8, cq = 2 * (lane & 3);
    const uint32_t aBuf[2] = {sbase, sbase + kGfBufA};
    const int HW = p.H * p.W;
    uint32_t slot = 0, wpar = 0;
    // one 64-column output slice: kcs records (K-chunks 0 .. kcs-1 of A buffer a_buf) into acc
    auto run_slice = [&](float (&acc)[32], uint32_t a_buf, int kcs) {
        for (int kc = 0; kc < kcs; ++kc) {
            mbar_wait(bar(slot), wpar, p.err, 920 + slot);
            const uint32_t w = sbase + kGfOffW + slot * kGfRec;
            const uint64_t ah = wgmma_desc(a_buf + kc * kGfTileA), al = wgmma_desc(a_buf + (4 + kc) * kGfTileA);
            const uint64_t bh = wgmma_desc(w), bl = wgmma_desc(w + 8192);
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, ah + 2 * j, bh + 2 * j, (kc | j) ? 1u : 0u);
#pragma unroll
            for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, al + 2 * j, bh + 2 * j, 1u);
#pragma unroll
            for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, ah + 2 * j, bl + 2 * j, 1u);
            wgmma_commit();
            wgmma_wait<0>();
            if (et == 0) mbar_arrive(bar(4 + slot));
            if (++slot == kGfSlots) { slot = 0; wpar ^= 1; }
        }
        wgmma_hold(acc);
    };
    // hidden epilogue: bias, LeakyReLU, bf16 hi/lo -> K-chunk j of a_out
    auto hidden_epilogue = [&](const float (&acc)[32], int j, const float* bias, uint32_t a_out) {
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + 64 * j + 8 * g + cq));
#pragma unroll
            for (int hb = 0; hb < 2; ++hb) {
                const int rr = hb ? rb : ra;
                float v0 = acc[4 * g + 2 * hb] + b2.x, v1 = acc[4 * g + 2 * hb + 1] + b2.y;
                v0 = v0 >= 0.f ? v0 : v0 * p.leaky;
                v1 = v1 >= 0.f ? v1 : v1 * p.leaky;
                const uint32_t hi = pack_bf16x2(v0, v1);
                const uint32_t lo = pack_bf16x2(v0 - __uint_as_float(hi << 16), v1 - __uint_as_float(hi & 0xffff0000u));
                const uint32_t off = (rr >> 3) * 1024 + (rr & 7) * 128 + ((g ^ (rr & 7)) << 4) + cq * 2;
                gf_st_b32(a_out + j * kGfTileA + off, hi);
                gf_st_b32(a_out + (4 + j) * kGfTileA + off, lo);
            }
        }
    };

    for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        // ---- GEMM 1 operand: im2col, k = c * 9 + tap (the natural flattening of W1[n, c, kh, kw]);
        //      thread = (pixel, half of every K-chunk) ----
        {
            const int r = et & (kGfRows - 1), half = et >> 6;
            const long long m = t * kGfRows + r;
            const bool live = m < p.M;
            const long long bi = live ? m / HW : 0;
            const int pix = live ? (int)(m - bi * HW) : 0;
            const int ph = pix / p.W, pw = pix - ph * p.W;
            const float* xb = p.x + (bi * p.ctot + p.c0) * (long long)HW;
            for (int kc = 0; kc < p.k1c; ++kc) {
#pragma unroll
                for (int g8 = 0; g8 < 4; ++g8) {
                    float v[8];
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int k = kc * 64 + half * 32 + g8 * 8 + j;
                        const int c = k / 9, tap = k - c * 9;
                        const int kh = tap / 3, kw = tap - kh * 3;
                        const int hh = ph + kh - 1, ww = pw + kw - 1;
                        v[j] = (live && c < p.cin && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W)
                                   ? __ldg(xb + (long long)c * HW + hh * p.W + ww) : 0.f;
                    }
                    gf_split_store8(v, aBuf[0] + kc * kGfTileA, aBuf[0] + (4 + kc) * kGfTileA, gf_chunk_off(r, half * 4 + g8));
                }
            }
            fence_proxy_async_smem();
            gf_bar_sync();
        }
        // ---- hidden GEMMs: buffer 0 -> buffer 1 -> buffer 0 ----
        for (int g = 0; g < 2; ++g) {
            const uint32_t a_in = aBuf[g], a_out = aBuf[g ^ 1];
            for (int j = 0; j < kch; ++j) {
                float acc[32];
                run_slice(acc, a_in, g == 0 ? p.k1c : kch);
                hidden_epilogue(acc, j, g == 0 ? p.b1 : p.b2, a_out);
            }
            fence_proxy_async_smem();
            gf_bar_sync();
        }
        // ---- output: Y[b, n, pix] = accumulator column n ----
        const long long ma = t * kGfRows + ra, mb = t * kGfRows + rb;
        const long long bia = ma / HW, bib = mb / HW;
        float* ya = p.y + bia * (long long)p.n3_real * HW + (ma - bia * HW);
        float* yb = p.y + bib * (long long)p.n3_real * HW + (mb - bib * HW);
        for (int j = 0; j < (p.n3 >> 6); ++j) {
            float acc[32];
            run_slice(acc, aBuf[0], kch);
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                const int c = 64 * j + 8 * (i >> 2) + cq + (i & 1);
                const bool hb = (i & 2) != 0;
                if (c < p.n3_real && (hb ? mb : ma) < p.M) (hb ? yb : ya)[(long long)c * HW] = acc[i];
            }
        }
        gf_bar_sync();   // every thread is done with this tile's A buffers before the next tile's im2col
    }
}

// weights -> bf16 hi | lo SWIZZLE_128B records, one per (64-row output slice j, K-chunk kc), slice-major.
// src: row-major [rows_real x k_real] (ld = k_real); rows >= rows_real and k >= k_real are zero.
__global__ void glow_pack_kernel(const float* __restrict__ w, int rows_real, int k_real, int n_slices, int kcs, float gain,
                                 uint8_t* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)n_slices * kcs * 64 * 64) return;
    const int kk = (int)(idx & 63), n = (int)((idx >> 6) & 63);
    const int rec = (int)(idx >> 12), j = rec / kcs, kc = rec - j * kcs;
    const int row = 64 * j + n, k = kc * 64 + kk;
    const float v = (row < rows_real && k < k_real) ? w[(long long)row * k_real + k] * gain : 0.f;
    const size_t off = (size_t)(n >> 3) * 1024 + (n & 7) * 128 + (((kk >> 3) ^ (n & 7)) << 4) + (kk & 7) * 2;
    uint8_t* r = out + (size_t)rec * 16384;  // hi tile, then lo tile
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    *reinterpret_cast<__nv_bfloat16*>(r + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(r + 8192 + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
}

bool glow_cond_supported(int cin, int hid, int cout, int k1, int k2, int k3) {
    return k1 == 3 && k2 == 1 && k3 == 3 && hid % 64 == 0 && hid >= 64 && hid <= 256 && cin >= 1 && 9 * cin <= 256 &&
           cout >= 1 && 9 * cout <= 512;
}

// packed weight image of one conditioner: GEMM 1 records, GEMM 2 records, GEMM 3 records (16 KB each)
size_t glow_cond_packed_bytes(int cin, int hid, int cout) {
    const int k1c = (9 * cin + 63) / 64, kch = hid / 64;
    const int n3 = (9 * cout + 63) / 64 * 64;
    return ((size_t)kch * k1c + (size_t)kch * kch + (size_t)(n3 / 64) * kch) * 16384;
}
// w3t: the last convolution's weights rearranged to [9 * cout, hid] (row tap * cout + n = W3[n, :, kh, kw]).
int launch_glow_cond_pack(const float* w1, const float* w2, const float* w3t, int cin, int hid, int cout,
                          float gain_per_step, uint8_t* packed, cudaStream_t st) {
    NFB_CHECK(glow_cond_supported(cin, hid, cout, 3, 1, 3), NFB_ERR_UNSUPPORTED, "glow conditioner: unsupported shape");
    const int k1 = 9 * cin, k1c = (k1 + 63) / 64, kch = hid / 64;
    const int n3_real = 9 * cout, n3 = (n3_real + 63) / 64 * 64;
    auto pack = [&](const float* w, int rows, int kreal, int n_slices, int kcs, uint8_t* dst) {
        const long long total = (long long)n_slices * kcs * 64 * 64;
        const float gain = 1.f + gain_per_step * (float)(12 * kcs);
        glow_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, rows, kreal, n_slices, kcs, gain, dst);
    };
    pack(w1, hid, k1, kch, k1c, packed);
    pack(w2, hid, hid, kch, kch, packed + (size_t)kch * k1c * 16384);
    pack(w3t, n3_real, hid, n3 / 64, kch, packed + ((size_t)kch * k1c + (size_t)kch * kch) * 16384);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
// packed != null: the caller keeps the packed image (one pack per parameter version); else packed per call
int launch_glow_conditioner(const float* x, int ctot, int c0, int cin, const float* w1, const float* b1, const float* w2,
                            const float* b2, const float* w3t, const uint8_t* packed, float* y_taps, long long B, int H,
                            int W, int hid, int cout, float leaky, float gain_per_step, int* err, cudaStream_t st) {
    static PerDevice per_dev;
    const int sm_count = per_dev.ensure([] {
        return cudaFuncSetAttribute(glow_cond_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGfSmem);
    });
    if (sm_count < 0) return NFB_ERR_CUDA;
    NFB_CHECK(glow_cond_supported(cin, hid, cout, 3, 1, 3), NFB_ERR_UNSUPPORTED, "glow conditioner: unsupported shape");
    const long long M = B * H * W;
    if (M == 0) return NFB_OK;
    const int k1 = 9 * cin, k1c = (k1 + 63) / 64;
    const int n3_real = 9 * cout, n3 = (n3_real + 63) / 64 * 64;
    uint8_t* scratch = nullptr;
    if (!packed) {
        NFB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&scratch), glow_cond_packed_bytes(cin, hid, cout), st));
        const int rc = launch_glow_cond_pack(w1, w2, w3t, cin, hid, cout, gain_per_step, scratch, st);
        if (rc) { cudaFreeAsync(scratch, st); return rc; }
        packed = scratch;
    }
    GlowCondParams p{};
    p.x = x; p.y = y_taps; p.b1 = b1; p.b2 = b2; p.wstream = packed; p.M = M; p.ctot = ctot; p.c0 = c0; p.cin = cin;
    p.H = H; p.W = W; p.hid = hid; p.k1c = k1c; p.n3 = n3; p.n3_real = n3_real; p.leaky = leaky; p.err = err;
    const long long n_tiles = (M + kGfRows - 1) / kGfRows;
    const unsigned grid = (unsigned)(n_tiles < sm_count ? n_tiles : sm_count);
    glow_cond_kernel<<<grid, kGfThreads, kGfSmem, st>>>(p);
    const cudaError_t e = cudaGetLastError();
    if (scratch) cudaFreeAsync(scratch, st);
    if (e != cudaSuccess) {
        nfb_set_error("glow_cond launch: %s", cudaGetErrorString(e));
        return NFB_ERR_CUDA;
    }
    return NFB_OK;
}

}  // namespace nfb
