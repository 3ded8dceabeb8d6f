// nfb_conv_tc.cu -- stride-1 "same" convolution of the Glow conditioner (nets/cnn.py:33-61, ConvNet2d) as an
// implicit GEMM on the sm_90a tensor core (wgmma).
//
//   y[b, n, h, w] = act( sum_{c,kh,kw} W[n, c, kh, kw] x[b, c0+c, h+kh-p, w+kw-p] + bias[n] )
//   M = B*H*W pixels (128 per work unit), N = cout in tiles of NT = 64 or 128 columns, K in chunks of 64.
//   K order: k = cb*(T*16) + tap*16 + ci for channel c = 16 cb + ci and tap = kh*k + kw (T = k*k), i.e. blocks
//   of 16 channels, tap-major inside a block.  A 16-wide group of k is then ONE tap of 16 consecutive channels:
//   one bounds check and one base address per group, the 16 loads differ by the plane stride only, while all T taps
//   of a channel block stay within 2-3 chunks, so the shifted re-reads of the same 16 planes hit L1.  Channels are
//   zero-padded to a multiple of 16.
//
// Numerics: the same split-bf16 scheme as the spline conditioner (a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo,
// fp32 accumulation, weights packed with the accumulate-truncation gain, see nfb_api.cu kAccStepGain).
//
// Structure (256 threads = two warpgroups, persistent over (pixel tile, n tile) units): thread = (pixel, half of the
// K-chunk) gathers 32 im2col values per chunk (consecutive threads = consecutive pixels -> coalesced; the taps of a
// channel hit L1), splits them to bf16 hi/lo into the SWIZZLE_128B A tile of a two-stage ring while the previous
// chunk is on the tensor core; thread 0 streams the pre-packed weight record of the chunk ([NT x 64] hi | lo) with
// 1-D bulk TMA.  Warpgroup w multiplies pixels [64 w, 64 w + 64); the epilogue (bias, LeakyReLU, NCHW store,
// coalesced per channel) goes through a shared-memory staging tile.
#include "nfb_kernels.h"

namespace nfb {

namespace {
constexpr int kCtThreads = 256;
constexpr uint32_t kCtTileA = 16384;   // [128 x 64] bf16
constexpr uint32_t kCtSmemMax = 232448;

__device__ __forceinline__ uint32_t ct_chunk_off(int r, int c8) {
    return (r >> 3) * 1024 + (r & 7) * 128 + ((c8 ^ (r & 7)) << 4);
}
__device__ __forceinline__ void ct_st_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void ct_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kCtThreads) : "memory"); }
constexpr int ct_n_tile(int n_pad) { return n_pad > 64 ? 128 : 64; }
}  // namespace

struct ConvTcParams {
    const float* x; float* y; const float* bias; const uint8_t* wstream;
    long long M; int ctot, c0, cin, H, W, cout, ks, n_tiles, k_chunks; float leaky; int* err;
};

template <int NT>
__global__ void __launch_bounds__(kCtThreads, 1) conv_tc_kernel(const ConvTcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int NREG = NT / 2;
    constexpr uint32_t b_tile = (uint32_t)NT * 128u;
    constexpr uint32_t stage_bytes = 2 * kCtTileA + 2 * b_tile;   // A hi | A lo | W hi | W lo
    constexpr int kStgLd = NT + 1;
    const uint32_t sbase = smem_u32(smem);
    const int bt = threadIdx.x, wg = bt >> 7, warp = (bt >> 5) & 3, lane = bt & 31;
    const uint32_t bars = sbase + 2 * stage_bytes;   // [0, 2): weight record of stage s landed
    float* stg = reinterpret_cast<float*>(smem + 2 * stage_bytes + 64);
    if (bt == 0) {
        mbar_init(bars, 1);
        mbar_init(bars + 8, 1);
        fence_mbar_init();
    }
    __syncthreads();
    const int KC = p.k_chunks;
    const long long m_tiles = (p.M + 127) / 128;
    const long long n_units = m_tiles * p.n_tiles;
    const int HW = p.H * p.W, pad = p.ks >> 1, ks = p.ks, kk2 = ks * ks;
    const int r = bt & 127, half = bt >> 7;   // A-tile row (pixel) and half of the K-chunk this thread gathers
    const int inv_ks = 65536 / ks + 1;        // tap / ks for tap < 25

    struct Pos { long long u, mt; int nt, kc; };
    auto unit_pos = [&](long long u, int kc) {
        Pos q;
        q.u = u; q.kc = kc;
        q.mt = u / p.n_tiles;
        q.nt = (int)(u - q.mt * p.n_tiles);
        return q;
    };
    // the two 16-wide k groups G = 4 kc + 2 half + {0, 1} of this thread: one tap of channel block cb each
    float v[2][16];
    auto gather = [&](const Pos& q) {
        const long long m = q.mt * 128 + r;
        const bool live = m < p.M;
        const long long bi = live ? m / HW : 0;
        const int pix = live ? (int)(m - bi * HW) : 0;
        const int h = pix / p.W, w = pix - h * p.W;
        const float* xb = p.x + (bi * p.ctot + p.c0) * (long long)HW;
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const int G = 4 * q.kc + 2 * half + g;
            const int cb = G / kk2, tap = G - cb * kk2;
            const int kh = (tap * inv_ks) >> 16, kw = tap - kh * ks;
            const int hh = h + kh - pad, ww = w + kw - pad;
            const bool ok = live && hh >= 0 && hh < p.H && ww >= 0 && ww < p.W;
            const int cbase = cb * 16;
            const int nvalid = ok ? p.cin - cbase : 0;  // channels of this block that exist (<= 0: none)
            const float* src = xb + ((cbase * p.H + hh) * p.W + ww);  // one pointer, stepped by the plane stride
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                v[g][j] = 0.f;
                if (j < nvalid) v[g][j] = __ldg(src);
                src += HW;
            }
        }
    };
    uint32_t full_use[2] = {0, 0};
    auto emit = [&](const Pos& q, int s) {   // weight record by TMA, A chunk split into the stage
        const uint32_t sa = sbase + s * stage_bytes;
        if (bt == 0) {
            mbar_expect_tx(bars + 8 * s, 2 * b_tile);
            bulk_g2s(sa + 2 * kCtTileA, p.wstream + ((size_t)q.nt * KC + q.kc) * (2 * b_tile), 2 * b_tile, bars + 8 * s);
        }
#pragma unroll
        for (int g = 0; g < 2; ++g)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float a = v[g][8 * e + 2 * i], b = v[g][8 * e + 2 * i + 1];
                    hi[i] = pack_bf16x2(a, b);
                    lo[i] = pack_bf16x2(a - __uint_as_float(hi[i] << 16), b - __uint_as_float(hi[i] & 0xffff0000u));
                }
                const uint32_t off = ct_chunk_off(r, 4 * half + 2 * g + e);
                ct_st_v4(sa + off, hi[0], hi[1], hi[2], hi[3]);
                ct_st_v4(sa + kCtTileA + off, lo[0], lo[1], lo[2], lo[3]);
            }
        fence_proxy_async_smem();
    };
    auto mma_chunk = [&](float (&acc)[NREG], int s, bool first) {
        const uint32_t sa = sbase + s * stage_bytes;
        const uint64_t ah = wgmma_desc(sa + wg * 8192u), al = wgmma_desc(sa + kCtTileA + wg * 8192u);
        const uint64_t bh = wgmma_desc(sa + 2 * kCtTileA), bl = wgmma_desc(sa + 2 * kCtTileA + b_tile);
        auto mma = [&](uint64_t a, uint64_t b, uint32_t sd) {
            if constexpr (NT == 64) wgmma_bf16_n64(acc, a, b, sd);
            else wgmma_bf16_n128(acc, a, b, sd);
        };
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) mma(ah + 2 * j, bh + 2 * j, (first && j == 0) ? 0u : 1u);
#pragma unroll
        for (int j = 0; j < 4; ++j) mma(al + 2 * j, bh + 2 * j, 1u);
#pragma unroll
        for (int j = 0; j < 4; ++j) mma(ah + 2 * j, bl + 2 * j, 1u);
        wgmma_commit();
    };
    auto epilogue = [&](const Pos& q, const float (&acc)[NREG]) {
        const int r0 = 64 * wg + 16 * warp + (lane >> 2);
#pragma unroll
        for (int i = 0; i < NREG; ++i)
            stg[(r0 + ((i & 2) ? 8 : 0)) * kStgLd + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1)] = acc[i];
        ct_bar_sync();
        const long long m = q.mt * 128 + r;
        if (m < p.M) {
            const long long bi = m / HW;
            const int pix = (int)(m - bi * HW);
            float* yb = p.y + bi * (long long)p.cout * HW + pix;
            for (int j = half; j < NT; j += 2) {   // consecutive threads: consecutive pixels of one channel
                const int n = q.nt * NT + j;
                if (n < p.cout) {
                    float val = stg[r * kStgLd + j] + (p.bias ? __ldg(p.bias + n) : 0.f);
                    if (p.leaky >= 0.f) val = val >= 0.f ? val : val * p.leaky;
                    yb[(long long)n * HW] = val;
                }
            }
        }
        ct_bar_sync();   // the staging tile is reused by the next unit
    };

    if ((long long)blockIdx.x >= n_units) return;
    float acc[NREG];
    Pos cur = unit_pos(blockIdx.x, 0);
    gather(cur);
    emit(cur, 0);
    ct_bar_sync();
    for (int s = 0;; s ^= 1) {
        Pos nxt = cur;
        if (++nxt.kc == KC) nxt = unit_pos(cur.u + gridDim.x, 0);
        const bool has_next = nxt.u < n_units;
        if (has_next) gather(nxt);   // in flight during this chunk's MMAs
        mbar_wait(bars + 8 * s, full_use[s] & 1u, p.err, 710 + s);
        ++full_use[s];
        mma_chunk(acc, s, cur.kc == 0);
        if (has_next) emit(nxt, s ^ 1);   // (stage s ^ 1 was read by the previous chunk: complete, see below)
        wgmma_wait<0>();
        wgmma_hold(acc);
        ct_bar_sync();   // both warpgroups are done with stage s, and stage s ^ 1 holds the next chunk
        if (cur.kc == KC - 1) epilogue(cur, acc);
        if (!has_next) break;
        cur = nxt;
    }
}

// weights [cout, cin, k, k] fp32 -> one record per (n tile, K-chunk): [NT x 64] hi | lo, SWIZZLE_128B, K in the kernel's
// order
__global__ void conv_pack_kernel(const float* __restrict__ w, int cout, int cin, int T, int NT, int n_tiles, int k_chunks,
                                 float gain, uint8_t* __restrict__ out) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)k_chunks * n_tiles * NT * 64;
    if (idx >= total) return;
    const int kk = (int)(idx & 63);
    const long long rowg = idx >> 6;                  // row of the padded [n_tiles * NT] weight matrix, chunk-major
    const int kc = (int)(rowg / ((long long)n_tiles * NT));
    const int ng = (int)(rowg - (long long)kc * n_tiles * NT);
    const int nt = ng / NT, n = ng - nt * NT;
    const int G = kc * 4 + (kk >> 4), ci = kk & 15;
    const int cb = G / T, tap = G - cb * T, c = cb * 16 + ci;
    const float v = (ng < cout && c < cin) ? w[((long long)ng * cin + c) * T + tap] * gain : 0.f;
    const size_t off = (size_t)(n >> 3) * 1024 + (n & 7) * 128 + (((kk >> 3) ^ (n & 7)) << 4) + (kk & 7) * 2;
    uint8_t* rec = out + ((size_t)nt * k_chunks + kc) * NT * 256;
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    *reinterpret_cast<__nv_bfloat16*>(rec + off) = hi;
    *reinterpret_cast<__nv_bfloat16*>(rec + (size_t)NT * 128 + off) = __float2bfloat16_rn(v - __bfloat162float(hi));
}

bool conv_tc_supported(int cin, int cout, int ks) {
    const int K = cin * ks * ks;
    // small square maps (the folded ActNorm + Invertible1x1Conv, which transforms z itself) stay on the fp32 kernel
    return (ks == 1 || ks == 3 || ks == 5) && cout >= 1 && cout <= 256 && (cout > 64 || K > 64);
}

template <int NT>
int launch_conv_tc_t(const ConvTcParams& p, cudaStream_t st) {
    static PerDevice per_dev;  // attribute + SM count of the device this launch goes to (not the first one seen)
    constexpr uint32_t smem = 2 * (2 * kCtTileA + 2 * (uint32_t)NT * 128u) + 64 + 128 * (NT + 1) * 4;
    static_assert(smem <= kCtSmemMax, "conv_tc: shared memory");
    const int sm_count = per_dev.ensure([] {
        return cudaFuncSetAttribute(conv_tc_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    });
    if (sm_count < 0) return NFB_ERR_CUDA;
    const long long n_units = (p.M + 127) / 128 * p.n_tiles;
    const unsigned grid = (unsigned)(n_units < sm_count ? n_units : sm_count);
    conv_tc_kernel<NT><<<grid, kCtThreads, smem, st>>>(p);
    return NFB_OK;
}

int launch_conv2d_tc(const float* x, int ctot, int c0, const float* w, const float* bias, float* y, long long B,
                     int cin, int H, int W, int cout, int ks, float leaky, float gain_per_step, int* err,
                     cudaStream_t st) {
    const long long M = B * H * W;
    if (M == 0) return NFB_OK;
    const int T = ks * ks;
    const int groups = (cin + 15) / 16 * T;  // 16-wide k groups: (channel block, tap)
    const int k_chunks = (groups + 3) / 4;
    const int NT = ct_n_tile(cout);
    const int n_tiles = (cout + NT - 1) / NT;
    const size_t bytes = (size_t)k_chunks * n_tiles * NT * 256;
    void* scratch = nullptr;
    NFB_CUDA(cudaMallocAsync(&scratch, bytes, st));  // stream-ordered: freed after the kernel that reads it
    const long long total = (long long)k_chunks * n_tiles * NT * 64;
    const float gain = 1.f + gain_per_step * (float)(3 * 4 * k_chunks);
    conv_pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w, cout, cin, T, NT, n_tiles, k_chunks, gain,
                                                                      static_cast<uint8_t*>(scratch));
    ConvTcParams p{};
    p.x = x; p.y = y; p.bias = bias; p.wstream = static_cast<const uint8_t*>(scratch);
    p.M = M; p.ctot = ctot; p.c0 = c0; p.cin = cin; p.H = H; p.W = W; p.cout = cout; p.ks = ks;
    p.n_tiles = n_tiles; p.k_chunks = k_chunks; p.leaky = leaky; p.err = err;
    int rc = NT == 64 ? launch_conv_tc_t<64>(p, st) : launch_conv_tc_t<128>(p, st);
    const cudaError_t e = cudaGetLastError();
    cudaFreeAsync(scratch, st);
    if (rc) return rc;
    if (e != cudaSuccess) {
        nfb_set_error("conv_tc launch: %s", cudaGetErrorString(e));
        return NFB_ERR_CUDA;
    }
    return NFB_OK;
}

}  // namespace nfb
