// nfb_conv_wgrad.cu -- weight (and bias) gradient of the stride-1 "same" convolution of nfb_conv_tc.cu on the sm_90a
// tensor core (wgmma), the hot path of the Glow training pass:
//
//   dW[n, c, kh, kw] (+)= sum_{b,h,w} gY[b, n, h, w] x[b, c0+c, h+kh-p, w+kw-p]         db[n] (+)= sum_{b,h,w} gY[b, n, h, w]
//
// As a GEMM: rows n (cout), columns j = c*T + tap (T = k*k, dW's natural layout), reduction over the M = B*H*W pixels.
// In NCHW the pixel axis is contiguous for both operands, so both are gathered K-major: gY plainly, the im2col side
// with the shifted, zero-padded addressing of conv_tc_kernel.  The larger of (cout, cin*T) is the 128-row A operand,
// the other the 64-row B operand.
//
// Numerics: split-bf16 (a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo) with fp32 accumulation, like gemm_tc_kernel.  The
// tensor core truncates each K=16 accumulate step (kAccStepGain ~ 2.4e-8 relative per step); instead of compensating,
// every accumulator runs over one pixel split of at most kMaxChunks * 64 pixels (32 * 64 = 2048: 32 chunks x 3 products
// x 4 steps = 384 truncating steps, ~1e-5 relative), and the splits are summed in fp64 by a second, fixed-order kernel
// (deterministic, no atomics).
//
// Structure (256 threads = two warpgroups, persistent over (A tile, B tile, pixel split) units): each thread gathers
// 8 consecutive pixels of 4 A rows and 2 B rows per 64-pixel chunk (consecutive threads: consecutive pixels -> coalesced),
// splits them to bf16 hi/lo into the SWIZZLE_128B tiles of a two-stage ring while the previous chunk is on the tensor core;
// warpgroup w multiplies A rows [64 w, 64 w + 64).  Each unit writes its fp32 partial [cout, cin*T] tile to a workspace.
#include "nfb_kernels.h"

namespace nfb {

namespace {
constexpr int kWgThreads = 256;
constexpr uint32_t kWgTileA = 16384;   // [128 x 64] bf16
constexpr uint32_t kWgTileB = 8192;    // [64 x 64] bf16
constexpr uint32_t kWgStage = 2 * kWgTileA + 2 * kWgTileB;
constexpr int kMaxChunks = 32;

__device__ __forceinline__ uint32_t wg_off(int r, int c8) {
    return (r >> 3) * 1024 + (r & 7) * 128 + ((c8 ^ (r & 7)) << 4);
}
__device__ __forceinline__ void wg_st_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void wg_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kWgThreads) : "memory"); }
}  // namespace

struct ConvWgradParams {
    const float* x; const float* gy; float* ws;
    long long M, m_chunks;
    int ctot, c0, cin, H, W, cout, ks, ncol;   // ncol = cin * ks * ks
    int a_is_x;                                // A rows are im2col columns (else gY channels)
    int a_tiles, b_tiles, splits, cps;         // cps = chunks per split
};

__global__ void __launch_bounds__(kWgThreads, 2) conv_wgrad_tc_kernel(const ConvWgradParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int bt = threadIdx.x, wg = bt >> 7, warp = (bt >> 5) & 3, lane = bt & 31;
    const int HW = p.H * p.W, pad = p.ks >> 1, T = p.ks * p.ks;
    const long long n_units = (long long)p.a_tiles * p.b_tiles * p.splits;
    const int c8 = bt & 7, row0 = bt >> 3;   // this thread: pixel group c8 of rows row0 + 32 i

    struct Pos { long long u; int at, btile, s, kc, nkc; };
    auto unit_pos = [&](long long u) {
        Pos q;
        q.u = u; q.kc = 0;
        q.at = (int)(u % p.a_tiles);
        const long long rest = u / p.a_tiles;
        q.btile = (int)(rest % p.b_tiles);
        q.s = (int)(rest / p.b_tiles);
        const long long left = p.m_chunks - (long long)q.s * p.cps;
        q.nkc = (int)(left < p.cps ? left : p.cps);
        return q;
    };
    // row value at pixel m: gY channel n or im2col column j
    auto load = [&](bool is_x, int row, long long bi, int pix, int h, int w, bool live) -> float {
        if (!live) return 0.f;
        if (!is_x) return row < p.cout ? __ldg(p.gy + (bi * p.cout + row) * HW + pix) : 0.f;
        if (row >= p.ncol) return 0.f;
        const int c = row / T, tap = row - c * T, kh = tap / p.ks, kw = tap - kh * p.ks;
        const int hh = h + kh - pad, ww = w + kw - pad;
        if (hh < 0 || hh >= p.H || ww < 0 || ww >= p.W) return 0.f;
        return __ldg(p.x + ((bi * p.ctot + p.c0 + c) * p.H + hh) * p.W + ww);
    };
    float va[4][8], vb[2][8];
    auto gather = [&](const Pos& q) {
        const long long mbase = ((long long)q.s * p.cps + q.kc) * 64 + 8 * c8;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const long long m = mbase + e;
            const bool live = m < p.M;
            const long long bi = live ? m / HW : 0;
            const int pix = live ? (int)(m - bi * HW) : 0;
            const int h = pix / p.W, w = pix - h * p.W;
#pragma unroll
            for (int i = 0; i < 4; ++i) va[i][e] = load(p.a_is_x, q.at * 128 + row0 + 32 * i, bi, pix, h, w, live);
#pragma unroll
            for (int i = 0; i < 2; ++i) vb[i][e] = load(!p.a_is_x, q.btile * 64 + row0 + 32 * i, bi, pix, h, w, live);
        }
    };
    auto split_store = [&](uint32_t hi_base, uint32_t lo_base, int r, const float (&v)[8]) {
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float a = v[2 * i], b = v[2 * i + 1];
            hi[i] = pack_bf16x2(a, b);
            lo[i] = pack_bf16x2(a - __uint_as_float(hi[i] << 16), b - __uint_as_float(hi[i] & 0xffff0000u));
        }
        const uint32_t off = wg_off(r, c8);
        wg_st_v4(hi_base + off, hi[0], hi[1], hi[2], hi[3]);
        wg_st_v4(lo_base + off, lo[0], lo[1], lo[2], lo[3]);
    };
    auto emit = [&](int s) {
        const uint32_t sa = sbase + s * kWgStage;
#pragma unroll
        for (int i = 0; i < 4; ++i) split_store(sa, sa + kWgTileA, row0 + 32 * i, va[i]);
#pragma unroll
        for (int i = 0; i < 2; ++i) split_store(sa + 2 * kWgTileA, sa + 2 * kWgTileA + kWgTileB, row0 + 32 * i, vb[i]);
        fence_proxy_async_smem();
    };
    auto mma_chunk = [&](float (&acc)[32], int s, bool first) {
        const uint32_t sa = sbase + s * kWgStage;
        const uint64_t ah = wgmma_desc(sa + wg * 8192u), al = wgmma_desc(sa + kWgTileA + wg * 8192u);
        const uint64_t bh = wgmma_desc(sa + 2 * kWgTileA), bl = wgmma_desc(sa + 2 * kWgTileA + kWgTileB);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, ah + 2 * j, bh + 2 * j, (first && j == 0) ? 0u : 1u);
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, al + 2 * j, bh + 2 * j, 1u);
#pragma unroll
        for (int j = 0; j < 4; ++j) wgmma_bf16_n64(acc, ah + 2 * j, bl + 2 * j, 1u);
        wgmma_commit();
    };
    auto epilogue = [&](const Pos& q, const float (&acc)[32]) {
        float* out = p.ws + (long long)q.s * p.cout * p.ncol;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int ar = q.at * 128 + 64 * wg + 16 * warp + (lane >> 2) + ((i & 2) ? 8 : 0);
            const int br = q.btile * 64 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
            const int n = p.a_is_x ? br : ar, j = p.a_is_x ? ar : br;
            if (n < p.cout && j < p.ncol) out[(long long)n * p.ncol + j] = acc[i];
        }
    };

    if ((long long)blockIdx.x >= n_units) return;
    float acc[32];
    Pos cur = unit_pos(blockIdx.x);
    gather(cur);
    emit(0);
    wg_bar_sync();
    for (int s = 0;; s ^= 1) {
        Pos nxt = cur;
        if (++nxt.kc == cur.nkc) nxt = unit_pos(cur.u + gridDim.x);
        const bool has_next = nxt.u < n_units;
        if (has_next) gather(nxt);   // loads in flight during this chunk's MMAs
        mma_chunk(acc, s, cur.kc == 0);
        if (has_next) emit(s ^ 1);   // stage s ^ 1 was read by the previous chunk, which has completed
        wgmma_wait<0>();
        wgmma_hold(acc);
        wg_bar_sync();               // both warpgroups are done with stage s, and stage s ^ 1 holds the next chunk
        if (cur.kc == cur.nkc - 1) epilogue(cur, acc);
        if (!has_next) break;
        cur = nxt;
    }
}

// dW (+)= sum over the pixel splits, in fp64 and a fixed order
__global__ void wgrad_reduce_kernel(const float* __restrict__ ws, float* __restrict__ gw, long long n, int splits,
                                    int accumulate) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = 0.0;
    for (int k = 0; k < splits; ++k) s += ws[(long long)k * n + i];
    gw[i] = accumulate ? (float)((double)gw[i] + s) : (float)s;
}

// db[n] (+)= sum_{b, pix} gY[b, n, pix]: one block per channel, fp64 partial sums, fixed-order block reduction
__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ gy, float* __restrict__ gb, long long B,
                                                        int cout, int HW, int accumulate) {
    const int n = blockIdx.x;
    double s = 0.0;
    for (long long b = 0; b < B; ++b) {
        const float* src = gy + (b * cout + n) * HW;
        for (int i = threadIdx.x; i < HW; i += 256) s += src[i];
    }
    __shared__ double red[256];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) gb[n] = accumulate ? (float)((double)gb[n] + red[0]) : (float)red[0];
}

int launch_conv2d_wgrad(const float* x, int ctot, int c0, const float* gy, float* gw, float* gb, long long B, int cin,
                        int H, int W, int cout, int ks, int accumulate, int max_chunks_per_split, cudaStream_t st) {
    NFB_CHECK(ks == 1 || ks == 3 || ks == 5, NFB_ERR_UNSUPPORTED, "conv2d_wgrad: kernel size %d", ks);
    NFB_CHECK(c0 >= 0 && cin >= 1 && c0 + cin <= ctot && cout >= 1, NFB_ERR_ARG, "conv2d_wgrad: channel slice out of range");
    const long long M = B * H * W;
    const int ncol = cin * ks * ks;
    const long long nw = (long long)cout * ncol;
    if (M == 0) {
        if (!accumulate) {
            if (gw) NFB_CUDA(cudaMemsetAsync(gw, 0, (size_t)nw * sizeof(float), st));
            if (gb) NFB_CUDA(cudaMemsetAsync(gb, 0, (size_t)cout * sizeof(float), st));
        }
        return NFB_OK;
    }
    if (gb) {
        bias_grad_kernel<<<(unsigned)cout, 256, 0, st>>>(gy, gb, B, cout, H * W, accumulate);
        NFB_LAUNCH_CHECK();
    }
    if (!gw) return NFB_OK;
    static PerDevice per_dev;
    constexpr uint32_t smem = 2 * kWgStage;
    const int sm_count = per_dev.ensure([] {
        return cudaFuncSetAttribute(conv_wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    });
    if (sm_count < 0) return NFB_ERR_CUDA;
    ConvWgradParams p{};
    p.x = x; p.gy = gy; p.M = M; p.m_chunks = (M + 63) / 64;
    p.ctot = ctot; p.c0 = c0; p.cin = cin; p.H = H; p.W = W; p.cout = cout; p.ks = ks; p.ncol = ncol;
    p.a_is_x = ncol > cout ? 1 : 0;
    const int arows = p.a_is_x ? ncol : cout, brows = p.a_is_x ? cout : ncol;
    p.a_tiles = (arows + 127) / 128;
    p.b_tiles = (brows + 63) / 64;
    // shorter splits (more units) until every SM has work, never longer than kMaxChunks chunks per accumulator
    int cps = max_chunks_per_split > 0 && max_chunks_per_split < kMaxChunks ? max_chunks_per_split : kMaxChunks;
    auto units = [&](int c) { return (long long)p.a_tiles * p.b_tiles * ((p.m_chunks + c - 1) / c); };
    while (cps > 4 && units(cps) < 2LL * sm_count) cps >>= 1;
    p.cps = cps;
    p.splits = (int)((p.m_chunks + cps - 1) / cps);
    void* ws = nullptr;
    NFB_CUDA(cudaMallocAsync(&ws, (size_t)p.splits * nw * sizeof(float), st));
    p.ws = static_cast<float*>(ws);
    const long long n_units = units(cps);
    const unsigned grid = (unsigned)(n_units < 2LL * sm_count ? n_units : 2LL * sm_count);   // two CTAs per SM
    conv_wgrad_tc_kernel<<<grid, kWgThreads, smem, st>>>(p);
    wgrad_reduce_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, st>>>(p.ws, gw, nw, p.splits, accumulate);
    const cudaError_t e = cudaGetLastError();
    cudaFreeAsync(ws, st);
    if (e != cudaSuccess) {
        nfb_set_error("conv_wgrad launch: %s", cudaGetErrorString(e));
        return NFB_ERR_CUDA;
    }
    return NFB_OK;
}

}  // namespace nfb
