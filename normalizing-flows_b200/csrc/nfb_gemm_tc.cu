// nfb_gemm_tc.cu -- general fp32-in / fp32-out GEMM on the sm_90a tensor core (wgmma), for the TRAINING pass of the
// neural-spline stacks (recompute of the conditioner activations, dgrad, wgrad; SURVEY 8f-1).
//
//   C[M x N] (+)= op_a(A) [M x K] * op_b(B)^T [N x K]           (fp32 row-major operands in global memory)
//
// Each operand is given as a row-major matrix plus a "major" flag that says which of its two dimensions is the
// contiguous one, so that all three products of a Linear layer read the tensors exactly as PyTorch stores them:
//   forward  Y  = X W^T   : A = X  [B x K]   K-major,  B = W  [N x K]   K-major
//   dgrad    gX = gY W    : A = gY [B x N']  K-major,  B = W  [N' x Kin] MN-major (the GEMM's N is W's column)
//   wgrad    dW = gY^T X  : A = gY [B x N']  MN-major, B = X  [B x Kin]  MN-major (reduction over the batch)
// MN-major operands use the canonical SWIZZLE_128B MN-major shared-memory layout (64 MN elements per 128-byte row,
// 8 k-rows per 1024-byte atom; LBO = stride between 64-wide MN blocks, SBO = stride between 8-row k groups) and the
// transpose operands of wgmma; nothing is transposed in memory.
//
// Numerics: split-bf16, fp32 accumulation: a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo (~2^-17 relative per product;
// bf16 keeps fp32's exponent range, so gradients of any magnitude need no scaling).  NFB_GEMM_TERMS=1 selects the
// single-pass bf16 product (measurement only).
//
// Structure (256 threads = two warpgroups, persistent over work units (m tile, n tile, k split)): every thread loads
// fp32 from global (float4 when aligned, guarded scalars otherwise), applies the optional ReLU on load, splits to bf16
// hi/lo and writes 16-byte chunks into the swizzled A and B tiles of a two-stage ring; warpgroup w multiplies rows
// [64 w, 64 w + 64) of the 128-row tile by the whole n tile (wgmma, accumulator in registers) while the next K-chunk
// is loaded and converted.  The epilogue goes through a shared-memory staging tile so that bias / ReLU-mask / residual
// loads and the stores (or red.add) are contiguous.
#include "nfb_kernels.h"

namespace nfb {

namespace {
constexpr int kGtThreads = 256;
constexpr uint32_t kGtTileA = 16384;            // [128 x 64] bf16
constexpr uint32_t kGtSmemMax = 232448;
__device__ __forceinline__ void gt_st_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void gt_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kGtThreads) : "memory"); }
}  // namespace

struct GemmTcParams {
    const float* A; const float* B; float* C;
    long long lda, ldb, ldc;
    long long M; int N; long long K;
    int a_relu, b_relu;      // max(x, 0) applied while loading
    const float* bias;       // [N] or null: added to every row
    const float* mask;       // [M x N] (ld = ldmask) or null: v *= (mask > 0)      (ReLU derivative)
    const float* mulm;       // [M x N] (ld = ldmask) or null: v *= mulm            (MADE mask on a weight gradient)
    long long ldmask;
    const float* resid;      // [M x N] (ld = ldres) or null: v += resid
    long long ldres;
    int relu_out;            // v = max(v, 0) before the store
    int atomic_out;          // red.global.add instead of a store (split-K partials; C must be pre-zeroed)
    int k_splits;            // >= 1
    long long k_per_split;   // multiple of 64
    int terms;               // 3 = split-bf16, 1 = plain bf16
    const uint8_t* b_packed; // optional: B pre-split to bf16 hi | lo tiles in the stage layout, one record per
                             // (n tile, K chunk): streamed by bulk TMA instead of being converted by the builders
    int* err;
};

// NT: n tile (64 or 128); AMN / BMN: the operand's M / N dimension is the contiguous one (element (i, k) at
// base[k * ld + i]); PACKED: B comes pre-packed (b_packed)
template <int NT, int AMN, int BMN, bool PACKED>
__global__ void __launch_bounds__(kGtThreads, 1) gemm_tc_kernel(const GemmTcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int NREG = NT / 2;
    constexpr uint32_t b_tile = (uint32_t)NT * 128u;             // one [NT x 64] bf16 tile
    constexpr uint32_t stage_bytes = 2 * kGtTileA + 2 * b_tile;  // A hi | A lo | B hi | B lo
    constexpr int kStgLd = NT + 4;
    const uint32_t sbase = smem_u32(smem);
    const int bt = threadIdx.x, wg = bt >> 7, warp = (bt >> 5) & 3, lane = bt & 31;
    const uint32_t offBars = 2 * stage_bytes;
    float* stg = reinterpret_cast<float*>(smem + offBars + 64);   // epilogue staging tile [128][kStgLd]
    const uint32_t bars = sbase + offBars;   // [0, 2): B stage full (PACKED)
    if (bt == 0) {
        mbar_init(bars, 1);
        mbar_init(bars + 8, 1);
        fence_mbar_init();
    }
    __syncthreads();

    const long long m_tiles = (p.M + 127) / 128;
    const int n_tiles = (p.N + NT - 1) / NT;
    const long long n_out_tiles = m_tiles * n_tiles;
    // units are K-split-major: the CTAs that run at the same time work on the SAME k range of different output tiles,
    // so an operand slab that several tiles share (the activations of a weight gradient) is re-read from L2, not HBM
    const long long n_units = n_out_tiles * p.k_splits;
    const bool a_al = (p.lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.A) & 15) == 0);
    const bool b_al = (p.ldb % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.B) & 15) == 0);

    // One operand tile = R "rows" of the GEMM's M/N dimension x 64 k, from a row-major fp32 matrix, handled in groups
    // of 8 contiguous source elements (one 16-byte bf16 chunk of the swizzled tile):
    //   K-major : element (i, k) at src[(i0+i)*ld + k0+k]; group g = (row = g>>3, 16-byte chunk c8 = g&7)
    //   MN-major: element (i, k) at src[(k0+k)*ld + i0+i]; group g = (k row = g / (R/8), chunk cm = g % (R/8))
    auto load_group = [&](const float* src, long long ld, int mn, bool al, long long i0, long long i_end, long long k0,
                          long long k_end, int R, int g, float (&v)[8], uint32_t& off) {
        long long row, col, row_end, col_end;
        if (!mn) {
            const int i = g >> 3, c8 = g & 7;
            row = i0 + i; col = k0 + c8 * 8; row_end = i_end; col_end = k_end;
            off = (uint32_t)((i >> 3) * 1024 + (i & 7) * 128 + ((c8 ^ (i & 7)) << 4));
        } else {
            const int per = R >> 3;
            const int kr = g / per, cm = g - kr * per;
            row = k0 + kr; col = i0 + cm * 8; row_end = k_end; col_end = i_end;
            off = (uint32_t)((cm >> 3) * 8192 + (kr >> 3) * 1024 + (kr & 7) * 128 + (((cm & 7) ^ (kr & 7)) << 4));
        }
        if (row < row_end && col + 8 <= col_end && al) {
            const float4* s4 = reinterpret_cast<const float4*>(src + row * ld + col);
            const float4 x0 = __ldg(s4), x1 = __ldg(s4 + 1);
            v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                v[j] = (row < row_end && col + j < col_end) ? __ldg(src + row * ld + col + j) : 0.f;
        }
    };
    auto store_group = [&](const float (&v)[8], int relu, uint32_t t_hi, uint32_t t_lo, uint32_t off) {
        uint32_t hi[4], lo[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float a = v[2 * i], b = v[2 * i + 1];
            if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
            hi[i] = pack_bf16x2(a, b);
            lo[i] = pack_bf16x2(a - __uint_as_float(hi[i] << 16), b - __uint_as_float(hi[i] & 0xffff0000u));
        }
        gt_st_v4(t_hi + off, hi[0], hi[1], hi[2], hi[3]);
        gt_st_v4(t_lo + off, lo[0], lo[1], lo[2], lo[3]);
    };

    struct Pos { long long u, mt, k0, k1; int nt, kc, KC; };
    auto unit_pos = [&](long long u, int kc) {
        Pos q;
        q.u = u; q.kc = kc;
        const int ks = (int)(u / n_out_tiles);
        const long long tile = u % n_out_tiles;
        q.mt = tile / n_tiles;
        q.nt = (int)(tile - q.mt * n_tiles);
        q.k0 = (long long)ks * p.k_per_split;
        q.k1 = q.k0 + p.k_per_split < p.K ? q.k0 + p.k_per_split : p.K;
        q.KC = (int)((q.k1 - q.k0 + 63) / 64);
        return q;
    };
    constexpr int kAG = 1024 / kGtThreads;              // A groups per thread and chunk (4)
    constexpr int kBG = NT * 8 / kGtThreads;            // B groups per thread and chunk (2 or 4)
    float va[kAG][8], vb[kBG][8];
    uint32_t oa[kAG], ob[kBG];
    auto load_chunk = [&](const Pos& q) {
#pragma unroll
        for (int i = 0; i < kAG; ++i)
            load_group(p.A, p.lda, AMN, a_al, q.mt * 128, p.M, q.k0 + (long long)q.kc * 64, q.k1, 128, bt + i * kGtThreads,
                       va[i], oa[i]);
        if (!PACKED) {
#pragma unroll
            for (int i = 0; i < kBG; ++i)
                load_group(p.B, p.ldb, BMN, b_al, (long long)q.nt * NT, p.N, q.k0 + (long long)q.kc * 64, q.k1, NT,
                           bt + i * kGtThreads, vb[i], ob[i]);
        }
    };
    uint32_t full_use[2] = {0, 0};
    auto store_chunk = [&](const Pos& q, int s) {
        const uint32_t sa = sbase + s * stage_bytes;
        if (PACKED && bt == 0) {
            const int kc_total = (int)((p.K + 63) / 64);   // (k_splits == 1 with a packed operand)
            mbar_expect_tx(bars + 8 * s, 2 * b_tile);
            bulk_g2s(sa + 2 * kGtTileA, p.b_packed + ((size_t)q.nt * kc_total + q.kc) * (2 * b_tile), 2 * b_tile, bars + 8 * s);
        }
#pragma unroll
        for (int i = 0; i < kAG; ++i) store_group(va[i], p.a_relu, sa, sa + kGtTileA, oa[i]);
        if (!PACKED) {
#pragma unroll
            for (int i = 0; i < kBG; ++i) store_group(vb[i], p.b_relu, sa + 2 * kGtTileA, sa + 2 * kGtTileA + b_tile, ob[i]);
        }
        fence_proxy_async_smem();
    };

    // wgmma descriptors.  K-major: 8-row groups 1024 B apart, a K=16 step is 32 B further along the row.  MN-major:
    // 64-wide MN blocks 8192 B apart (LBO), 8-row k groups 1024 B apart (SBO), a K=16 step = 2 groups.
    constexpr uint32_t a_lbo = AMN ? 512u : 1u, b_lbo = BMN ? 512u : 1u;
    constexpr uint32_t a_step = AMN ? 128u : 2u, b_step = BMN ? 128u : 2u;   // descriptor address units (16 B)
    // this warpgroup's 64 rows: 8 row groups further (K-major) or the second 64-wide M block (MN-major): 8 KB either way
    const uint32_t a_wg = (uint32_t)wg * 8192u;
    auto mma_chunk = [&](float (&acc)[NREG], int s, bool first) {
        const uint32_t sa = sbase + s * stage_bytes;
        const uint64_t ah = wgmma_desc(sa + a_wg, a_lbo), al = wgmma_desc(sa + kGtTileA + a_wg, a_lbo);
        const uint64_t bh = wgmma_desc(sa + 2 * kGtTileA, b_lbo), bl = wgmma_desc(sa + 2 * kGtTileA + b_tile, b_lbo);
        auto mma = [&](uint64_t a, uint64_t b, uint32_t sd) {
            if constexpr (NT == 64) wgmma_bf16_n64<AMN, BMN>(acc, a, b, sd);
            else wgmma_bf16_n128<AMN, BMN>(acc, a, b, sd);
        };
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) mma(ah + a_step * j, bh + b_step * j, (first && j == 0) ? 0u : 1u);
        if (p.terms == 3) {
#pragma unroll
            for (int j = 0; j < 4; ++j) mma(al + a_step * j, bh + b_step * j, 1u);
#pragma unroll
            for (int j = 0; j < 4; ++j) mma(ah + a_step * j, bl + b_step * j, 1u);
        }
        wgmma_commit();
    };

    const bool vec_ok = (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0) && !p.atomic_out;
    auto epilogue = [&](const Pos& q, const float (&acc)[NREG]) {
        // accumulator register i: row 16 warp + lane / 4 (+ 8), column 8 (i / 4) + 2 (lane % 4) (+ 1)
        const int r0 = 64 * wg + 16 * warp + (lane >> 2);
#pragma unroll
        for (int i = 0; i < NREG; i += 2) {
            const int c = 8 * (i >> 2) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(stg + (r0 + ((i & 2) ? 8 : 0)) * kStgLd + c) = make_float2(acc[i], acc[i + 1]);
        }
        gt_bar_sync();
        const int cq = (bt & 15) * 4;   // this thread's 4 columns inside a 64-column slab
        for (int cb = 0; cb < NT; cb += 64) {
            const int n0 = q.nt * NT + cb + cq;
#pragma unroll 2
            for (int j = 0; j < 8; ++j) {
                const int rr = (bt >> 4) + 16 * j;
                const long long m = q.mt * 128 + rr;
                if (m >= p.M || n0 >= p.N) continue;
                float v[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) v[t] = stg[rr * kStgLd + cb + cq + t];
                const bool full = n0 + 4 <= p.N;
                if (p.bias) {
#pragma unroll
                    for (int t = 0; t < 4; ++t) if (n0 + t < p.N) v[t] += __ldg(p.bias + n0 + t);
                }
                if (p.mask) {
#pragma unroll
                    for (int t = 0; t < 4; ++t)
                        if (n0 + t < p.N) v[t] = __ldg(p.mask + m * p.ldmask + n0 + t) > 0.f ? v[t] : 0.f;
                }
                if (p.mulm) {
#pragma unroll
                    for (int t = 0; t < 4; ++t) if (n0 + t < p.N) v[t] *= __ldg(p.mulm + m * p.ldmask + n0 + t);
                }
                if (p.resid) {
#pragma unroll
                    for (int t = 0; t < 4; ++t) if (n0 + t < p.N) v[t] += __ldg(p.resid + m * p.ldres + n0 + t);
                }
                if (p.relu_out) {
#pragma unroll
                    for (int t = 0; t < 4; ++t) v[t] = fmaxf(v[t], 0.f);
                }
                float* dst = p.C + m * p.ldc + n0;
                if (p.atomic_out) {
#pragma unroll
                    for (int t = 0; t < 4; ++t) if (n0 + t < p.N) atomicAdd(dst + t, v[t]);
                } else if (full && vec_ok) {
                    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                } else {
#pragma unroll
                    for (int t = 0; t < 4; ++t) if (n0 + t < p.N) dst[t] = v[t];
                }
            }
        }
        gt_bar_sync();  // the staging tile is reused by the next unit
    };

    // The CTA walks its K chunks as ONE stream across unit boundaries: while the tensor core multiplies chunk i, the
    // global loads of chunk i + 1 are in flight and then converted into the other stage.
    if ((long long)blockIdx.x >= n_units) return;
    float acc[NREG];
    Pos cur = unit_pos(blockIdx.x, 0);
    load_chunk(cur);
    store_chunk(cur, 0);
    gt_bar_sync();
    for (int s = 0;; s ^= 1) {
        Pos nxt = cur;
        if (++nxt.kc == cur.KC) nxt = unit_pos(cur.u + gridDim.x, 0);
        const bool has_next = nxt.u < n_units;
        if (has_next) load_chunk(nxt);
        if (PACKED) { mbar_wait(bars + 8 * s, full_use[s] & 1u, p.err, 810 + s); ++full_use[s]; }
        mma_chunk(acc, s, cur.kc == 0);
        if (has_next) store_chunk(nxt, s ^ 1);   // (stage s ^ 1 was read by the previous chunk: complete, see below)
        wgmma_wait<0>();
        wgmma_hold(acc);
        gt_bar_sync();   // both warpgroups are done with stage s, and stage s ^ 1 holds the next chunk
        if (cur.kc == cur.KC - 1) epilogue(cur, acc);
        if (!has_next) break;
        cur = nxt;
    }
}

// Pre-pack a B operand (weights: reused by every 128-row tile of the batch) into bf16 hi | lo records in the exact stage
// layout of gemm_tc_kernel, one record per (n tile, K chunk).  Same group addressing as the builders.
__global__ void gemm_pack_b_kernel(const float* __restrict__ B, long long ldb, int b_mn, int N, long long K, int NT,
                                   uint8_t* __restrict__ out) {
    const int kc_total = (int)((K + 63) / 64);
    const int groups = NT * 8;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int n_tiles = (N + NT - 1) / NT;
    if (gid >= (long long)n_tiles * kc_total * groups) return;
    const int g = (int)(gid % groups);
    const long long t = gid / groups;
    const int kc = (int)(t % kc_total), nt = (int)(t / kc_total);
    const long long i0 = (long long)nt * NT, k0 = (long long)kc * 64;
    long long row, col, row_end, col_end;
    uint32_t off;
    if (!b_mn) {
        const int i = g >> 3, c8 = g & 7;
        row = i0 + i; col = k0 + c8 * 8; row_end = N; col_end = K;
        off = (uint32_t)((i >> 3) * 1024 + (i & 7) * 128 + ((c8 ^ (i & 7)) << 4));
    } else {
        const int per = NT >> 3;
        const int kr = g / per, cm = g - kr * per;
        row = k0 + kr; col = i0 + cm * 8; row_end = K; col_end = N;
        off = (uint32_t)((cm >> 3) * 8192 + (kr >> 3) * 1024 + (kr & 7) * 128 + (((cm & 7) ^ (kr & 7)) << 4));
    }
    uint32_t hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float v[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const long long c = col + 2 * i + j;
            v[j] = (row < row_end && c < col_end) ? B[row * ldb + c] : 0.f;
        }
        hi[i] = pack_bf16x2(v[0], v[1]);
        lo[i] = pack_bf16x2(v[0] - __uint_as_float(hi[i] << 16), v[1] - __uint_as_float(hi[i] & 0xffff0000u));
    }
    const uint32_t b_tile = (uint32_t)NT * 128u;
    uint8_t* rec = out + ((size_t)nt * kc_total + kc) * (2 * b_tile);
    *reinterpret_cast<uint4*>(rec + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
    *reinterpret_cast<uint4*>(rec + b_tile + off) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
}

// n tile: 128 columns (one B tile is reused by the whole 128-row A tile) or 64 for narrow products
int gemm_tc_n_tile(long long N, int b_mn) {
    (void)b_mn;
    return N > 64 ? 128 : 64;
}
size_t gemm_tc_packed_b_bytes(long long N, long long K, int b_mn) {
    const int nt = gemm_tc_n_tile(N, b_mn);
    return (size_t)((N + nt - 1) / nt) * (size_t)((K + 63) / 64) * (size_t)nt * 256;
}
int launch_gemm_pack_b(const float* B, long long ldb, int b_mn, long long N, long long K, uint8_t* out, cudaStream_t st) {
    const int nt = gemm_tc_n_tile(N, b_mn);
    const long long total = (N + nt - 1) / nt * ((K + 63) / 64) * (long long)nt * 8;
    if (total == 0) return NFB_OK;
    gemm_pack_b_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(B, ldb, b_mn, (int)N, K, nt, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -------------------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------------------
template <int NT, int AMN, int BMN, bool PACKED>
int launch_gemm_tc_t(const GemmTcParams& p, long long n_units, cudaStream_t st) {
    static PerDevice per_dev;
    constexpr uint32_t stage_bytes = 2 * kGtTileA + 2 * (uint32_t)NT * 128u;
    constexpr uint32_t smem = 2 * stage_bytes + 64 + 128 * (NT + 4) * 4;
    static_assert(smem <= kGtSmemMax, "gemm_tc: shared memory");
    const int sm_count = per_dev.ensure([] {
        return cudaFuncSetAttribute(gemm_tc_kernel<NT, AMN, BMN, PACKED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)smem);
    });
    if (sm_count < 0) return NFB_ERR_CUDA;
    const unsigned grid = (unsigned)(n_units < sm_count ? n_units : sm_count);
    gemm_tc_kernel<NT, AMN, BMN, PACKED><<<grid, kGtThreads, smem, st>>>(p);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
template <int NT, int AMN, int BMN>
int launch_gemm_tc_p(const GemmTcParams& p, long long n_units, cudaStream_t st) {
    return p.b_packed ? launch_gemm_tc_t<NT, AMN, BMN, true>(p, n_units, st) : launch_gemm_tc_t<NT, AMN, BMN, false>(p, n_units, st);
}
template <int NT>
int launch_gemm_tc_n(const GemmTcParams& p, int a_mn, int b_mn, long long n_units, cudaStream_t st) {
    if (!a_mn) return b_mn ? launch_gemm_tc_p<NT, 0, 1>(p, n_units, st) : launch_gemm_tc_p<NT, 0, 0>(p, n_units, st);
    return b_mn ? launch_gemm_tc_p<NT, 1, 1>(p, n_units, st) : launch_gemm_tc_p<NT, 1, 0>(p, n_units, st);
}

int launch_gemm_tc(const GemmTcArgs& a, int* err, cudaStream_t st) {
    static PerDevice per_dev;
    const int sm_count = per_dev.ensure([] { return cudaSuccess; });
    if (sm_count < 0) return NFB_ERR_CUDA;
    NFB_CHECK(a.A && a.B && a.C, NFB_ERR_ARG, "gemm_tc: null operand");
    if (a.M <= 0 || a.N <= 0) return NFB_OK;
    NFB_CHECK(a.K > 0, NFB_ERR_ARG, "gemm_tc: K must be positive");
    static const int terms = [] { const char* e = getenv("NFB_GEMM_TERMS"); return (e && atoi(e) == 1) ? 1 : 3; }();
    GemmTcParams p{};
    p.A = a.A; p.B = a.B; p.C = a.C; p.lda = a.lda; p.ldb = a.ldb; p.ldc = a.ldc;
    p.M = a.M; p.N = (int)a.N; p.K = a.K; p.a_relu = a.a_relu; p.b_relu = a.b_relu;
    p.bias = a.bias; p.mask = a.mask; p.mulm = a.mulm; p.ldmask = a.ldmask; p.resid = a.resid; p.ldres = a.ldres;
    p.relu_out = a.relu_out; p.terms = terms; p.err = err;
    const int nt = gemm_tc_n_tile(a.N, a.b_mn);
    const long long m_tiles = (a.M + 127) / 128;
    const int n_tiles = (int)((a.N + nt - 1) / nt);
    // split K only when there are too few output tiles to fill the machine (weight gradients: K = batch), and only
    // for a linear epilogue (the partial products are added with red.global.add)
    int ks = 1;
    const long long tiles = m_tiles * n_tiles;
    const bool linear_epilogue = !a.bias && !a.mask && !a.resid && !a.relu_out;
    if (tiles < sm_count && a.K >= 2048 && linear_epilogue) {
        ks = (int)((2LL * sm_count) / tiles);  // <= 2 units per CTA: no third, mostly empty wave
        const long long max_ks = (a.K + 511) / 512;  // at least 8 chunks per split
        if (ks > max_ks) ks = (int)max_ks;
        if (ks < 1) ks = 1;
    }
    long long kps = ((a.K + ks - 1) / ks + 63) / 64 * 64;
    ks = (int)((a.K + kps - 1) / kps);
    p.k_splits = ks; p.k_per_split = kps;
    p.b_packed = (ks == 1 && !a.b_relu) ? a.b_packed : nullptr;  // (a split or ReLU-on-load product converts B itself)
    p.atomic_out = (ks > 1 || a.accumulate) ? 1 : 0;
    if (ks > 1) NFB_CHECK(!a.bias && !a.mask && !a.resid && !a.relu_out, NFB_ERR_ARG, "gemm_tc: split-K with a non-linear epilogue");
    if (ks > 1 && !a.accumulate)  // the partial products are added with red.global.add: start from zero
        NFB_CUDA(cudaMemset2DAsync(a.C, (size_t)a.ldc * 4, 0, (size_t)a.N * 4, (size_t)a.M, st));
    const long long n_units = tiles * ks;
    return nt == 64 ? launch_gemm_tc_n<64>(p, a.a_mn, a.b_mn, n_units, st) : launch_gemm_tc_n<128>(p, a.a_mn, a.b_mn, n_units, st);
}

}  // namespace nfb
