// nfb_fused_rqs.cu -- the fused sm_90a kernel of the neural-spline coupling blocks (one block, or a whole stack).
//
// Per 64-row tile, without leaving the SM:
//   [LULinearPermute.inverse  (flows/mixing.py:560-563)]      x  = z[:,perm] (LU)^T + b
//   conditioner  MADE (nets/made.py:296-304) or ResidualNet (nets/resnet.py:92-104)
//   RQ spline    (utils/splines.py:16-219) on every transformed feature
//   [unconditional CDF spline on the identity features (neural_spline/coupling.py:221-253)]
//   log_q += sum_j logabsdet_j (+ LU logabsdet)                 (core.py:98-100)
// z is read once and written once per block; the [B, T*(3K-1)] parameter tensor the reference
// materialises never exists.
//
// Tensor-core numerics: every GEMM runs as a split-fp16 product on wgmma (fp32 accumulation in registers), operands
// scaled by powers of two (nfb_api.cu plan_scales):
//   a*w ~= a_hi*w_hi + a_lo*w_hi + a_hi*w_lo     (conditioner layers; ~2^-22 relative per product)
//   all four terms for the LU linear map that transforms z itself.
// Plain bf16/tf32 fail the rtol 1e-4 log_prob bar (SURVEY 7.2); this is why.
//
// Structure (384 threads, 1 CTA/SM, persistent over (layer, tile) work units of the whole stack):
//   warp 8     weight producer: 1-D bulk TMA (cp.async.bulk) of pre-swizzled fp16 records from the packed weight stream
//              (read from L2) into a 3 x 32 KB ring.  A record is one W_hi tile and its W_lo twin for one K-chunk: the
//              output slices of BOTH consumer warpgroups stacked (rows [0, 8 n8) for warpgroup 0, [8 n8, 16 n8) for 1).
//              Its warpgroup gives its registers to the consumers (setmaxnreg); warps 9-11 exit.
//   warps 0-7  two warpgroups; each issues the wgmma (M = the 64 rows of the tile, K = 16) of its half of every record
//              and runs its epilogues.  A hidden GEMM's output columns are split between them (warpgroup w: 64-column
//              slices [w h, w h + h), h = ceil(H / 128)), so the whole output -- and the conditioner's residual stream,
//              64 x H fp32 -- lives in registers (2 x 32 per thread each) and ONE A-operand buffer suffices: both
//              warpgroups finish the GEMM, then overwrite its input with its output (bias, ReLU, fp16 hi/lo split).  The
//              second GEMM of each residual block accumulates straight onto the residual stream (h += W2 relu(...));
//              the biases are pre-summed by the packer.  The final layer is computed two features (N = 48) per
//              warpgroup at a time and staged through shared memory, so that each thread evaluates one (row, feature)
//              spline; the two warpgroups drift apart by up to the ring depth, so one's splines overlap the other's
//              products.
// Shared memory: A operand 64 KB (hi|lo x K=256), weight ring 96 KB, x/y tile 16 KB (XOR-swizzled, conflict-free
// column access), final-layer staging 2 x 13 KB.
#include <type_traits>

#include "nfb_kernels.h"
#include "nfb_spline.cuh"

namespace nfb {

constexpr int kRows = kFusedTileRows;             // 64
constexpr int kCons = 256;                        // the consumer warpgroups (warps 0-7)
constexpr int kFusedThreads = kCons + 128;        // + the producer warpgroup (warp 8 streams the weights)
// Register budget: the producer warpgroup gives most of its registers to the two consumer warpgroups (setmaxnreg), so
// that the residual-stream halves, the GEMM accumulators and the spline evaluation stay in registers:
// 128 x 24 + 256 x 240 <= 64 K, and per SM sub-partition (3 warps) 2 x 240 x 32 + 24 x 32 <= 16 K.
constexpr int kProducerRegs = 24, kConsumerRegs = 240;
constexpr uint32_t kTileA = 8192;                 // one [64 x 64] fp16 SW128 tile
constexpr uint32_t kSlotBytes = 32768;            // one record: [<= 128 rows x 64 K] hi + lo
constexpr uint32_t kSlots = 3;
constexpr uint32_t kOffW = 8 * kTileA;                      // 65536: after the A operand (hi K-chunks 0..3 | lo 0..3)
constexpr uint32_t kOffX = kOffW + kSlots * kSlotBytes;     // 163840: x/y tile
constexpr int kStgLd = 52;                                  // final-layer staging row stride (floats)
constexpr uint32_t kStgBytes = kRows * kStgLd * 4;
constexpr uint32_t kOffStg = kOffX + kRows * 64 * 4;        // 180224: one staging tile per warpgroup
constexpr uint32_t kOffMisc = kOffStg + 2 * kStgBytes;      // log-det partials [3][64], row exponents [64]
constexpr uint32_t kOffBars = kOffMisc + 4 * kRows * 4;
constexpr uint32_t kNumBars = 10;
constexpr uint32_t kOffUnitQ = kOffBars + kNumBars * 8;     // claimed work units (layer, tile), 4-deep
constexpr uint32_t kFusedSmem = kOffUnitQ + 32;
static_assert(kFusedSmem <= 232448, "shared memory budget");
static_assert(2 * kFusedFeaturesPerChunk * 24 * 64 * 4 <= (int)kSlotBytes, "final-layer record must fit a ring slot");

constexpr int kBarWFull = 0 /* +slot */, kBarWEmpty = 3 /* +slot */, kBarUnit = 6 /* +slot, 4 */;

__device__ __forceinline__ uint32_t xs_index(int r, int c) { return r * 64 + (c ^ (r & 31)); }

// A-operand tile address of element chunk (row r, 16-byte chunk c8 in 0..7) inside a SW128 tile
__device__ __forceinline__ uint32_t a_chunk_off(int r, int c8) {
    return (r >> 3) * 1024 + (r & 7) * 128 + ((c8 ^ (r & 7)) << 4);
}

__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c,
                                             uint32_t d) {
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d)
                 : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void cons_bar_sync() {  // both consumer warpgroups
    asm volatile("bar.sync 1, %0;" ::"n"(kCons) : "memory");
}
__device__ __forceinline__ void wg_bar_sync(int wg) {  // one consumer warpgroup
    asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
}
// mbarrier arrive by one thread of the warpgroup, as a predicated instruction: a branch around it would make ptxas
// serialise the warpgroup's wgmma
__device__ __forceinline__ void mbar_arrive_if(uint32_t bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}"
                 ::"r"(bar), "r"((uint32_t)pred) : "memory");
}

// split 8 consecutive fp32 values (already in the GEMM's scaled units) into fp16 hi / lo chunks and store them at
// the same chunk offset of the two A tiles.  hi + lo reproduces the value to ~2^-23 relative (11 + 11 bits + sign).
__device__ __forceinline__ void split_store8(const float* v, uint32_t t0, uint32_t t1, uint32_t off) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float a = v[2 * i], b = v[2 * i + 1];
        h[i] = pack_f16x2(a, b);
        const float2 hf = unpack_f16x2(h[i]);
        l[i] = pack_f16x2(a - hf.x, b - hf.y);
    }
    st_shared_v4(t0 + off, h[0], h[1], h[2], h[3]);
    st_shared_v4(t1 + off, l[0], l[1], l[2], l[3]);
}
// a value every lane of the warp holds, broadcast from lane 0 so that ptxas can prove it warp-uniform: a wgmma under
// a branch it cannot prove uniform is serialised
template <typename T> __device__ __forceinline__ T uniform(T v) {
    return (T)__shfl_sync(0xffffffffu, (int)v, 0);
}
// 2^e as a float, e in [-126, 127]
__device__ __forceinline__ float pow2i(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }

// the products of one record: acc (+)= A[K-chunk] W^T as W_hi A_hi + W_hi A_lo + W_lo A_hi (+ W_lo A_lo), four K=16
// slabs each, in that order (first: the first product overwrites the accumulator; on = 0: none)
template <int NREG, bool QUAD>
__device__ __forceinline__ void mma_record(float (&acc)[NREG], uint32_t a_hi, uint32_t a_lo, uint32_t w_hi, uint32_t w_lo,
                                           bool first, uint32_t on) {
    const uint64_t ah = wgmma_desc(a_hi), al = wgmma_desc(a_lo), bh = wgmma_desc(w_hi), bl = wgmma_desc(w_lo);
    auto mma = [&](uint64_t a, uint64_t b, uint32_t sd) {
        if constexpr (NREG == 32) wgmma_f16_n64(acc, a, b, sd, on);
        else wgmma_f16_n48(acc, a, b, sd, on);
    };
    uint32_t sd = first ? 0u : 1u;
#pragma unroll
    for (int s = 0; s < 4; ++s) { mma(ah + 2 * s, bh + 2 * s, sd); sd = 1u; }
#pragma unroll
    for (int s = 0; s < 4; ++s) mma(al + 2 * s, bh + 2 * s, 1u);
#pragma unroll
    for (int s = 0; s < 4; ++s) mma(ah + 2 * s, bl + 2 * s, 1u);
    if constexpr (QUAD) {
#pragma unroll
        for (int s = 0; s < 4; ++s) mma(al + 2 * s, bl + 2 * s, 1u);
    }
}

// SAMPLE = false: density direction (Flow.inverse of every layer: x -> z, core.py:70-85).
// SAMPLE = true : sampling direction of coupling-layer stacks (Flow.forward: z -> x, core.py:40-55): the unit is
//   still "LU map, then spline block" -- the packer hands it the INVERSE LU map of the previous layer -- but the
//   unconditional spline runs first and in its inverse branch, the conditioner sees its result, and the
//   conditional spline is inverted (Coupling.inverse, neural_spline/coupling.py:100-128).
template <bool SAMPLE>
__global__ void __launch_bounds__(kFusedThreads, 1) fused_rqs_kernel(const FusedParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t sbase = smem_u32(smem);
    const int warp = uniform((int)(threadIdx.x >> 5)), lane = threadIdx.x & 31;
    float* xs = reinterpret_cast<float*>(smem + kOffX);
    float* ldsum = reinterpret_cast<float*>(smem + kOffMisc);
    int* rowexp = reinterpret_cast<int*>(smem + kOffMisc + 3 * kRows * 4);
    float* rowmax = reinterpret_cast<float*>(smem + kOffStg);  // (the staging tiles are free while a tile is loaded)
    const uint32_t bars = sbase + kOffBars;
    auto bar = [bars](int i) { return bars + 8u * i; };

    if ((sbase & 1023u) != 0) {
        if (threadIdx.x == 0 && p.err) atomicExch(p.err, 900);
        return;
    }
    if (threadIdx.x == 0) {
        for (int i = 0; i < (int)kSlots; ++i) {
            mbar_init(bar(kBarWFull + i), 1);
            mbar_init(bar(kBarWEmpty + i), 2);   // one arrival per consumer warpgroup
        }
        for (int i = 0; i < 4; ++i) mbar_init(bar(kBarUnit + i), 1);
        fence_mbar_init();
    }
    __syncthreads();

    volatile int* unit_q = reinterpret_cast<volatile int*>(smem + kOffUnitQ);   // [4][layer, tile]
    if (warp >= kCons / 32) {
        setmaxnreg_dec<kProducerRegs>();
        if (warp != kCons / 32) return;
        const long long n_tiles = (p.rows + kRows - 1) / kRows;
        // Unit index -> (layer, tile).  Default: layer-major.  Host batch in flight (wave_order): the tiles are split into
        // groups in arrival order and the (layer, group) elements are walked DIAGONALLY -- (l, g) sorted by l + g, then g -- so
        // that the first groups move through the layers while the later groups' rows are still on the PCIe bus; every element
        // still comes after (l - 1, g), so claiming in increasing order stays deadlock-free.  wave_order[2 e] = layer |
        // group << 8, wave_order[2 e + 1] = first unit index of element e; each role walks it with its own cursor (the units
        // a role sees are increasing).  Every unit is a real tile -- an empty unit would let the producer lap the unit queue.
        const long long n_units = n_tiles * p.n_layers;
        auto decode = [&](long long u, int& cursor, int& layer, long long& tile) {
            if (!p.wave_order) {
                layer = (int)(u / n_tiles);
                tile = u - (long long)layer * n_tiles;
                return;
            }
            while (cursor + 1 < p.wave_elems && u >= (long long)__ldg(p.wave_order + 2 * (cursor + 1) + 1)) ++cursor;
            const uint32_t w = __ldg(p.wave_order + 2 * cursor);
            layer = (int)(w & 0xffu);
            tile = (long long)(w >> 8) * p.wave_tpg + (u - (long long)__ldg(p.wave_order + 2 * cursor + 1));
        };
        // Which unit a CTA works on next is decided by its producer warp and handed to the consumers, decoded to (layer,
        // tile), through a 4-deep queue in shared memory.  With a ticket counter (whole-stack launches) units are CLAIMED in increasing order from a global
        // atomic: a unit's dependency (layer - 1, same tile) has a smaller index, so it was claimed earlier by a CTA that is
        // running -- no co-residency of the whole grid is assumed, and faster CTAs take more units.  Without a counter
        // (single-layer launches: no dependencies) the static assignment is used.
        // ------------------------------ weight producer -----------------------------------
        // whole warp walks the table (warp-uniform control flow); one elected lane issues the copy
        uint32_t slot = 0, par = 0;
        int wcur = 0;
        for (uint32_t ui = 0;; ++ui) {
            long long u;
            if (p.ticket) {
                int t = 0;
                if (lane == 0) t = atomicAdd(p.ticket, 1);
                u = (long long)__shfl_sync(0xffffffffu, t, 0);
            } else {
                u = (long long)blockIdx.x + (long long)ui * gridDim.x;
            }
            const bool more = u < n_units;
            int ulayer = -1;
            long long utile = 0;
            if (more) decode(u, wcur, ulayer, utile);
            if (lane == 0) {
                unit_q[2 * (ui & 3u)] = ulayer;
                unit_q[2 * (ui & 3u) + 1] = (int)utile;
                mbar_arrive(bar(kBarUnit + (ui & 3u)));   // (release: the queue entry is visible to whoever passes the wait)
            }
            __syncwarp();
            if (!more) break;
            const FusedLayer& L = p.layers[ulayer];
            const FusedStep* steps = L.steps;  // global (L2-resident)
            const int n_steps = L.n_steps;
            // autoregressive sampling (SAMPLE, ar_passes = D): the LU record is streamed once, the block's D times
            const int lu_steps = L.has_lu ? 1 : 0;
            const int reps = (SAMPLE && L.ar_passes > 0) ? L.ar_passes : 1;
            const int total = n_steps ? lu_steps + reps * (n_steps - lu_steps) : 0;
            const uint32_t lu_bytes = L.has_lu ? 2u * 8192u : 0u;
            int s = 0;
            uint32_t off = 0;
            uint32_t bytes = total ? (uint32_t)__ldg(&steps[0].bytes16) << 4 : 0u;
            for (int i = 0; i < total; ++i) {
                int sn = s + 1;
                uint32_t offn = off + bytes;
                if (sn == n_steps) { sn = lu_steps; offn = lu_bytes; }
                const uint32_t nbytes = i + 1 < total ? (uint32_t)__ldg(&steps[sn].bytes16) << 4 : 0u;
                mbar_wait(bar(kBarWEmpty + slot), par ^ 1, p.err, 100 + slot);
                if (elect_one_sync()) {
                    mbar_expect_tx(bar(kBarWFull + slot), bytes);
                    bulk_g2s(sbase + kOffW + slot * kSlotBytes, L.wstream + off, bytes, bar(kBarWFull + slot));
                }
                __syncwarp();
                s = sn;
                off = offn;
                bytes = nbytes;
                if (++slot == kSlots) { slot = 0; par ^= 1; }
            }
        }
        return;
    }

    // ------------------------------ consumer warpgroups -----------------------------------
    setmaxnreg_inc<kConsumerRegs>();
    const int et = threadIdx.x;                    // 0..255
    const int wg = uniform(et >> 7);               // consumer warpgroup
    const int wl = warp & 3;                       // warp within the warpgroup
    const int ra = 16 * wl + (lane >> 2);          // accumulator rows of this thread: ra, ra + 8
    const int rb = ra + 8;
    const int cq = 2 * (lane & 3);                 // first of its two columns in every 8-column group
    const uint32_t aA = sbase;                     // the A operand
    const uint32_t skip_bit = wg ? kStepSkip1 : kStepSkip0;
    float* stg = reinterpret_cast<float*>(smem + kOffStg + wg * kStgBytes);
    uint32_t slot = 0, wpar = 0;

    for (uint32_t ui = 0;; ++ui) {
        mbar_wait(bar(kBarUnit + (ui & 3u)), (ui >> 2) & 1u, p.err, 600 + (int)(ui & 3u));
        const int layer = uniform(unit_q[2 * (ui & 3u)]);
        const long long tile = uniform(unit_q[2 * (ui & 3u) + 1]);
        if (layer < 0) break;
        const FusedLayer& L = p.layers[layer];
        const int D = L.D, ns = uniform(L.H >> 6), half = (ns + 1) >> 1;
        const int n_steps = uniform(L.n_steps), lu_steps = uniform(L.has_lu ? 1 : 0);
        const int n_hidden = uniform(L.n_hidden), n_pairs = uniform(L.n_chunks >> 1);
        int sidx = 0;
        // The records of one output slice (until the one flagged last): this warpgroup's half of each goes into acc
        // (live: the warpgroup has a slice here; a record's skip bit: its half is all zero).  Every record is waited
        // for and handed back by both warpgroups; a slot is handed back as soon as the products that read it have
        // completed (an empty wgmma group stands in for a skipped half, so the group count stays uniform).
        auto run_slice = [&](auto& acc, bool live, auto quad) {
            int prev = -1;
            for (;;) {
                union { uint2 raw; FusedStep s; } st;
                st.raw = __ldg(reinterpret_cast<const uint2*>(L.steps) + sidx);
                st.raw.x = uniform(st.raw.x);
                st.raw.y = uniform(st.raw.y);
                sidx = sidx + 1 == n_steps ? lu_steps : sidx + 1;
                mbar_wait(bar(kBarWFull + slot), wpar, p.err, 220 + slot);
                const uint32_t w = sbase + kOffW + slot * kSlotBytes + (uint32_t)wg * st.s.n8 * 1024u;
                const uint32_t kc = st.s.kc;
                wgmma_fence();
                mma_record<sizeof(acc) / sizeof(float), decltype(quad)::value>(
                    acc, aA + kc * kTileA, aA + (4 + kc) * kTileA, w, w + ((uint32_t)st.s.bytes16 << 3),
                    (st.s.flags & kStepFirst) != 0, (uint32_t)(live && !(st.s.flags & skip_bit)));
                wgmma_commit();
                wgmma_wait<1>();   // the previous record's products are complete: hand its slot back
                mbar_arrive_if(bar(kBarWEmpty + (prev < 0 ? 0 : prev)), prev >= 0 && (et & 127) == 0);
                prev = (int)slot;
                if (++slot == kSlots) { slot = 0; wpar ^= 1; }
                if (st.s.flags & kStepLast) break;
            }
            wgmma_wait<0>();
            wgmma_hold(acc);
            mbar_arrive_if(bar(kBarWEmpty + prev), (et & 127) == 0);
        };
        using NoQuad = std::integral_constant<bool, false>;

        // layers >= 1 update z in place (z_stride = 0) or, for the training pass, every layer writes its own
        // buffer zout + layer * z_stride so that the backward finds each layer's input
        float* zdst = p.zout + (long long)layer * p.z_stride;
        const float* zsrc = layer == 0 ? p.zin : p.zout + (long long)(layer - 1) * p.z_stride;
        const long long row0 = tile * kRows;
        const int r = et & (kRows - 1);           // row of the per-row work (splines, log-det) of this thread
        const int rq = et >> 6;                   // ... and its quarter of the 256 threads
        const long long grow = row0 + r;
        const bool row_live = grow < p.rows;

        // ---- layer-to-layer dependency: this tile's rows must have left layer-1 (any CTA) ----
        if (layer > 0) {
            if (lane == 0) {  // one lane per warp spins (keeps the warp converged for the .aligned ops below)
                const int* flag = p.progress + tile;
                int seen;
                const long long t0 = clock64();
                do {
                    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(flag) : "memory");
                    if (seen < layer && clock64() - t0 > 4000000000LL) fail_timeout(p.err, 500);
                } while (seen < layer);
            }
            __syncwarp();
            {   // every thread performs its own acquire of the (now set) flag before touching the rows
                int seen;
                asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(seen) : "l"(p.progress + tile) : "memory");
                if (seen < layer) fail_timeout(p.err, 501);
            }
        }
        // ---- host batch still in flight (nfb_api.cu h2d_prepare / h2d_copies): layer-0 tiles wait for their rows ----
        if (layer == 0 && p.in_ready) {
            const int need = (int)min(row0 + kRows, p.rows);
            if (lane == 0) {
                int seen;
                const long long t0 = clock64();
                do {
                    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(seen) : "l"(p.in_ready) : "memory");
                    if (seen < need && clock64() - t0 > 20000000000LL) fail_timeout(p.err, 510);  // ~10 s: no copy
                } while (seen < need);
            }
            __syncwarp();
            {   // every thread acquires the (now sufficient) counter itself before reading the rows
                int seen;
                asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(seen) : "l"(p.in_ready) : "memory");
                if (seen < need) fail_timeout(p.err, 511);
            }
        }
        // this row's running log_q (only this tile's units touch it): fetched now, used at the end of the unit
        float lq_old = 0.f;
        if (rq == 0 && row_live && (layer > 0 || p.accumulate)) lq_old = __ldcg(p.logq + grow);
        // ---- load z tile -> xs (coalesced global, swizzled shared) ----
        if (D == 64) {
            float4 v[kRows * 16 / kCons];
#pragma unroll
            for (int k = 0; k < kRows * 16 / kCons; ++k) {
                const int i4 = et + k * kCons, rr = i4 >> 4;
                const long long gr = row0 + rr;
                v[k] = gr < p.rows ? __ldcg(reinterpret_cast<const float4*>(zsrc + gr * 64) + (i4 & 15))
                                   : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int k = 0; k < kRows * 16 / kCons; ++k) {
                const int i4 = et + k * kCons, rr = i4 >> 4, c0 = (i4 & 15) * 4;
                xs[xs_index(rr, c0)] = v[k].x;
                xs[xs_index(rr, c0 + 1)] = v[k].y;
                xs[xs_index(rr, c0 + 2)] = v[k].z;
                xs[xs_index(rr, c0 + 3)] = v[k].w;
                // max |z| of row rr: its 64 values sit in the 16 consecutive lanes of this half-warp
                float m = fmaxf(fmaxf(fabsf(v[k].x), fabsf(v[k].y)), fmaxf(fabsf(v[k].z), fabsf(v[k].w)));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 8));
                if ((et & 15) == 0) rowmax[rr] = m;
            }
        } else {
            for (int i = et; i < kRows * D; i += kCons) {
                const int rr = i / D, cc = i - rr * D;
                const long long gr = row0 + rr;
                xs[xs_index(rr, cc)] = gr < p.rows ? __ldcg(zsrc + gr * D + cc) : 0.f;
            }
        }
        cons_bar_sync();
        // Row unit u = 2^-e, e = clamp(floor(log2 max|x_row|) + 1, 0, 40): |x| u < 1 for every input of the row, so every
        // fp16 operand of this unit stays inside the static bounds the packer derived (nfb_api.cu plan_scales) whatever
        // the magnitude of the data; u = 1 for ordinary rows (|x| < 1 .. 2).
        auto set_row_exp = [&](float zmax) {
            int e = (int)((__float_as_uint(zmax) >> 23) & 0xffu) - 126;
            rowexp[r] = max(0, min(40, e));
        };
        if (rq == 0) {
            float zmax = 0.f;
            if (D == 64) zmax = rowmax[r];
            else
                for (int c = 0; c < D; ++c) zmax = fmaxf(zmax, fabsf(xs[xs_index(r, c)]));
            set_row_exp(zmax);
        }
        cons_bar_sync();
        auto ru = [&](int row) { return pow2i(-rowexp[row]); };
        auto ruinv = [&](int row) { return pow2i(rowexp[row]); };
        auto get_x = [&](int c) -> float { return xs[xs_index(r, c)]; };
        auto put_y = [&](int c, float y) { xs[xs_index(r, c)] = y; };
        // A[:, 0:64] (K-chunk 0): fp16 hi/lo split of value(row, k) * u_row * sc; thread = (row, quarter of k)
        const int ar = et >> 2, aq = et & 3;
        auto store_a = [&](auto value, float sc_base) {
            const float sc = sc_base * ru(ar);
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = value(aq * 16 + j) * sc;
#pragma unroll
            for (int g = 0; g < 2; ++g) split_store8(v + 8 * g, aA, aA + 4 * kTileA, a_chunk_off(ar, 2 * aq + g));
            fence_proxy_async_smem();
            cons_bar_sync();
        };
        // conditioner input: column in_idx[k] of the (LU-transformed) row
        auto build_a_net = [&]() {
            store_a([&](int k) {
                const int c = L.in_idx[k];
                return c >= 0 ? xs[xs_index(ar, c)] : 0.f;
            }, L.a_sc[1]);
        };
        float ladsum = 0.f;
        // fold_lu (density direction): the packer multiplied the first conditioner matrix into the LU map, so the first
        // hidden GEMM reads the SAME A operand as the LU stage (the split of z)
        const bool folded = uniform(!SAMPLE && L.has_lu && L.fold_lu);
        if (lu_steps) {
            store_a([&](int k) { return k < D ? xs[xs_index(ar, k)] : 0.f; }, L.a_sc[0]);
            float acc[32];
            run_slice(acc, wg == 0, std::integral_constant<bool, true>());   // (no half for warpgroup 1)
            if (wg == 0) {
                // x' = acc + b (this thread: rows ra / rb, two columns of every 8-column group)
                const float ia = L.a_inv[0] * ruinv(ra), ib = L.a_inv[0] * ruinv(rb);
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int c = 8 * (i >> 2) + cq + (i & 1);
                    const int rr = (i & 2) ? rb : ra;
                    if (c < D) xs[xs_index(rr, c)] = fmaf(acc[i], (i & 2) ? ib : ia, __ldg(L.bias_lu + c));
                }
            }
            cons_bar_sync();   // x' of the whole tile is visible to both warpgroups
        }
        auto store_tile = [&]() {  // xs -> global, coalesced
            if (D == 64) {
#pragma unroll
                for (int k = 0; k < kRows * 16 / kCons; ++k) {
                    const int i4 = et + k * kCons, rr = i4 >> 4, c0 = (i4 & 15) * 4;
                    const long long gr = row0 + rr;
                    const float4 v = make_float4(xs[xs_index(rr, c0)], xs[xs_index(rr, c0 + 1)],
                                                 xs[xs_index(rr, c0 + 2)], xs[xs_index(rr, c0 + 3)]);
                    if (gr < p.rows) __stcg(reinterpret_cast<float4*>(zdst + gr * 64) + (i4 & 15), v);
                }
            } else {
                for (int i = et; i < kRows * D; i += kCons) {
                    const int rr = i / D, cc = i - rr * D;
                    const long long gr = row0 + rr;
                    if (gr < p.rows) __stcg(zdst + gr * D + cc, xs[xs_index(rr, cc)]);
                }
            }
        };
        // ---- autoregressive block, sampling direction (flows/affine/autoregressive.py:29-38): D conditioner
        // passes over a running output that starts at zero; every pass inverts the spline on the SAME input S
        // (this tile after the LU stage) with parameters computed from the current output; after pass j the
        // first j features are exact.  S is parked in this tile's rows of `zout` (L2) and read back per element,
        // the running output lives in xs, and nothing else leaves the SM between passes.
        const bool arsamp = uniform(SAMPLE && L.ar_passes > 0);
        const int reps = uniform(arsamp ? L.ar_passes : 1);
        if (arsamp) {
            store_tile();
            if (rq == 0) {
                float zmax = L.tail;  // |output| <= max(|S|, tail): bound of every pass's conditioner input
                for (int c = 0; c < D; ++c) zmax = fmaxf(zmax, fabsf(xs[xs_index(r, c)]));
                set_row_exp(zmax);
            }
            cons_bar_sync();  // every row is scanned; S is in L2 for every thread of the CTA
            for (int i = et; i < kRows * 64; i += kCons) xs[i] = 0.f;
            cons_bar_sync();
        }
        for (int rep = 0; rep < reps; ++rep) {
            if (rep > 0) {
                ladsum = 0.f;     // the log-det of the last pass is the layer's (autoregressive.py:36-38)
                cons_bar_sync();  // the previous pass's outputs (every thread's) are in xs
            }
            // ---- unconditional spline on the identity features (coupled layer only).
            // density: the conditioner input is taken from the RAW values first (Coupling.forward,
            //   neural_spline/coupling.py:80-92) and the spline then runs; sampling: the inverse spline comes first and
            //   the conditioner sees its output (:100-128).
            auto uncond = [&]() {
                for (int i = rq; i < L.n_id; i += kCons / kRows) {
                    const int c = L.id_idx[i];
                    const float* tb = L.uncond + i * 23;
                    auto acc = [tb](int k) { return __ldg(tb + k); };
                    float y, l;
                    rqs_eval<8, SAMPLE>(get_x(c), acc, L.tail, 1.0f, y, l);
                    put_y(c, y);
                    ladsum += l;
                }
            };
            if (SAMPLE && L.n_id > 0) {
                uncond();
                cons_bar_sync();  // build_a reads this row's columns written by the other threads
            }
            if (!folded) build_a_net();   // (ends with a barrier: every thread has read its raw identity columns)
            if (!SAMPLE && L.n_id > 0) uncond();

            // ---- hidden layers: warpgroup wg owns the 64-column slices [wg half, wg half + half) of every output ----
            float hres[2][32];   // its part of the residual stream h
            for (int ph = 0; ph < n_hidden; ++ph) {
                const bool t_phase = (ph & 1) != 0;   // first GEMM of a residual block: its own accumulator
                const bool relu = ph + 1 < n_hidden;
                float tacc[2][32];
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    if (q < half) {
                        const bool live = wg * half + q < ns;
                        if (t_phase) run_slice(tacc[q], live, NoQuad());
                        else run_slice(hres[q], live, NoQuad());
                    }
                }
                cons_bar_sync();   // every product of this GEMM has read the A operand: overwrite it with the output
                const float inv_a = L.a_inv[1 + ph] * ruinv(ra), inv_b = L.a_inv[1 + ph] * ruinv(rb);
                const float sc_a = L.a_sc[2 + ph] * ru(ra), sc_b = L.a_sc[2 + ph] * ru(rb);
                // output slice j: bias, ReLU, scale to the next GEMM's units, fp16 hi/lo -> A K-chunk j
                auto epilogue = [&](const float (&acc)[32], int j) {
                    const float* bias = L.bias_h + ph * 256 + 64 * j;
#pragma unroll
                    for (int g = 0; g < 8; ++g) {
                        const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + 8 * g + cq));
#pragma unroll
                        for (int hb = 0; hb < 2; ++hb) {
                            const int rr = hb ? rb : ra;
                            float v0 = fmaf(acc[4 * g + 2 * hb], hb ? inv_b : inv_a, b2.x);
                            float v1 = fmaf(acc[4 * g + 2 * hb + 1], hb ? inv_b : inv_a, b2.y);
                            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                            v0 *= hb ? sc_b : sc_a;
                            v1 *= hb ? sc_b : sc_a;
                            const uint32_t hi = pack_f16x2(v0, v1);
                            const float2 hf = unpack_f16x2(hi);
                            const uint32_t off = (rr >> 3) * 1024 + (rr & 7) * 128 + ((g ^ (rr & 7)) << 4) + cq * 2;
                            st_shared_b32(aA + j * kTileA + off, hi);
                            st_shared_b32(aA + (4 + j) * kTileA + off, pack_f16x2(v0 - hf.x, v1 - hf.y));
                        }
                    }
                };
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int j = wg * half + q;   // output slice = A K-chunk j of the next GEMM
                    if (q < half && j < ns) {
                        if (t_phase) epilogue(tacc[q], j);
                        else epilogue(hres[q], j);
                    }
                }
                fence_proxy_async_smem();
                cons_bar_sync();   // the next GEMM's A operand is complete
            }

            // ---- final layer: record c = chunks 2c (warpgroup 0) and 2c + 1 (warpgroup 1), kFusedFeaturesPerChunk
            //      features (x 24 columns) each -> staging -> one spline per thread ----
            const float inv_f = L.a_inv[1 + n_hidden] * ruinv(r);
            const int f = (et >> 6) & 1;   // feature of the warpgroup's chunk this thread evaluates (for row r)
            for (int ci = 0; ci < n_pairs; ++ci) {
                float acc[kFusedFeaturesPerChunk * 12];
                run_slice(acc, true, NoQuad());
#pragma unroll
                for (int i = 0; i < kFusedFeaturesPerChunk * 12; i += 2) {
                    const int c = 8 * (i >> 2) + cq;
                    *reinterpret_cast<float2*>(stg + ((i & 2) ? rb : ra) * kStgLd + c) = make_float2(acc[i], acc[i + 1]);
                }
                wg_bar_sync(wg);
                const int t = (2 * ci + wg) * L.F + f;
                if (t < L.T) {
                    // the packer folded log2(e) (and the layer's 1/sqrt(H)) into the w/h columns and biases
                    const float4* sp = reinterpret_cast<const float4*>(stg + r * kStgLd + 24 * f);
                    const float4* bp = reinterpret_cast<const float4*>(L.bias_f + t * 24);
                    float pv[24];
#pragma unroll
                    for (int q = 0; q < 6; ++q) {
                        const float4 s4 = sp[q], b4 = __ldg(bp + q);
                        pv[4 * q] = fmaf(s4.x, inv_f, b4.x);
                        pv[4 * q + 1] = fmaf(s4.y, inv_f, b4.y);
                        pv[4 * q + 2] = fmaf(s4.z, inv_f, b4.z);
                        pv[4 * q + 3] = fmaf(s4.w, inv_f, b4.w);
                    }
                    float lw[8], lh[8], dd[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) { lw[q] = pv[q]; lh[q] = pv[8 + q]; dd[q] = pv[16 + q]; }
                    const int col = L.tr_idx[t];
                    float y, l;
                    float xin = get_x(col);
                    if (arsamp) xin = row_live ? __ldcg(zdst + grow * D + col) : 0.f;
                    rqs_core<8, SAMPLE>(xin, lw, lh, [&dd](int k) { return dd[k]; }, L.tail, y, l);
                    put_y(col, y);
                    ladsum += l;
                }
                wg_bar_sync(wg);   // the staging tile is free again
            }
            cons_bar_sync();   // (AR sampling: every output of this pass is in xs before the next pass reads it)
        }  // passes
        // ---- log-det reduction over the four threads of each row, then store ----
        if (rq > 0) ldsum[(rq - 1) * kRows + r] = ladsum;
        cons_bar_sync();
        if (rq == 0 && row_live) {
            const float tot = ladsum + ldsum[r] + ldsum[kRows + r] + ldsum[2 * kRows + r] +
                              (L.lu_logdet ? __ldg(L.lu_logdet) : 0.f);
            __stcg(p.logq + grow, tot + lq_old);
        }
        store_tile();
        // publish this tile: each thread makes ITS OWN global stores visible device-wide, then the barrier,
        // then one thread releases the flag (a fence by thread 0 alone would not cover stores that other
        // warps still have in flight to L2)
        if (p.progress) __threadfence();
        cons_bar_sync();
        if (p.progress && et == 0) {
            __threadfence();
            asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p.progress + tile), "r"(layer + 1) : "memory");
        }
    }
}

int launch_fused_rqs(const FusedParams& p, int sm_count, int sample, cudaStream_t st) {
    static PerDevice per_dev;  // the opt-in shared-memory size is a per-device function attribute
    const int dev_sms = per_dev.ensure([] {
        cudaError_t e = cudaFuncSetAttribute(fused_rqs_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kFusedSmem);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(fused_rqs_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFusedSmem);
        return e;
    });
    if (dev_sms < 0) return NFB_ERR_CUDA;
    if (sm_count <= 0 || sm_count > dev_sms) sm_count = dev_sms;  // co-residency bound of the CURRENT device
    NFB_CHECK(p.n_layers >= 1 && (p.n_layers == 1 || p.progress), NFB_ERR_ARG, "fused rqs: bad layer list");
    const long long n_tiles = (p.rows + kRows - 1) / kRows;
    if (n_tiles == 0) return NFB_OK;
    const long long n_units = n_tiles * p.n_layers;
    // every CTA must be resident (units wait on flags published by other CTAs): grid <= #SMs, 1 CTA/SM
    const unsigned grid = (unsigned)(n_units < sm_count ? n_units : sm_count);
    if (sample) fused_rqs_kernel<true><<<grid, kFusedThreads, kFusedSmem, st>>>(p);
    else fused_rqs_kernel<false><<<grid, kFusedThreads, kFusedSmem, st>>>(p);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// -----------------------------------------------------------------------------------------
// packing: fp32 effective matrix [n_pad x k_pad] -> stream of swizzled bf16 split records
// record order: for row-block rb: for kc: for split s: [rows_per_rec x 64] tile
// -----------------------------------------------------------------------------------------
// stage 1: E[i,j] = scale[i] * W[src_row[i], src_col[j]] * (mask ? mask[...] : 1), zero if index < 0
__global__ void build_effective_kernel(const float* __restrict__ W, const float* __restrict__ M,
                                       int src_cols, const int* __restrict__ src_row,
                                       const int* __restrict__ src_col,
                                       const float* __restrict__ row_scale, float* __restrict__ E,
                                       int n_pad, int k_pad, float gain) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_pad * k_pad) return;
    const int i = idx / k_pad, j = idx - i * k_pad;
    const int sr = src_row[i], sc = src_col[j];
    float v = 0.f;
    if (sr >= 0 && sc >= 0) {
        const long long o = (long long)sr * src_cols + sc;
        v = W[o];
        if (M) v *= M[o];
        if (row_scale) v *= row_scale[i];
        v *= gain;
    }
    E[idx] = v;
}
// stage 2
__global__ void swizzle_split_kernel(const float* __restrict__ E, int n_pad, int k_pad,
                                     int rows_per_rec, int nsplit, float scale, uint8_t* __restrict__ out) {
    const int kcs = k_pad / 64;
    const long long total = (long long)n_pad * k_pad;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int i = (int)(idx / k_pad), j = (int)(idx - (long long)i * k_pad);
    const int rb = i / rows_per_rec, rr = i - rb * rows_per_rec;
    const int kc = j >> 6, kk = j & 63;
    const float v = E[idx] * scale;
    const size_t rec_bytes = (size_t)rows_per_rec * 128;
    const size_t in_rec = (size_t)(rr >> 3) * 1024 + (rr & 7) * 128 + (((kk >> 3) ^ (rr & 7)) << 4) +
                          (kk & 7) * 2;
    float rem = v;
    for (int s = 0; s < nsplit; ++s) {
        const __half h = __float2half_rn(rem);
        rem -= __half2float(h);
        const size_t rec = ((size_t)rb * kcs + kc) * nsplit + s;
        *reinterpret_cast<__half*>(out + rec * rec_bytes + in_rec) = h;
    }
}

// all records of one GEMM in ONE launch: blockIdx.y = record (table entry), blockIdx.x = 256-element slice of it
__global__ void pack_records_kernel(const float* __restrict__ E, int k_pad, const PackRec* __restrict__ recs, float scale,
                                    uint8_t* __restrict__ base) {
    const PackRec r = recs[blockIdx.y];
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= r.nrows * 64) return;
    const int rr = idx >> 6, kk = idx & 63;
    const float v = E[(size_t)(r.row0 + rr) * k_pad + r.kc * 64 + kk] * scale;
    const size_t off = (size_t)(rr >> 3) * 1024 + (rr & 7) * 128 + (((kk >> 3) ^ (rr & 7)) << 4) + (kk & 7) * 2;
    const __half h = __float2half_rn(v);
    *reinterpret_cast<__half*>(base + r.off_hi + off) = h;
    *reinterpret_cast<__half*>(base + r.off_lo + off) = __float2half_rn(v - __half2float(h));
}
int launch_pack_records(const float* E, int k_pad, const PackRec* recs_dev, int n_recs, int max_rows, float scale,
                        uint8_t* base, cudaStream_t st) {
    if (n_recs == 0) return NFB_OK;
    NFB_CHECK(max_rows > 0 && max_rows % 8 == 0, NFB_ERR_ARG, "pack_records: bad row count %d", max_rows);
    const dim3 grid((unsigned)((max_rows * 64 + 255) / 256), (unsigned)n_recs);
    pack_records_kernel<<<grid, 256, 0, st>>>(E, k_pad, recs_dev, scale, base);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
// LU fold: G[i, c] = gain * sum_k E0[i, k] Elu[in_idx[k], c],  delta[i] = sum_k E0[i, k] blu[in_idx[k]]
// (E0: [H x 64] first conditioner matrix in sorted hidden order, column k <-> conditioner input k = x'[in_idx[k]];
//  Elu: [64 x 64] with x' = Elu z + blu).  fp64 accumulation, one block per row i.
__global__ void fold_lu_kernel(const float* __restrict__ E0, const float* __restrict__ Elu, const float* __restrict__ blu,
                               const int* __restrict__ in_idx, int d, float gain, float* __restrict__ G,
                               float* __restrict__ delta) {
    const int i = blockIdx.x, c = threadIdx.x;
    double acc = 0.0;
    for (int k = 0; k < 64; ++k) {
        const int src = in_idx[k];
        if (src < 0 || src >= d) continue;
        const double w = (double)E0[(size_t)i * 64 + k];
        acc += w * (c < 64 ? (double)Elu[(size_t)src * 64 + c] : (double)blu[src]);
    }
    if (c < 64) G[(size_t)i * 64 + c] = (float)(acc * (double)gain);
    else delta[i] = (float)acc;
}
int launch_fold_lu(const float* E0, const float* Elu, const float* blu, const int* in_idx, int H, int d, float gain,
                   float* G, float* delta, cudaStream_t st) {
    fold_lu_kernel<<<H, 65, 0, st>>>(E0, Elu, blu, in_idx, d, gain, G, delta);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// Norms of an effective matrix E [n x k] (row-major): out[0] = max_i sum_j |E_ij| (infinity norm),
// out[1] = max_i max(sum_j E_ij^+, sum_j E_ij^-) (the tighter bound for non-negative inputs, i.e. post-ReLU),
// out[2] = max |E_ij|.  `out` must be zero-initialised; values are >= 0 so integer atomicMax orders them.
__global__ void matrix_norms_kernel(const float* __restrict__ E, int n, int k, float* __restrict__ out) {
    const int row = blockIdx.x;
    float sp = 0.f, sn = 0.f, mx = 0.f;
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        const float v = E[(size_t)row * k + j];
        sp += fmaxf(v, 0.f);
        sn += fmaxf(-v, 0.f);
        mx = fmaxf(mx, fabsf(v));
    }
    __shared__ float s[3][4];
    sp = warp_sum(sp);
    sn = warp_sum(sn);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s[0][w] = sp; s[1][w] = sn; s[2][w] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float p = 0.f, q = 0.f, m = 0.f;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { p += s[0][i]; q += s[1][i]; m = fmaxf(m, s[2][i]); }
        atomicMax(reinterpret_cast<int*>(out), __float_as_int(p + q));
        atomicMax(reinterpret_cast<int*>(out + 1), __float_as_int(fmaxf(p, q)));
        atomicMax(reinterpret_cast<int*>(out + 2), __float_as_int(m));
    }
    (void)n;
}
int launch_matrix_norms(const float* E, int n, int k, float* out3, cudaStream_t st) {
    NFB_CUDA(cudaMemsetAsync(out3, 0, 3 * sizeof(float), st));
    matrix_norms_kernel<<<n, 128, 0, st>>>(E, n, k, out3);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_build_effective(const float* W, const float* M, int src_cols, const int* src_row,
                           const int* src_col, const float* row_scale, float* E, int n_pad,
                           int k_pad, float gain, cudaStream_t st) {
    const int n = n_pad * k_pad;
    build_effective_kernel<<<(n + 255) / 256, 256, 0, st>>>(W, M, src_cols, src_row, src_col,
                                                            row_scale, E, n_pad, k_pad, gain);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
int launch_swizzle_split(const float* E, int n_pad, int k_pad, int rows_per_rec, int nsplit, float scale,
                         uint8_t* out, cudaStream_t st) {
    NFB_CHECK(n_pad % rows_per_rec == 0 && k_pad % 64 == 0 && rows_per_rec % 8 == 0, NFB_ERR_ARG,
              "swizzle_split: bad shape %d x %d / %d", n_pad, k_pad, rows_per_rec);
    const long long n = (long long)n_pad * k_pad;
    swizzle_split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(E, n_pad, k_pad, rows_per_rec,
                                                                      nsplit, scale, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
