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
//              (read from L2) into a 3 x 32 KB ring.  A record is one W_hi tile and its W_lo twin: one half per
//              consumer warpgroup stacked (rows [0, 8 n8) for warpgroup 0, [8 n8, 16 n8) for 1), each with its own
//              K-chunk, or a single half at offset 0 (nfb_fused_plan.h).
//              Its warpgroup gives its registers to the consumers (setmaxnreg); warps 9-11 exit.
//   warps 0-7  two warpgroups; each issues the wgmma (M = the 64 rows of the tile, K = 16) of its half of every record
//              and runs its epilogues.  A hidden GEMM's output columns are split between them (warpgroup w owns up to
//              ceil(H / 128) 64-column slices, FusedLayer::own, chosen by the packer so that the non-zero blocks of the
//              MADE masks split evenly), so the whole output -- and the conditioner's residual stream,
//              64 x H fp32 -- lives in registers (2 x 32 per thread each) and ONE A-operand buffer suffices: both
//              warpgroups finish the GEMM, then overwrite its input with its output (bias, ReLU, fp16 hi/lo split).  The
//              second GEMM of each residual block accumulates straight onto the residual stream (h += W2 relu(...));
//              the biases are pre-summed by the packer.
//              In the final layer the warpgroups take different roles: warpgroup 0 multiplies both halves of every
//              record (two features, N = 48, per half; both halves as one N = 96 product) into two alternating
//              accumulators and stores each pair of chunks, unscaled and with its biases, to two staging tiles in shared
//              memory; warpgroup 1 copies its (row, feature) parameters of both chunks out of the tiles, hands them
//              back before any spline runs and evaluates the two splines per thread as one two-lane chain
//              (rqs_core_lanes, nfb_spline.cuh).  The hand-off is a pair of named barriers
//              ("full" / "free", one side arrives, the other waits), so the products of one pair of chunks run under the
//              splines of the pair before.
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
__device__ __forceinline__ void cons_bar_sync() {  // both consumer warpgroups
    asm volatile("bar.sync 1, %0;" ::"n"(kCons) : "memory");
}
// Final-layer hand-off between the product warpgroup and the spline warpgroup (producer / consumer form of the named
// barriers: one side arrives, the other waits; both count kCons).  The arriving side fences first: bar.arrive by
// itself does not order its thread's earlier shared-memory accesses.
constexpr int kBarStgFull = 2, kBarStgFree = 3;
template <int ID> __device__ __forceinline__ void stg_bar_arrive() {
    __threadfence_block();
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(kCons) : "memory");
}
template <int ID> __device__ __forceinline__ void stg_bar_wait() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(kCons) : "memory");
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

// the products of one record: acc (+)= A[K-chunk] W^T as W_hi A_hi + W_hi A_lo + W_lo A_hi (+ W_lo A_lo), the first
// SLABS K = 16 slabs each, in that order (the slabs after SLABS are all zero).  One straight chain: no wgmma of it has a
// predicate of its own, so ptxas issues them back to back behind one warpgroup.arrive.  Whether a record has products at
// all is decided by one uniform branch around the chain.
// N = 64 (32 registers): a hidden GEMM's slice or the LU map; N = 96 (48): both halves of a final-layer record at once,
// half 0 in registers 0..23 and half 1 in 24..47 (rows [0, 48) and [48, 96) of the record's tiles).
// FIRST: the record opens acc (the packer's kStepFirst), and its first product overwrites acc with an immediate scale-d
// of 0, so acc needs no value before it; every other product accumulates.  Callers issue an opening record as FIRST
// unconditionally, so that to the compiler acc is written before it is read.
struct MmaOps { uint32_t a_hi, a_lo, w_hi, w_lo, on, slabs; };
template <int SLABS, bool QUAD, int NREG, bool FIRST = false>
__device__ __forceinline__ void mma_record(float (&acc)[NREG], const MmaOps& x) {
    static_assert(NREG == 32 || NREG == 48, "N = 64 or 96");
    const uint64_t ah = wgmma_desc(x.a_hi), al = wgmma_desc(x.a_lo), bh = wgmma_desc(x.w_hi), bl = wgmma_desc(x.w_lo);
    auto pass = [&](uint64_t a, uint64_t b, bool opens) {
#pragma unroll
        for (int s = 0; s < SLABS; ++s) {
            if constexpr (NREG == 32) {
                if (FIRST && opens && s == 0) wgmma_f16_n64_zero(acc, a, b);
                else wgmma_f16_n64(acc, a + 2 * s, b + 2 * s, 1u);
            } else {
                if (FIRST && opens && s == 0) wgmma_f16_n96_zero(acc, a, b);
                else wgmma_f16_n96(acc, a + 2 * s, b + 2 * s, 1u);
            }
        }
    };
    pass(ah, bh, true);
    pass(al, bh, false);
    pass(ah, bl, false);
    if constexpr (QUAD) pass(al, bl, false);
}

// Phase clocks (make CLOCKS=1, a separate library; tools/fused_phase_clocks.py): every thread of a role adds the SM
// cycles between two consecutive stamps to the phase the second stamp names, and thread 0 of each consumer warpgroup and
// lane 0 of the producer warp add their sums to g_phase_clocks when the CTA runs out of units.  Without the macro a
// stamp is nothing and the product kernel is unchanged.
enum { kClkClaim,       // unit queue, layer-to-layer flag, rows of a host batch in flight
       kClkLoad,        // z tile -> shared memory, row units, A operand of the first GEMM (and its barriers)
       kClkLu,          // LU stage: ring wait, products, epilogue
       kClkHidRing,     // hidden GEMMs: wait for the record (full barrier)
       kClkHidMma,      // hidden GEMMs: wgmma issue -> complete (wait_group), slot hand-back
       kClkHidEpi,      // hidden GEMMs: epilogues and the barriers around them; unconditional splines
       kClkFinRing,     // final layer: wait for the record
       kClkFinMma,      // final layer: wgmma issue -> complete within a pair, slot hand-back
       kClkFinTail,     // final layer: the wait at a pair boundary that completes the previous pair's products
       kClkFinStage,    // final layer: accumulators <-> staging tiles, hand-off waits
       kClkFinSpline,   // final layer: spline evaluation
       kClkStore,       // log-det reduction, tile store, publish
       kClkProdEmpty,   // producer: wait for an empty slot
       kClkProdOther,   // producer: everything else (claim, step table, issue)
       kClkUnits,       // (a count, not cycles) units this role worked on
       kClkCount };
// the phases a run of records charges its ring waits, its products and its first record's wait to
template <int RING, int MMA, int TAIL> struct WalkClk { static constexpr int ring = RING, mma = MMA, tail = TAIL; };
using LuClk = WalkClk<kClkLu, kClkLu, kClkLu>;
using HidClk = WalkClk<kClkHidRing, kClkHidMma, kClkHidMma>;
using FinClk = WalkClk<kClkFinRing, kClkFinMma, kClkFinTail>;
#ifdef NFB_PHASE_CLOCKS
__device__ unsigned long long g_phase_clocks[3][kClkCount];   // [consumer warpgroup 0, 1, producer][phase]
struct PhaseClock {   // 32-bit sums: one launch is far below 2^32 cycles
    uint32_t last, sum[kClkCount];
    __device__ PhaseClock() {
        last = (uint32_t)clock64();
#pragma unroll
        for (int i = 0; i < kClkCount; ++i) sum[i] = 0;
    }
    template <int P> __device__ __forceinline__ void stamp() {
        const uint32_t t = (uint32_t)clock64();
        sum[P] += t - last;
        last = t;
    }
    __device__ void flush(int role) const {
#pragma unroll
        for (int i = 0; i < kClkCount; ++i) atomicAdd(&g_phase_clocks[role][i], (unsigned long long)sum[i]);
    }
};
#define NFB_CLK_BEGIN() PhaseClock clk
#define NFB_CLK(P) clk.template stamp<P>()
#define NFB_CLK_UNIT() (++clk.sum[kClkUnits])
#define NFB_CLK_END(role, pred) do { if (pred) clk.flush(role); } while (0)
#else
#define NFB_CLK_BEGIN() ((void)0)
#define NFB_CLK(P) ((void)0)
#define NFB_CLK_UNIT() ((void)0)
#define NFB_CLK_END(role, pred) ((void)0)
#endif

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
        NFB_CLK_BEGIN();
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
            NFB_CLK_UNIT();
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
                NFB_CLK(kClkProdOther);
                mbar_wait(bar(kBarWEmpty + slot), par ^ 1, p.err, 100 + slot);
                NFB_CLK(kClkProdEmpty);
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
        NFB_CLK(kClkProdOther);
        NFB_CLK_END(2, lane == 0);
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
    float* stg0 = reinterpret_cast<float*>(smem + kOffStg);   // staging tile of a pair's even chunk; the odd one follows
    uint32_t slot = 0, wpar = 0;
    NFB_CLK_BEGIN();

    for (uint32_t ui = 0;; ++ui) {
        mbar_wait(bar(kBarUnit + (ui & 3u)), (ui >> 2) & 1u, p.err, 600 + (int)(ui & 3u));
        const int layer = uniform(unit_q[2 * (ui & 3u)]);
        const long long tile = uniform(unit_q[2 * (ui & 3u) + 1]);
        if (layer < 0) break;
        NFB_CLK_UNIT();
        const FusedLayer& L = p.layers[layer];
        const int D = L.D;
        auto own = [&](int q) { return uniform((int)L.own[wg][q]); };   // this warpgroup's slices (-1: none)
        const int n_steps = uniform(L.n_steps), lu_steps = uniform(L.has_lu ? 1 : 0);
        const int n_hidden = uniform(L.n_hidden), n_pairs = uniform(L.n_chunks >> 1);
        int sidx = 0;
        // A run of consecutive records, until the one whose products `issue` reports as the last of its accumulator(s).
        // Every record is waited for, and its slot handed back as soon as the products that read it have completed
        // (an empty wgmma group stands in for skipped products, so the group count stays uniform).  A slot's empty
        // barrier expects one arrival per consumer warpgroup: `arrivals` is 1 where both warpgroups walk the records
        // (LU stage, hidden GEMMs) and 2 where one walks them for both (final layer).
        auto hand_back = [&](auto arrivals, int s, bool pred) {
#pragma unroll
            for (int i = 0; i < decltype(arrivals)::value; ++i) mbar_arrive_if(bar(kBarWEmpty + s), pred && (et & 127) == 0);
        };
        // The walker itself leaves the last record's products in flight and its slot in `prev` (-1: none), so that a run
        // can start while the one before still multiplies.  OPEN: the first record is issued as issue(step, true_type)
        // and completes the products in flight before it (its wait_group 1), which hands back `prev` and then runs
        // `retire` -- the previous run's accumulator is final there.  Every other record is issue(step, false_type).
        // phases: the clock phases its ring waits, its products and its first record's wait are charged to.
        auto walk_records = [&](auto issue, auto arrivals, auto phases, int& prev, auto open, auto retire) {
            using Clk = decltype(phases);
            auto record = [&](auto first) {
                union { uint2 raw; FusedStep s; } st;
                st.raw = __ldg(reinterpret_cast<const uint2*>(L.steps) + sidx);
                st.raw.x = uniform(st.raw.x);
                st.raw.y = uniform(st.raw.y);
                sidx = sidx + 1 == n_steps ? lu_steps : sidx + 1;
                NFB_CLK(Clk::mma);
                mbar_wait(bar(kBarWFull + slot), wpar, p.err, 220 + slot);
                NFB_CLK(Clk::ring);
                wgmma_fence();
                const bool last = issue(st.s, first);   // (commits its own group)
                if constexpr (decltype(first)::value) NFB_CLK(Clk::mma);
                wgmma_wait<1>();   // the previous record's products are complete: hand its slot back
                hand_back(arrivals, prev < 0 ? 0 : prev, prev >= 0);
                if constexpr (decltype(first)::value) NFB_CLK(Clk::tail);
                prev = (int)slot;
                if (++slot == kSlots) { slot = 0; wpar ^= 1; }
                return last;
            };
            bool last = false;
            if constexpr (decltype(open)::value) {
                last = record(std::true_type());
                retire();
            }
            while (!last) last = record(std::false_type());
        };
        // operands of half h of the record in the current slot (the skip bit: the record has no half h, or an all-zero one)
        auto half_ops = [&](const FusedStep& s, int h) {
            const uint32_t kc = h ? s.kc1 : s.kc, fl = h ? s.flags1 : s.flags;
            const uint32_t w = sbase + kOffW + slot * kSlotBytes + ((fl & kStepHalf) ? 0u : (uint32_t)h * s.n8 * 1024u);
            return MmaOps{aA + kc * kTileA, aA + (4 + kc) * kTileA, w, w + ((uint32_t)s.bytes16 << 3),
                          (uint32_t)!(fl & kStepSkip), 4u - ((fl >> kStepSlabShift) & 3u)};
        };
        // The records of one output slice of this warpgroup (until the one its flags mark last): its half of each goes
        // into acc, multiplied with its K-chunk.  OPENS: the slice's first record opens acc (FIRST; the packer keeps
        // K-chunk 0 of every slice, so that record always has products); otherwise every product accumulates onto acc.
        // Each record commits inside its own branch: a commit after the join would close the chain's group at the end
        // of its block and add a second, empty one, and wait_group 1 would then wait for the record's own products.
        // (The packer sets slab bits on final-layer records only: the LU map and the hidden GEMMs multiply all four.)
        auto slice_products = [&](float (&acc)[32], auto opens, auto quad) {
            return [&](const FusedStep& s, auto first) {
                constexpr bool Q = decltype(quad)::value;
                const MmaOps x = half_ops(s, wg);
                if constexpr (decltype(first)::value && decltype(opens)::value) {
                    mma_record<4, Q, 32, true>(acc, x);
                    wgmma_commit();
                } else if (x.on) {
                    mma_record<4, Q, 32>(acc, x);
                    wgmma_commit();
                } else {
                    wgmma_commit();
                }
                return ((wg ? s.flags1 : s.flags) & kStepLast) != 0;
            };
        };
        // a warpgroup without a slice passes the GEMM's records as one slice with no products
        auto no_products = [&](const FusedStep& s, auto) {
            wgmma_commit();
            return ((wg ? s.flags1 : s.flags) & kStepLast) != 0;
        };
        using One = std::integral_constant<int, 1>;
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
        NFB_CLK(kClkClaim);
        float lq_old = 0.f;
        if (rq == 2 && row_live && (layer > 0 || p.accumulate)) lq_old = __ldcg(p.logq + grow);
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
        // Row unit u = 2^-e, e = clamp(floor(log2 max|x_row|) + 1, 0, 126): |x| u < 1 for every input below 2^126, and < 4
        // up to the largest finite float.  Every fp16 operand of this unit stays inside the static bounds the packer
        // derived (nfb_api.cu plan_scales), which sit at least 4x (2 binades) below the fp16 maximum, whatever the magnitude
        // of the data; u = 1 for ordinary rows (|x| < 1 .. 2).  (126: 2^-e and 2^e are both normal floats.)
        auto set_row_exp = [&](float zmax) {
            int e = (int)((__float_as_uint(zmax) >> 23) & 0xffu) - 126;
            rowexp[r] = max(0, min(126, e));
        };
        if (rq == 0) {
            float zmax = 0.f;
            if (D == 64) zmax = rowmax[r];
            else
                for (int c = 0; c < D; ++c) zmax = fmaxf(zmax, fabsf(xs[xs_index(r, c)]));
            set_row_exp(zmax);
        }
        cons_bar_sync();
        auto ru = [&](float s, int row) { return s * pow2i(-rowexp[row]); };      // s u_row
        auto ruinv = [&](float s, int row) { return s * pow2i(rowexp[row]); };    // s / u_row
        auto get_x = [&](int c) -> float { return xs[xs_index(r, c)]; };
        auto put_y = [&](int c, float y) { xs[xs_index(r, c)] = y; };
        // A[:, 0:64] (K-chunk 0): fp16 hi/lo split of value(row, k) * u_row * sc; thread = (row, quarter of k)
        const int ar = et >> 2, aq = et & 3;
        auto store_a = [&](auto value, float sc_base) {
            const float sc = ru(sc_base, ar);
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
        float ladsum = 0.f, lad_even = 0.f;   // (lad_even: warpgroup 1 in the final layer, see there)
        // fold_lu (density direction): the packer multiplied the first conditioner matrix into the LU map, so the first
        // hidden GEMM reads the SAME A operand as the LU stage (the split of z)
        const bool folded = uniform(!SAMPLE && L.has_lu && L.fold_lu);
        if (lu_steps) {
            store_a([&](int k) { return k < D ? xs[xs_index(ar, k)] : 0.f; }, L.a_sc[0]);
            NFB_CLK(kClkLoad);
            int prev = -1;
            if (wg == 0) {
                float acc[32];
                walk_records(slice_products(acc, std::true_type(), std::true_type()), One(), LuClk(), prev,
                             std::true_type(), [] {});
                wgmma_wait<0>();
                hand_back(One(), prev, true);
                wgmma_hold(acc);
                // x' = acc + b (this thread: rows ra / rb, two columns of every 8-column group)
                const float ia = ruinv(L.a_inv[0], ra), ib = ruinv(L.a_inv[0], rb);
#pragma unroll
                for (int i = 0; i < 32; ++i) {
                    const int c = 8 * (i >> 2) + cq + (i & 1);
                    const int rr = (i & 2) ? rb : ra;
                    if (c < D) xs[xs_index(rr, c)] = fmaf(acc[i], (i & 2) ? ib : ia, __ldg(L.bias_lu + c));
                }
            } else {   // (the LU record has no half for warpgroup 1)
                walk_records(no_products, One(), LuClk(), prev, std::false_type(), [] {});
                wgmma_wait<0>();
                hand_back(One(), prev, true);
            }
            cons_bar_sync();   // x' of the whole tile is visible to both warpgroups
            NFB_CLK(kClkLu);
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
            NFB_CLK(kClkLoad);

            // the final layer's splines all run on warpgroup 1: warpgroup 0's sums so far go with them
            if (wg == 0) ldsum[rq * kRows + r] = ladsum;
            // ---- hidden layers: warpgroup wg owns the 64-column slices own(0), own(1) of every output (the packer's
            //      choice, nfb_fused_plan.h); a warpgroup without a slice passes the GEMM's records as one slice with
            //      no products ----
            // One walk per GEMM and warpgroup: slice own(1)'s first record is issued while own(0)'s last one multiplies,
            // its wait_group 1 completes own(0), and own(0)'s epilogue arithmetic (unscale + pre-summed bias, ReLU, scale
            // to the next GEMM's units, fp16 hi/lo) runs under own(1)'s products.  The tensor core drains once per GEMM;
            // only the stores wait for the barrier after that: the products of both warpgroups read the one A operand
            // that the output overwrites.
            // The slice count NS (0, 1, 2) is a template argument, and the residual stream and each t-phase temporary
            // are opened by a FIRST record on every path that reads them, so to the compiler they are written before
            // they are read: they are not live outside the hidden layers (the splines and the final layer's
            // accumulators need those registers), and nothing but a wgmma defines them while products are in flight
            // (anything else makes ptxas serialise every wgmma of the kernel, C7515).
            auto hidden = [&](auto ns) {
                constexpr int NA = decltype(ns)::value > 0 ? decltype(ns)::value : 1;
                // GEMM ph into acc (OPENS: its first record of each slice opens it), then its output -> A K-chunks own(q)
                auto gemm = [&](auto& acc, auto opens, int ph) {
                    constexpr int NS = decltype(ns)::value, NA = NS > 0 ? NS : 1;
                    const bool relu = ph + 1 < n_hidden;
                    const float inv_a = ruinv(L.a_inv[1 + ph], ra), inv_b = ruinv(L.a_inv[1 + ph], rb);
                    const float sc_a = ru(L.a_sc[2 + ph], ra), sc_b = ru(L.a_sc[2 + ph], rb);
                    // this thread's bias pairs (columns 8 g + cq, + 1 of each of its slices), loaded before the first
                    // record: the layer flag's acquire emptied L1, and the L2 round trip hides under the products
                    float2 bias[NA][8];
#pragma unroll
                    for (int q = 0; q < NS; ++q)
#pragma unroll
                        for (int g = 0; g < 8; ++g)
                            bias[q][g] = __ldg(reinterpret_cast<const float2*>(L.bias_h + ph * 256 + 64 * own(q) + 8 * g + cq));
                    // slice q's output as packed fp16 pairs, hi (pk[q][0]) and lo (pk[q][1]); pair p = 2 g + hb holds
                    // row (hb ? rb : ra), columns 8 g + cq, + 1 -- accumulator registers 2 p, 2 p + 1
                    uint32_t pk[NA][2][16];
                    auto pack = [&](int q, float (&a)[32]) {
                        wgmma_hold(a);
#pragma unroll
                        for (int p = 0; p < 16; ++p) {
                            const int g = p >> 1, hb = p & 1;
                            float v0 = fmaf(a[2 * p], hb ? inv_b : inv_a, bias[q][g].x);
                            float v1 = fmaf(a[2 * p + 1], hb ? inv_b : inv_a, bias[q][g].y);
                            if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                            v0 *= hb ? sc_b : sc_a;
                            v1 *= hb ? sc_b : sc_a;
                            const uint32_t hi = pack_f16x2(v0, v1);
                            const float2 hf = unpack_f16x2(hi);
                            pk[q][0][p] = hi;
                            pk[q][1][p] = pack_f16x2(v0 - hf.x, v1 - hf.y);
                        }
                    };
                    int prev = -1;
                    if constexpr (NS == 0) {
                        walk_records(no_products, One(), HidClk(), prev, std::false_type(), [] {});
                    } else {
                        walk_records(slice_products(acc[0], opens, NoQuad()), One(), HidClk(), prev, std::true_type(),
                                     [] {});
                        if constexpr (NS == 2)
                            walk_records(slice_products(acc[1], opens, NoQuad()), One(), HidClk(), prev, std::true_type(),
                                         [&] { pack(0, acc[0]); NFB_CLK(kClkHidEpi); });
                    }
                    wgmma_wait<0>();
                    hand_back(One(), prev, true);
                    NFB_CLK(kClkHidMma);
                    if constexpr (NS > 0) pack(NS - 1, acc[NS - 1]);
                    cons_bar_sync();   // every product of this GEMM has read the A operand: overwrite it with the output
                    // Each 8 x 8 block of a warp's accumulator rows and columns is one stmatrix matrix: stmatrix k writes
                    // column groups 2 k, 2 k + 1 of rows 16 wl .. 16 wl + 15, lane l giving row 16 wl + l % 16 of group
                    // 2 k + l / 16 (its SW128 chunk address).
#pragma unroll
                    for (int q = 0; q < NS; ++q)
#pragma unroll
                        for (int h = 0; h < 2; ++h)
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                stmatrix_x4(aA + (4 * h + own(q)) * kTileA + a_chunk_off(16 * wl + (lane & 15), 2 * k + (lane >> 4)),
                                            pk[q][h][4 * k], pk[q][h][4 * k + 1], pk[q][h][4 * k + 2], pk[q][h][4 * k + 3]);
                    fence_proxy_async_smem();
                    cons_bar_sync();   // the next GEMM's A operand is complete
                    NFB_CLK(kClkHidEpi);
                };
                float hres[NA][32];   // its part of the residual stream h
                gemm(hres, std::true_type(), 0);
                // residual blocks (n_hidden = 1 + 2 x blocks): the first GEMM into a temporary of its own, the second
                // onto the residual stream (h += W2 relu(...))
                for (int ph = 1; ph + 1 < n_hidden; ph += 2) {
                    float tacc[NA][32];
                    gemm(tacc, std::true_type(), ph);
                    gemm(hres, std::false_type(), ph + 1);
                }
            };
            if (own(0) < 0) hidden(std::integral_constant<int, 0>());
            else if (own(1) < 0) hidden(std::integral_constant<int, 1>());
            else hidden(std::integral_constant<int, 2>());

            // ---- final layer: record c = chunks 2c and 2c + 1, kFusedFeaturesPerChunk features (x 24 columns) each.
            //      Warpgroup 0 multiplies both halves of every record and stores the two accumulators to the staging
            //      tiles; warpgroup 1 takes them from there and evaluates the splines, two per thread and pair.  Neither
            //      waits for the other except through the tiles ("full" / "free"), so the products of pair c + 1 run
            //      under the splines of pair c. ----
            if (wg == 0) {
                static_assert(kFusedFeaturesPerChunk == 2, "a final-layer record is one N = 96 product");
                // The pairs alternate between two accumulators (half 0 in registers 0..23, half 1 in 24..47), so the
                // tensor core does not drain at a pair boundary: pair c + 1's first record is issued, its wait_group 1
                // completes pair c, and pair c goes to the staging tiles while that record multiplies.  The ring then
                // holds two of this warpgroup's slots at most (pair c's last record, pair c + 1's first).  Neither
                // accumulator is written by anything but wgmma while products are in flight: each pair's first product
                // overwrites its accumulator (scale-d 0, an immediate), and each is read only after the wait that
                // completes it -- any other definition makes ptxas serialise every wgmma of the kernel (C7515).
                auto products = [&](float (&acc)[48]) {
                    return [&](const FusedStep& s, auto first) {
                        // Both halves share the K-chunk and the first / last flags; one N = 96 product covers them, over
                        // the larger of their slab counts.  A half the record skips, and the slabs past a half's own
                        // count, are multiplied too: their weights are the masked-out zeros the packer wrote, which add
                        // an exact zero to every accumulator.  (A record always has a live half: the packer keeps only
                        // K-chunk 0 and the K-chunks one of the two chunks reaches; K-chunk 0 opens the pair.)
                        constexpr bool F = decltype(first)::value;
                        const MmaOps x = half_ops(s, 0), x1 = half_ops(s, 1);
                        const uint32_t n = max(x.on ? x.slabs : 0u, x1.on ? x1.slabs : 0u);
                        switch (n) {
                            case 1: mma_record<1, false, 48, F>(acc, x); wgmma_commit(); break;
                            case 2: mma_record<2, false, 48, F>(acc, x); wgmma_commit(); break;
                            case 3: mma_record<3, false, 48, F>(acc, x); wgmma_commit(); break;
                            default: mma_record<4, false, 48, F>(acc, x); wgmma_commit(); break;
                        }
                        return (s.flags & kStepLast) != 0;   // (the pair's last record is the same for both halves)
                    };
                };
                // The tiles carry the spline parameters themselves, acc / (scale u_row) + bias -- the same fmaf the spline
                // warpgroup applied to the raw accumulators before -- so the splines wait for no bias load.  This thread's
                // 12 bias pairs of pair ci (columns 8 g + cq, cq + 1 of either half) are loaded one pair ahead, behind the
                // hand-off that stages the pair before, where the products hide their latency.
                const float fin_a = ruinv(L.a_inv[1 + n_hidden], ra), fin_b = ruinv(L.a_inv[1 + n_hidden], rb);
                float2 fbias[2][6];
                auto load_bias = [&](int ci) {
                    if (ci >= n_pairs) return;
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int g = 0; g < 6; ++g)
                            fbias[h][g] = __ldg(reinterpret_cast<const float2*>(L.bias_f + (2 * ci + h) * L.F * 24 + 8 * g + cq));
                };
                // pair ci's products are complete: to the staging tiles once the previous pair's have been taken
                auto stage = [&](float (&acc)[48], int ci) {
                    wgmma_hold(acc);
                    if (ci > 0) stg_bar_wait<kBarStgFree>();
#pragma unroll
                    for (int i = 0; i < 24; i += 2) {
                        const int g = i >> 2;
                        const float u = (i & 2) ? fin_b : fin_a;
                        float* dst = stg0 + ((i & 2) ? rb : ra) * kStgLd + 8 * g + cq;
                        *reinterpret_cast<float2*>(dst) =
                            make_float2(fmaf(acc[i], u, fbias[0][g].x), fmaf(acc[i + 1], u, fbias[0][g].y));
                        *reinterpret_cast<float2*>(dst + kRows * kStgLd) =
                            make_float2(fmaf(acc[24 + i], u, fbias[1][g].x), fmaf(acc[25 + i], u, fbias[1][g].y));
                    }
                    stg_bar_arrive<kBarStgFull>();
                    load_bias(ci + 1);
                    NFB_CLK(kClkFinStage);
                };
                using Two = std::integral_constant<int, 2>;
                int prev = -1;
                // pair ci into acc; `done` holds pair ci - 1, staged under the first record of pair ci
                auto pair = [&](float (&acc)[48], float (&done)[48], int ci) __attribute__((always_inline)) {
                    walk_records(products(acc), Two(), FinClk(), prev, std::true_type(), [&] { stage(done, ci - 1); });
                };
                // after the last pair: its products complete, its last slot back
                auto finish = [&](float (&acc)[48], int ci) {
                    wgmma_wait<0>();
                    hand_back(Two(), prev, true);
                    NFB_CLK(kClkFinTail);
                    stage(acc, ci);
                };
                // (unrolled by two, so that accA and accB stay two fixed register sets; pair 0 is peeled so that every
                // read of either comes after a pair has written it)
                float accA[48], accB[48];
                if (n_pairs > 0) {
                    load_bias(0);
                    walk_records(products(accA), Two(), FinClk(), prev, std::true_type(), [] {});
                    for (int ci = 1;; ci += 2) {
                        if (ci == n_pairs) { finish(accA, ci - 1); break; }
                        pair(accB, accA, ci);
                        if (ci + 1 == n_pairs) { finish(accB, ci); break; }
                        pair(accA, accB, ci + 1);
                    }
                }
            } else {
                // It does not walk the final layer's records (the last of the step table): its cursors move past them
                // as walk_records moves warpgroup 0's.
                if (n_pairs > 0) {
                    const uint32_t adv = slot + (uint32_t)(n_steps - sidx);
                    slot = adv % kSlots;
                    wpar ^= (adv / kSlots) & 1u;
                    sidx = lu_steps;
                }
                // Row r's log-det partial sums keep their membership and order: lad_even continues the sum of the
                // warpgroup-0 thread of (row, f) over the even chunks, ladsum this thread's own over the odd chunks.
                const int f = (et >> 6) & 1;   // feature of each chunk this thread evaluates (for row r)
                lad_even = ldsum[f * kRows + r];
                const int F = L.F, T = L.T;
                for (int ci = 0; ci < n_pairs; ++ci) {
                    stg_bar_wait<kBarStgFull>();
                    // Both splines' parameters to registers (chunk 2 ci's tile, then 2 ci + 1's), and the tiles go back
                    // before any spline runs, so that the next pair can be staged under both.  (The packer folded log2(e)
                    // and the layer's 1/sqrt(H) into the w/h columns and biases; the product warpgroup has unscaled the
                    // products and added the biases.)
                    float pv[2][24];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const float4* sp = reinterpret_cast<const float4*>(stg0 + (h * kRows + r) * kStgLd + 24 * f);
#pragma unroll
                        for (int q = 0; q < 6; ++q) {
                            const float4 s4 = sp[q];
                            pv[h][4 * q] = s4.x;
                            pv[h][4 * q + 1] = s4.y;
                            pv[h][4 * q + 2] = s4.z;
                            pv[h][4 * q + 3] = s4.w;
                        }
                    }
                    if (ci + 1 < n_pairs) stg_bar_arrive<kBarStgFree>();   // (the last pair's tiles have no next writer)
                    NFB_CLK(kClkFinStage);
                    // The features t0 (even chunk) and t0 + F (odd chunk): both as one two-lane evaluation, whose
                    // chains interleave, when both are transformed, else the even one alone.  (Warp-uniform: t0
                    // depends on ci and f only.)
                    const int t0 = 2 * ci * F + f;
                    auto splines = [&](auto lanes) {
                        constexpr int N = decltype(lanes)::value;
                        int col[N];
                        float xin[N], y[N], l[N];
#pragma unroll
                        for (int h = 0; h < N; ++h) {
                            col[h] = L.tr_idx[t0 + h * F];
                            xin[h] = get_x(col[h]);
                            if (arsamp) xin[h] = row_live ? __ldcg(zdst + grow * D + col[h]) : 0.f;
                        }
                        rqs_core_lanes<N, 8, SAMPLE>(xin, [&pv](int h, int i) { return pv[h][i]; },
                                                     [&pv](int h, int i) { return pv[h][8 + i]; },
                                                     [&pv](int h, int i) { return pv[h][16 + i]; }, L.tail, y, l);
#pragma unroll
                        for (int h = 0; h < N; ++h) put_y(col[h], y[h]);
                        lad_even += l[0];
                        if constexpr (N == 2) ladsum += l[1];
                    };
                    if (t0 + F < T) splines(std::integral_constant<int, 2>());
                    else if (t0 < T) splines(std::integral_constant<int, 1>());
                    NFB_CLK(kClkFinSpline);
                }
            }
            cons_bar_sync();   // (AR sampling: every output of this pass is in xs before the next pass reads it)
        }  // passes
        // ---- log-det reduction over the four partial sums of each row (warpgroup 1 holds them: threads f = 0 the sums
        //      that began in quarters 0 and 2 of the threads, threads f = 1 those of quarters 1 and 3; added in quarter
        //      order), then store ----
        NFB_CLK(kClkFinStage);
        if (rq == 3) {
            ldsum[r] = lad_even;
            ldsum[kRows + r] = ladsum;
        }
        cons_bar_sync();
        if (rq == 2 && row_live) {
            const float tot = lad_even + ldsum[r] + ladsum + ldsum[kRows + r] +
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
        NFB_CLK(kClkStore);
    }
    NFB_CLK_END(wg, (et & 127) == 0);
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

#ifdef NFB_PHASE_CLOCKS
// out[3][kClkCount]: the sums of every fused launch on the current device since the last reset (synchronises the device)
extern "C" __attribute__((visibility("default"))) int nfb_phase_clocks_read(unsigned long long* out, int reset) {
    NFB_CUDA(cudaDeviceSynchronize());
    if (out) NFB_CUDA(cudaMemcpyFromSymbol(out, g_phase_clocks, sizeof(g_phase_clocks)));
    if (reset) {
        const unsigned long long zero[3][kClkCount] = {};
        NFB_CUDA(cudaMemcpyToSymbol(g_phase_clocks, zero, sizeof(zero)));
    }
    return NFB_OK;
}
// the phases per role in nfb_phase_clocks_read's rows, the unit count (the last entry) included
extern "C" __attribute__((visibility("default"))) int nfb_phase_clocks_count() { return kClkCount; }
#endif

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
