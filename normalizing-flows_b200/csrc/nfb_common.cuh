// nfb_common.cuh -- shared device helpers for the normflows-b200 kernels (sm_90a).
// PTX wrappers for mbarrier / bulk-copy (TMA) / wgmma + error plumbing for the C-ABI.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>

#define NFB_OK 0
#define NFB_ERR_CUDA 1
#define NFB_ERR_ARG 2
#define NFB_ERR_UNSUPPORTED 3
#define NFB_ERR_STATE 4

void nfb_set_error(const char* fmt, ...);

#define NFB_CUDA(call)                                                                   \
    do {                                                                                 \
        cudaError_t e__ = (call);                                                        \
        if (e__ != cudaSuccess) {                                                        \
            nfb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,                  \
                          cudaGetErrorString(e__));                                      \
            return NFB_ERR_CUDA;                                                         \
        }                                                                                \
    } while (0)

#define NFB_CHECK(cond, code, ...)                                                       \
    do {                                                                                 \
        if (!(cond)) {                                                                   \
            nfb_set_error(__VA_ARGS__);                                                  \
            return (code);                                                               \
        }                                                                                \
    } while (0)

#define NFB_LAUNCH_CHECK() NFB_CUDA(cudaGetLastError())

namespace nfb {

constexpr float kMinBinWidth = 1e-3f;    // utils/splines.py:6
constexpr float kMinBinHeight = 1e-3f;   // utils/splines.py:7
constexpr float kMinDerivative = 1e-3f;  // utils/splines.py:8
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// One lane of a fully-converged warp.  Issuing cp.async.bulk under this predicate (instead of `lane == 0`) lets
// ptxas keep the operands in uniform registers.
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .b32 %%rx;\n\t.reg .pred %%px;\n\t"
        "elect.sync %%rx|%%px, %1;\n\t"
        "@%%px mov.s32 %0, 1;\n\t}"
        : "+r"(pred)
        : "r"(0xffffffffu));
    return pred != 0;
}

// ----------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}
// A wait that can never end (a protocol bug) records `tag` in *err and traps: the host sees a launch failure instead
// of a hung device.  Out of line: a trap inlined into a warp-specialised kernel keeps ptxas from giving its consumer
// warps the registers setmaxnreg hands them.
static __device__ __noinline__ void fail_timeout(int* err, int tag) {
    if (err) atomicExch(err, tag);
    __threadfence_system();
    asm volatile("trap;");
}

// Bounded wait (~2 s): a protocol bug must never hang the device.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err, int tag) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) fail_timeout(err, tag);
    }
}

// Warp-level wait: ONE lane polls, the others park at the warp barrier (bar.warp.sync orders lane 0's acquire before
// the other lanes' subsequent accesses).  Used where a whole warp waits for one event.
__device__ __forceinline__ void mbar_wait_warp(uint32_t bar, uint32_t parity, int* err, int tag) {
    if ((threadIdx.x & 31) == 0 && !mbar_try_wait(bar, parity)) {
        long long t0 = clock64();
        while (!mbar_try_wait(bar, parity)) {
            if (clock64() - t0 > 4000000000LL) fail_timeout(err, tag);
        }
    }
    __syncwarp();
}

// ----------------------------------------------------------------------------------------
// TMA: 1-D bulk copy global -> shared with mbarrier completion (SASS: UBLKCP)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes,
                                         uint32_t bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
        ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------
// wgmma (sm_90a): one warpgroup (4 consecutive warps, the first a multiple of 4) multiplies a [64 x 16] A tile by a
// [16 x N] B tile from shared memory into fp32 accumulators held in its registers.  Accumulator register i of lane l
// in warp w of the group holds row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l % 4) + (i & 1).
// ----------------------------------------------------------------------------------------
// K-major SWIZZLE_128B canonical tile (rows of 128 B = 64 16-bit elements, 8-row groups 1024 B apart) or, with
// lbo16 / sbo16 set accordingly, the MN-major one (64-wide MN blocks LBO apart, 8-row k groups SBO apart).
// desc: [0,14) addr >> 4 | [16,30) LBO >> 4 | [32,46) SBO >> 4 | [62,64) layout = 1 (SWIZZLE_128B)
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo16 = 1, uint32_t sbo16 = 64) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)lbo16 << 16) | ((uint64_t)sbo16 << 32) | (1ull << 62);
}
// orders this thread's register / shared-memory writes before the warpgroup's next wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses to an accumulator across a wgmma that is still in flight
template <int R> __device__ __forceinline__ void wgmma_hold(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D (+)= A * B^T, A [64 x 16] and B [N x 16] both K-major (TA / TB = 1: MN-major); scale_d = 0 overwrites D;
// bf16 forms, on = 0: no operation (a predicate, which must be the same for the whole warpgroup, instead of a branch:
// ptxas serialises the wgmma of a warpgroup when one sits in a branch it cannot prove warp-uniform).
// The f16 forms (the fused spline kernel's) have no `on`: ptxas lowers a predicated wgmma to a branch around it, so each
// one lands in a basic block of its own with a warpgroup.arrive in front.  Their caller issues a record's products as
// one unpredicated chain and skips a whole chain with one warp-uniform branch around it.
__device__ __forceinline__ void wgmma_f16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_f16_n96(float (&d)[48], uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
        "}, %48, %49, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
        : "l"(a), "l"(b), "r"(scale_d));
}
// D = A * B^T with scale-d an immediate 0: D is written, not read, so it needs no value before (a zero-initialised
// accumulator would be instructions defining it, which ptxas does not allow while another wgmma of the stage is in flight)
__device__ __forceinline__ void wgmma_f16_n64_zero(float (&d)[32], uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, 0, 1, 1, 0, 0;"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]),
          "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]),
          "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]),
          "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31])
        : "l"(a), "l"(b));
}
__device__ __forceinline__ void wgmma_f16_n96_zero(float (&d)[48], uint64_t a, uint64_t b) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
        "}, %48, %49, 0, 1, 1, 0, 0;"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]), "=f"(d[8]),
          "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]), "=f"(d[16]),
          "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]), "=f"(d[24]),
          "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31]), "=f"(d[32]),
          "=f"(d[33]), "=f"(d[34]), "=f"(d[35]), "=f"(d[36]), "=f"(d[37]), "=f"(d[38]), "=f"(d[39]), "=f"(d[40]),
          "=f"(d[41]), "=f"(d[42]), "=f"(d[43]), "=f"(d[44]), "=f"(d[45]), "=f"(d[46]), "=f"(d[47])
        : "l"(a), "l"(b));
}
template <int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d, uint32_t on = 1) {
    asm volatile(
        "{\n\t.reg .pred p, q;\n\tsetp.ne.b32 p, %34, 0;\n\tsetp.ne.b32 q, %37, 0;\n\t"
        "@q wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
        "}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB), "r"(on));
}
template <int TA = 0, int TB = 0>
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d, uint32_t on = 1) {
    asm volatile(
        "{\n\t.reg .pred p, q;\n\tsetp.ne.b32 p, %66, 0;\n\tsetp.ne.b32 q, %69, 0;\n\t"
        "@q wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{"
        "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
        "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
        "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
        "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
        "}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
          "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
          "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d), "n"(TA), "n"(TB), "r"(on));
}

// warpgroup-wide register budget changes (the whole warpgroup executes them): a producer warpgroup hands registers to
// the consumer warpgroups of the same CTA
template <int N> __device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N> __device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------
// bf16 split helpers: v ~= hi + lo (+ lo2), each term a bf16 (round-to-nearest-even)
// ----------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo_elem, float hi_elem) {
    uint32_t r;  // cvt.rn.bf16x2.f32 d, a, b: a -> upper half, b -> lower half
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo_elem, float hi_elem) {
    uint32_t r;  // cvt.rn.f16x2.f32 d, a, b: a -> upper half, b -> lower half
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi_elem), "f"(lo_elem));
    return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t h) {  // .x = lower half, .y = upper half
    return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
// four 8 x 8 b16 matrices to shared memory (whole warp): lanes 8 i .. 8 i + 7 give the row addresses of matrix i, and
// r[i] of lane l holds its row l / 4, columns 2 (l % 4), + 1 -- the layout of a wgmma accumulator's packed halves
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r0), "r"(r1),
                 "r"(r2), "r"(r3) : "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

}  // namespace nfb
