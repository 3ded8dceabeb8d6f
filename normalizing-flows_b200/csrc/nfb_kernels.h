// nfb_kernels.h -- internal launch interface between the C-ABI layer (nfb_api.cu) and the kernels.
#pragma once
#include "nfb_common.cuh"

#include <mutex>

namespace nfb {

// Per-DEVICE one-time setup (function attributes and SM counts are per device/context, not per process):
// `fn(dev, sm_count)` runs once for each device ordinal a kernel is first launched on; thread-safe.
struct PerDevice {
    static constexpr int kMaxDev = 64;
    std::mutex mu;
    bool done[kMaxDev] = {};
    int sm_count[kMaxDev] = {};
    // returns the device's SM count (> 0) or -1 with the error set
    template <typename Fn> int ensure(Fn&& fn) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDev) {
            nfb_set_error("cudaGetDevice failed or device ordinal out of range");
            return -1;
        }
        std::lock_guard<std::mutex> lock(mu);
        if (!done[dev]) {
            int sms = 0;
            if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) {
                nfb_set_error("cudaDeviceGetAttribute(MultiProcessorCount) failed");
                return -1;
            }
            if (fn() != cudaSuccess) {
                nfb_set_error("per-device kernel attribute setup failed: %s", cudaGetErrorString(cudaGetLastError()));
                return -1;
            }
            sm_count[dev] = sms;
            done[dev] = true;
        }
        return sm_count[dev];
    }
};

// ---- generic kernels (nfb_kernels.cu) ----
int launch_rqs_rows(const float* zin, const float* params, float* zout, float* logdet,
                    long long rows, int feats, int ld, const int* fidx, int K, float tail,
                    float wh_scale, int inverse, cudaStream_t st);
int launch_rqs_rows_tails(const float* zin, const float* params, float* zout, float* logdet, long long rows, int feats,
                          int K, int nd, const float* tail, const int* circ, float wh_scale, int inverse,
                          cudaStream_t st);
int launch_periodic_features(const float* x, float* y, long long rows, int dim, const int* slot, const float* w,
                             const float* scale, const float* bias, cudaStream_t st);
int launch_rqs_shared(const float* zin, const float* table, float* zout, float* logdet,
                      long long rows, int feats, int ld, const int* fidx, int K, float tail,
                      int inverse, cudaStream_t st);
int launch_linear(const float* X, int ldx, const int* xidx, const float* W, const float* bias,
                  const float* R, int ldr, float* Y, int ldy, long long M, int N, int K, int act_in,
                  int act_out, float slope, cudaStream_t st);
int launch_maf_affine(const float* x, const float* params, float* y, float* logdet, long long rows, int d, int inverse,
                      int accumulate, cudaStream_t st);
int launch_mask_mul(const float* w, const float* m, float* out, long long n, cudaStream_t st);
struct LuPackArgs {
    const float* lower_e; const float* upper_e; const float* udiag; float eps; int n;
    float* W; float* Winv; float* logabsdet;
};
int launch_lu_pack_batched(const LuPackArgs* args_dev, int count, int n_max, cudaStream_t st);
int launch_lu_pack(const float* lower_e, const float* upper_e, const float* udiag, float eps, int n,
                   float* W, float* Winv, float* logabsdet, cudaStream_t st);
int launch_add_scalar(float* v, long long n, const float* c, float sign, cudaStream_t st);
int launch_fill(float* v, long long n, float c, cudaStream_t st);
int launch_gather_cols(const float* in, float* out, const int* idx, long long rows, int d,
                       long long inner, cudaStream_t st);
int launch_diag_gauss(const float* z, const float* loc, const float* log_scale, float* logq,
                      long long rows, int d, int accumulate, cudaStream_t st);
int launch_sum(const float* v, long long n, double scale, double* scratch, float* out,
               double* out_sum, cudaStream_t st);

// ---- image-shaped Glow pieces (nfb_glow.cu) ----
int launch_conv2d(const float* x, int ctot, int c0, const float* w, const float* bias, float* y, long long B,
                  int cin, int H, int W, int cout, int ks, float leaky, cudaStream_t st);
int launch_glow_fold(const float* P, const float* L, const float* U, const float* sign_S, const float* log_S,
                     const float* s, const float* t, int C, int HW, float* w_out, float* b_out, float* logdet,
                     cudaStream_t st);
int launch_coupling_image(float* z, const float* param, float* logdet, const float* logdet_const, long long B,
                          int C, int HW, int scale, int smap, int inv_split, int direction, int accumulate,
                          cudaStream_t st);
int launch_squeeze(const float* in, float* out, long long B, int C, int H, int W, int direction, cudaStream_t st);
int launch_glow_fold_fwd(const float* P, const float* L, const float* U, const float* sign_S, const float* log_S,
                         const float* s, const float* t, int C, int HW, float* w_out, float* b_out, float* logdet,
                         cudaStream_t st);
int launch_paste_channels(const float* in, float* out, long long B, int C, int c0, int n, int HW, cudaStream_t st);
int launch_copy_channels(const float* in, float* out, long long B, int C, int c0, int n, int HW, cudaStream_t st);
bool glow_cond_supported(int cin, int hid, int cout, int k1, int k2, int k3);
size_t glow_cond_packed_bytes(int cin, int hid, int cout);
int launch_glow_cond_pack(const float* w1, const float* w2, const float* w3t, int cin, int hid, int cout,
                          float gain_per_step, uint8_t* packed, cudaStream_t st);
int launch_glow_conditioner(const float* x, int ctot, int c0, int cin, const float* w1, const float* b1, const float* w2,
                            const float* b2, const float* w3t, const uint8_t* packed, float* y_taps, long long B, int H,
                            int W, int hid, int cout, float leaky, float gain_per_step, int* err, cudaStream_t st);
bool coupling_taps_supported(int C, int H, int W, int scale);
int launch_coupling_taps(float* z, const float* Y, const float* bias, float* logdet, const float* logdet_const, long long B,
                         int C, int H, int W, int scale, int smap, int inv_split, int direction, int accumulate,
                         cudaStream_t st);
int launch_tap_shift_add(const float* Y, const float* bias, float* out, long long B, int cout, int H, int W, int ks,
                         cudaStream_t st);
int launch_logit(const float* in, float* out, float* logdet, long long B, long long inner, float alpha, int direction,
                 int accumulate, cudaStream_t st);
int launch_class_cond_gauss(const float* z, const long long* y, const float* loc, const float* log_scale,
                            float* logq, long long B, int dim, int ncls, int accumulate, cudaStream_t st);

// ---- small-dimension affine stack (nfb_affine.cu) ----
constexpr int kAffMaxD = 16;
constexpr int kAffMaxW = 128;  // widest MLP layer supported
constexpr int kAffMaxLayers = 6;

struct AffMlp {
    int n_layers;                  // number of Linear layers (0 = absent)
    int sizes[kAffMaxLayers + 1];  // sizes[0] = in, sizes[n_layers] = out
    const float* w[kAffMaxLayers];
    const float* b[kAffMaxLayers];
};
enum { kOpMasked = 0, kOpConst = 1, kOpCoupling = 2, kOpPermute = 3 };
struct AffineOp {
    int type;
    int flags;      // coupling: bit0 scale, bits1-2 scale_map (0 exp,1 sigmoid,2 sigmoid_inv), bit3 channel_inv
    float slope;    // LeakyReLU slope of the MLPs
    int pad_;
    AffMlp s;       // masked: s-net ; coupling: param_map
    AffMlp t;       // masked: t-net
    const float* p0;  // masked: b[D] ; const: s[D]
    const float* p1;  // const: t[D]
    const int* fwd_idx;  // permute: forward index list
    const int* inv_idx;  // permute: inverse index list
};

size_t affine_op_size();
int launch_affine_stack(const void* ops_dev, int n_ops, const float* zin, float* zout, float* logq,
                        long long rows, int d, int accumulate, int direction, cudaStream_t st);

// ---- fused neural-spline block (nfb_fused_rqs.cu) ----
constexpr int kFusedTileRows = 64;          // rows of a work unit (the M of one wgmma)
constexpr int kFusedFeaturesPerChunk = 2;   // spline features per final-layer record (N = 24 per feature)
// One weight record of the packed stream: a W_hi tile followed by its W_lo twin, multiplied with K-chunk kc of the A
// operand.  Each tile stacks the [8 n8 x 64] halves of the two consumer warpgroups of the fused kernel (warpgroup 0's
// output slice, then warpgroup 1's).  The records of a slice are consecutive; the slices come in the order the kernel
// consumes them (LU map, hidden GEMMs slice by slice, final-layer chunks).
enum { kStepFirst = 1,    // first record of its slice: overwrites the accumulator
       kStepLast = 2,     // last record of its slice: the slice's epilogue follows
       kStepQuad = 4,     // four products (W_lo A_lo as well): the LU map, which transforms z itself
       kStepSkip0 = 8,    // warpgroup 0's half is all zero (MADE mask): no products
       kStepSkip1 = 16 }; // the same for warpgroup 1
struct __align__(8) FusedStep {
    uint16_t bytes16;    // record size / 16
    uint8_t n8;          // rows of each warpgroup's half of a tile / 8 (MMA N / 8)
    uint8_t kc;          // A-operand K-chunk
    uint8_t flags;       // kStep*
    uint8_t pad_[3];
};

// One fused [LULinearPermute +] spline block, packed.  Device-resident (uploaded at pack time): the kernel
// reads it through a pointer so that ONE persistent launch can walk a whole stack of blocks.
struct FusedLayer {
    int D, H, n_hidden, has_lu, T, F, n_chunks, n_id, n_steps;  // F = features per final-layer chunk
    int ar_passes;  // sampling direction of an autoregressive block: number of conditioner passes (= D), else 0
    int fold_lu;    // density unit with an LU stage: the first conditioner GEMM was folded into the LU map (it reads the
                    // split of z, like the LU stage), see nfb_api.cu repack_pair
    float tail;
    const uint8_t* wstream;
    const FusedStep* steps;
    const float* bias_lu;    // [64]
    const float* uncond;     // [n_id][23]
    const float* lu_logdet;  // device scalar or null
    signed char in_idx[64];    // conditioner input column per k (-1 = zero pad)
    unsigned char tr_idx[64];  // transformed feature columns
    unsigned char id_idx[64];  // identity feature columns (coupled layer)
    // fp16 operand scaling (all powers of two; nfb_api.cu plan_scales): index 0 = LU stage, 1 + g = GEMM g of the
    // conditioner (g = n_hidden: final layer).  A operand = true value * u_row * a_sc; true value = acc * a_inv / u_row.
    float a_sc[10], a_inv[10];
    alignas(16) float bias_h[7 * 256];   // [n_hidden <= 7][256], residual biases pre-summed along the stream
    alignas(16) float bias_f[64 * 24];   // [n_chunks * F <= 64][24] final-layer bias in chunk/column order
};
// Launch arguments.  Work units are (layer, kFusedTileRows-row tile) pairs in layer-major order; unit (l, t) may start
// once progress[t] >= l.  Rows of a tile are private to it, so layers l >= 1 update `zout` in place.
struct FusedParams {
    const FusedLayer* layers;  // [n_layers], in application order
    int n_layers;
    const float* zin;          // input of layer 0
    float* zout;               // output of every layer (and input of layers >= 1)
    long long z_stride;        // 0: layers update zout in place; > 0: layer l writes zout + l * z_stride (training pass)
    float* logq;
    long long rows;
    int accumulate;            // layer 0: logq += (1) or = (0); later layers always accumulate
    int* progress;             // [n_tiles] zero-initialised, or null when n_layers == 1
    int* ticket;               // zero-initialised unit counter (units are claimed in increasing order), or null: static
                               // assignment CTA b -> units b, b + grid, ... (single-layer launches)
    const unsigned int* wave_order;    // optional (with in_ready): diagonal (layer, tile group) order, two words per element:
    int wave_elems, wave_tpg;          //   layer | group << 8, first unit index; tiles per group (last group may be short)
    const int* in_ready;       // optional: number of rows of `zin` that have landed (chunked H2D in flight, written
                               // by the copy engine); layer-0 tiles wait for their rows.  null = all resident
    int* err;
};
int launch_fused_rqs(const FusedParams& p, int sm_count, int sample, cudaStream_t st);
int launch_fold_lu(const float* E0, const float* Elu, const float* blu, const int* in_idx, int H, int d, float gain,
                   float* G, float* delta, cudaStream_t st);

// general fp32 GEMM on the tensor core (csrc/nfb_gemm_tc.cu): training pass of the conditioners
struct GemmTcArgs {
    const float* A; const float* B; float* C;
    long long lda, ldb, ldc, M, N, K;
    int a_mn = 0, b_mn = 0, a_relu = 0, b_relu = 0, relu_out = 0, accumulate = 0;
    const float* bias = nullptr; const float* mask = nullptr; const float* mulm = nullptr; long long ldmask = 0;
    const float* resid = nullptr; long long ldres = 0;
    const uint8_t* b_packed = nullptr;  // optional: B pre-packed by launch_gemm_pack_b (same B, ldb, b_mn, N, K)
};
int launch_gemm_tc(const GemmTcArgs& a, int* err, cudaStream_t st);
size_t gemm_tc_packed_b_bytes(long long N, long long K, int b_mn);
int launch_gemm_pack_b(const float* B, long long ldb, int b_mn, long long N, long long K, uint8_t* out, cudaStream_t st);

// ---- training pass: element-wise / reduction kernels (nfb_backward.cu) ----
int launch_spline_bwd_rows(const float* xin, int ldx, const float* params, const float* g_out, const float* g_lq,
                           const int* fidx, long long rows, int T, int K, float tail, float wh_scale, float* g_params,
                           float* gx, cudaStream_t st);
int launch_spline_bwd_shared(const float* xin, int ldx, const float* table, const float* g_out, const float* g_lq,
                             const int* fidx, long long rows, int n_id, int K, float tail, float* g_table, float* gx,
                             cudaStream_t st);
int launch_colsum(const float* G, long long ld, long long M, int N, float* out, cudaStream_t st);
int launch_diag_gauss_bwd(const float* z, const float* loc, const float* ls, const float* g_lq, long long rows, int d,
                          float* gz, float* t_loc, float* t_ls, cudaStream_t st);
int launch_lu_param_bwd(const float* dW, const float* lower_e, const float* upper_e, const float* udiag, float eps,
                        int n, const float* g_logdet, float* g_lower, float* g_upper, float* g_udiag, cudaStream_t st);
int launch_scatter_cols(const float* in, float* out, const int* idx, long long rows, int n_in, int ld_out, int accumulate,
                        cudaStream_t st);
int launch_gather_cols_ld(const float* in, int ld_in, float* out, int n_out, const int* idx, long long rows,
                          cudaStream_t st);
int launch_axpy(const float* x, float a, float* y, long long n, int accumulate, cudaStream_t st);
int launch_split_table(const float* tab, int n, float* gw, float* gh, float* gd, cudaStream_t st);

// ---- invertible residual block, element-wise pieces (nfb_residual.cu) ----
int launch_swish(const float* x, float b, long long n, float* a, float* da, cudaStream_t st);
int launch_mul_rows(const float* S, const float* m, long long n, int nt, float* T, cudaStream_t st);
int launch_logdet2(const float* jt, long long B, float* out, cudaStream_t st);
int launch_glu_residual(const float* h, const float* t, const float* c, long long n, float* out, cudaStream_t st);
int launch_rowdot(const float* a, const float* b, long long rows, int d, float c, int accumulate, float* out,
                  cudaStream_t st);

// tensor-core fp32 accumulation truncates: relative loss per K=16 MMA step, compensated at pack time (nfb_api.cu)
constexpr float kAccStepGain = 2.4e-8f;
// implicit-GEMM convolution on the tensor core (csrc/nfb_conv_tc.cu)
bool conv_tc_supported(int cin, int cout, int ks);
int launch_conv2d_tc(const float* x, int ctot, int c0, const float* w, const float* bias, float* y, long long B,
                     int cin, int H, int W, int cout, int ks, float leaky, float gain_per_step, int* err,
                     cudaStream_t st);
int launch_build_effective(const float* W, const float* M, int src_cols, const int* src_row,
                           const int* src_col, const float* row_scale, float* E, int n_pad,
                           int k_pad, float gain, cudaStream_t st);
struct PackRec { int row0, nrows, kc, pad_; unsigned long long off_hi, off_lo; };  // one weight record of a GEMM
int launch_pack_records(const float* E, int k_pad, const PackRec* recs_dev, int n_recs, int max_rows, float scale,
                        uint8_t* base, cudaStream_t st);
int launch_swizzle_split(const float* E, int n_pad, int k_pad, int rows_per_rec, int nsplit, float scale,
                         uint8_t* out, cudaStream_t st);
int launch_matrix_norms(const float* E, int n, int k, float* out3, cudaStream_t st);

}  // namespace nfb
