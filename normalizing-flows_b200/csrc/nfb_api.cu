// nfb_api.cu -- the extern "C" surface declared in include/nfb200.h.
//
// A `nfb_flow` is the packed, device-resident image of `NormalizingFlow(q0, flows)`
// (normflows/core.py:9-25): the ordered layer list, each layer's parameters re-laid-out for the
// kernels, and the execution plan for the density pass (core.py:98-100 walks the layers
// last-to-first calling `.inverse`) and the sampling pass (core.py:52-54).
//
// Execution plan ("groups"):
//   FUSED  : [LULinearPermute +] neural-spline block on the wgmma kernel (nfb_fused_rqs.cu)
//   AFFINE : a maximal run of low-dimensional affine-family layers in one kernel (nfb_affine.cu)
//   SINGLE : any other layer through the generic fp32 kernels (nfb_kernels.cu)
#include <algorithm>
#include <cstdarg>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include <memory>
#include <string>
#include <vector>

#include "../../include/nfb200.h"
#include "nfb_kernels.h"

static thread_local std::string g_err;
static constexpr float kLog2eHost = 1.4426950408889634f;

// The tensor core adds each K=16 step into the fp32 accumulator with truncation (round toward zero), so a chain
// of n MMA steps comes out short by a small one-sided amount: per step half an ulp of the running sum,
// E[ulp(s)/|s|] = 2^-23 / (2 ln 2) = 8.6e-8 for a log-uniform mantissa, times 2/3 because the partial sums of a
// random-sign dot product grow like sqrt(k/n): ~2.9e-8 per step.  The packer therefore scales each GEMM's weights by
// 1 + kAccStepGain * steps.  Measured on H100 (wgmma) against the fp64 oracle (tools/gpu_debug.py bias: 4-layer d=64
// stacks, 3000 rows, |log_prob| ~ 270): mean signed log_prob error +8.0e-4 (autoregressive) / +4.0e-4 (coupling)
// uncompensated, +3.5e-4 / +1.2e-4 at 1.5e-8 per step, -8.6e-5 / -1.4e-4 at 2.9e-8, and +1.2e-4 / -7e-6 at 2.4e-8 =
// kAccStepGain, between the two stacks' zero crossings.  The plain-fp32 kernels' own bias on the same rows is
// -4.8e-5 / -2.9e-5; test_trained_weights_parity pins the residual.  NFB_ACC_COMP_STEP overrides the constant
// (calibration runs).
static float acc_gain(int mma_steps) {
    static const float per_step = [] {
        const char* e = getenv("NFB_ACC_COMP_STEP");
        return e ? (float)atof(e) : nfb::kAccStepGain;
    }();
    return 1.f + per_step * (float)mma_steps;
}
void nfb_set_error(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
}

namespace {
using namespace nfb;

struct DevBuf {
    void* p = nullptr;
    size_t bytes = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) { release(); p = o.p; bytes = o.bytes; o.p = nullptr; o.bytes = 0; }
        return *this;
    }
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
    int reserve(size_t n) {
        if (n <= bytes) return NFB_OK;
        release();
        NFB_CUDA(cudaMalloc(&p, n ? n : 16));
        bytes = n;
        return NFB_OK;
    }
    template <typename T> T* as() const { return static_cast<T*>(p); }
    template <typename T> int upload(const std::vector<T>& v) {
        int rc = reserve(v.size() * sizeof(T));
        if (rc) return rc;
        if (!v.empty()) NFB_CUDA(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
        return NFB_OK;
    }
};

// A batch of small device->host reads through ONE pinned staging buffer and ONE stream synchronisation (every blocking
// cudaMemcpy of a few hundred bytes costs ~15 us of host time and a device sync; the packer used to issue ~25 per layer
// pair and optimizer step).  add() queues a copy, run() waits once, get() hands the floats out.
struct StagedReads {
    float* host = nullptr;   // pinned
    size_t cap = 0, used = 0;
    ~StagedReads() { if (host) cudaFreeHost(host); }
    int reserve(size_t floats) {
        if (floats <= cap) return NFB_OK;
        if (host) cudaFreeHost(host);
        host = nullptr; cap = 0;
        NFB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&host), floats * sizeof(float)));
        cap = floats;
        return NFB_OK;
    }
    void reset() { used = 0; }
    // returns the offset of the queued block (floats); the buffer must have been reserved large enough
    int add(const float* dev, size_t n, cudaStream_t st, size_t* off) {
        NFB_CHECK(used + n <= cap, NFB_ERR_STATE, "staged reads: buffer too small (%zu + %zu > %zu)", used, n, cap);
        *off = used;
        if (n) NFB_CUDA(cudaMemcpyAsync(host + used, dev, n * sizeof(float), cudaMemcpyDeviceToHost, st));
        used += n;
        return NFB_OK;
    }
    int run(cudaStream_t st) { NFB_CUDA(cudaStreamSynchronize(st)); return NFB_OK; }
    void get(size_t off, size_t n, std::vector<float>& out) const { out.assign(host + off, host + off + n); }
};

template <typename T>
int download(const T* dev, size_t n, std::vector<T>& out) {
    out.resize(n);
    if (n) NFB_CUDA(cudaMemcpy(out.data(), dev, n * sizeof(T), cudaMemcpyDeviceToHost));
    return NFB_OK;
}

#define NFB_TRY(expr) do { int rc__ = (expr); if (rc__) return rc__; } while (0)

enum LayerKind { L_AR_RQS, L_COUPLED_RQS, L_LU, L_MASKED_AFFINE, L_AFFINE_COUPLING, L_AFFINE_CONST, L_PERMUTE };

struct NetDesc {  // deep copy of nfb_resnet_desc_t
    int in = 0, H = 0, out = 0, nb = 0;
    const float *w0 = nullptr, *b0 = nullptr, *m0 = nullptr, *wf = nullptr, *bf = nullptr, *mf = nullptr;
    std::vector<const float*> wb, bb, mb;
};

struct NetPack {  // generic path: effective (mask-multiplied) fp32 weights
    std::vector<DevBuf> owned;
    const float* w0 = nullptr;
    const float* wf = nullptr;
    std::vector<const float*> wb;
};

struct FusedPack {
    bool ok = false;
    int D = 0, H = 0, n_hidden = 0, T = 0, F = 0, n_chunks = 0, n_id = 0, n_steps = 0;
    float tail = 3.f;
    size_t rqs_bytes = 0;
    std::vector<FusedStep> steps_host;
    DevBuf wstream, steps, uncond;
    std::vector<float> bias_h, bias_f;
    std::vector<int> in_idx, tr_idx, id_idx;
    struct Rec { int row0, nrows, kc; size_t off_hi, off_lo; };
    struct Gemm { DevBuf src_row, src_col, row_scale, recs_dev; const float* W; const float* M; int src_cols, n_pad, k_pad;
                  int max_rows = 0; std::vector<Rec> recs; };
    std::vector<int> hperm;  // sorted-by-degree order of the hidden units (identity for unmasked nets)
    std::vector<Gemm> gemms;
    // LU + this block as one launch (built when the next layer in list order is an LU)
    bool pair_ok = false;
    int pair_steps = 0;
    DevBuf pair_wstream, pair_steps_dev, lu_src_row, lu_src_col, bias_lu;
    // LU fold (density pair): first conditioner matrix times the LU map, packed as GEMM 0 of the pair (repack_fused)
    bool images_dirty = true;              // per-layer device images (layer_dev, layer_fwd_dev, pair_dev) need a refresh
    int ar_passes_fwd = 0;
    bool fold_ok = false;                  // decided per repack (scale plan permitting)
    DevBuf in_idx_dev, fold_lu, fold_G, fold_delta, fold_recs;
    std::vector<float> fold_delta_host;    // W0 b_lu in sorted hidden order
    int pw_fold = 0;
    FusedLayer host_layer{}, host_pair{};  // packed descriptors (host copies)
    float b_in0 = 1.f;                     // bound on |conditioner input| * u_row this block was planned for
    int pa[10] = {}, pw[10] = {};          // per-GEMM power-of-two exponents (A operand / weights), see plan_scales
    DevBuf layer_dev, pair_dev;           // ... and their device images (one FusedLayer each)
    DevBuf layer_fwd_dev;                 // block alone in the sampling direction (ar_passes = D for autoregressive)
    // sampling direction (coupling layers only): [inverse LU map of the PREVIOUS layer in list order + this
    // block, spline inverted] as one unit of the forward whole-stack launch
    bool fwd_ok = false;
    DevBuf fwd_wstream, fwd_steps_dev, fwd_src_row, fwd_src_col, fwd_bias_lu;
    FusedLayer host_fwd{};
};

struct Layer {
    LayerKind kind;
    int D = 0, K = 8;
    float tail = 3.f;
    // rqs
    NetDesc net;
    NetPack pack;
    FusedPack fused;
    float wh_scale = 1.f;
    int n_id = 0, n_tr = 0;
    const int64_t *id64 = nullptr, *tr64 = nullptr;
    DevBuf id_idx, tr_idx;  // int32 on device
    const float *uw = nullptr, *uh = nullptr, *ud = nullptr;
    DevBuf uncond;          // [n_id][3K-1]
    // lu
    nfb_lu_desc_t lu{};
    DevBuf lu_Wd, lu_Ws, lu_bs, lu_logdet, lu_logdet_neg, lu_perm, lu_tmp;
    // fp16 operand planning: {inf-norm, max|w|} of W (density map) and W^-1 (sampling map), max |bias| of each
    float lu_norm_d = 1.f, lu_max_d = 1.f, lu_bmax_d = 0.f, lu_norm_s = 1.f, lu_max_s = 1.f, lu_bmax_s = 0.f;
    std::vector<int> perm_host, inv_perm_host;
    std::vector<float> lu_bs_host, lu_bias_host;
    // affine family
    AffineOp op{};
    std::vector<int> perm_fwd, perm_inv;
    DevBuf perm_fwd_dev, perm_inv_dev;
};

enum GroupKind { G_FUSED_PAIR, G_FUSED, G_AFFINE, G_SINGLE };
struct Group { GroupKind kind; int first, last; DevBuf ops; };

}  // namespace

struct nfb_flow {
    int D = 0;
    bool finalized = false;
    bool use_tc = true;
    int sm_count = 132;
    std::vector<std::unique_ptr<Layer>> layers;
    std::vector<Group> groups;
    const float* base_loc = nullptr;
    const float* base_log_scale = nullptr;
    // workspaces
    StagedReads reads;              // pinned staging for the packer's small device->host reads
    DevBuf wave_order;              // diagonal unit order of gated host passes (launch_fused_stack)
    int wave_layers = 0;
    long long wave_tiles = 0;
    DevBuf lu_args;                 // batched LU pack: one LuPackArgs per LULinearPermute layer
    DevBuf stack_layers, progress;  // whole-stack launch: FusedLayer[stack_n] in density order + tile flags
    int stack_n = 0;
    // sampling-direction plan: units (LU index or -1, spline index) in list order, optional trailing LU
    std::vector<std::pair<int, int>> fwd_units;
    int fwd_trailing_lu = -1, fwd_n = 0;
    DevBuf fwd_layers;
    DevBuf zA, zB, logq, hA, hB, hT, params, E, scratch_sum, loss, err, ar_tmp, pair_tmp, host_x, zfinal, norms;
    long long launches = 0;
    // host-buffer entry points: chunked H2D on a copy stream, gated tile by tile inside the whole-stack kernel
    cudaStream_t copy_stream = nullptr;
    cudaEvent_t ev_reset = nullptr, ev_copied = nullptr;
    int* h_seq = nullptr;            // pinned: h_seq[c] = rows resident after chunk c
    DevBuf in_ready;                 // device int: rows of the current host batch that have landed
    // training pass workspaces (nfb_flow_backward)
    DevBuf tr_store, tr_h, tr_P, tr_gP, tr_ga, tr_gb, tr_xp, tr_gxp, tr_zp, tr_gzp, tr_in, tr_gin, tr_g0, tr_g1, tr_small,
        tr_glq, tr_t0, tr_t1, tr_wpack;
    const int* cur_in_ready = nullptr;
    ~nfb_flow() {
        if (copy_stream) cudaStreamDestroy(copy_stream);
        if (ev_reset) cudaEventDestroy(ev_reset);
        if (ev_copied) cudaEventDestroy(ev_copied);
        if (h_seq) cudaFreeHost(h_seq);
    }
};

namespace {

// ------------------------------------------------------------------------------------------
// generic conditioner
// ------------------------------------------------------------------------------------------
int copy_net(const nfb_resnet_desc_t& d, NetDesc& n) {
    NFB_CHECK(d.in_features > 0 && d.hidden_features > 0 && d.out_features > 0 && d.num_blocks >= 0,
              NFB_ERR_ARG, "resnet desc: bad sizes");
    NFB_CHECK(d.w_initial && d.b_initial && d.w_final && d.b_final, NFB_ERR_ARG, "resnet desc: null weights");
    n.in = d.in_features; n.H = d.hidden_features; n.out = d.out_features; n.nb = d.num_blocks;
    n.w0 = d.w_initial; n.b0 = d.b_initial; n.m0 = d.m_initial;
    n.wf = d.w_final; n.bf = d.b_final; n.mf = d.m_final;
    for (int i = 0; i < 2 * n.nb; ++i) {
        NFB_CHECK(d.w_blocks && d.b_blocks && d.w_blocks[i] && d.b_blocks[i], NFB_ERR_ARG, "resnet desc: null block weights");
        n.wb.push_back(d.w_blocks[i]);
        n.bb.push_back(d.b_blocks[i]);
        n.mb.push_back(d.m_blocks ? d.m_blocks[i] : nullptr);
    }
    return NFB_OK;
}

int pack_net_generic(const NetDesc& n, NetPack& p, cudaStream_t st) {
    p.wb.clear();
    size_t slot = 0;  // the masked-weight buffers are kept across repacks (a cudaFree + cudaMalloc pair per matrix and
                      // optimizer step was most of the packer's host time)
    auto eff = [&](const float* w, const float* m, size_t cnt, const float** out) -> int {
        if (!m) { *out = w; return NFB_OK; }
        if (slot == p.owned.size()) p.owned.emplace_back();
        DevBuf& b = p.owned[slot++];
        NFB_TRY(b.reserve(cnt * sizeof(float)));
        NFB_TRY(launch_mask_mul(w, m, b.as<float>(), (long long)cnt, st));
        *out = b.as<float>();
        return NFB_OK;
    };
    NFB_TRY(eff(n.w0, n.m0, (size_t)n.H * n.in, &p.w0));
    for (int i = 0; i < 2 * n.nb; ++i) {
        const float* w;
        NFB_TRY(eff(n.wb[i], n.mb[i], (size_t)n.H * n.H, &w));
        p.wb.push_back(w);
    }
    NFB_TRY(eff(n.wf, n.mf, (size_t)n.out * n.H, &p.wf));
    return NFB_OK;
}

// params[rows, out] = net(X[:, xidx])
int run_net_generic(nfb_flow* f, const NetDesc& n, const NetPack& p, const float* X, int ldx,
                    const int* xidx, long long rows, float* params, cudaStream_t st) {
    NFB_TRY(f->hA.reserve((size_t)rows * n.H * 4));
    NFB_TRY(f->hB.reserve((size_t)rows * n.H * 4));
    NFB_TRY(f->hT.reserve((size_t)rows * n.H * 4));
    float* h = f->hA.as<float>();
    float* h2 = f->hB.as<float>();
    float* t = f->hT.as<float>();
    NFB_TRY(launch_linear(X, ldx, xidx, p.w0, n.b0, nullptr, 0, h, n.H, rows, n.H, n.in, 0, 0, 0.f, st));
    f->launches++;
    for (int b = 0; b < n.nb; ++b) {  // nets/resnet.py:37-50 / nets/made.py:199-214
        NFB_TRY(launch_linear(h, n.H, nullptr, p.wb[2 * b], n.bb[2 * b], nullptr, 0, t, n.H, rows, n.H, n.H, 1, 0, 0.f, st));
        NFB_TRY(launch_linear(t, n.H, nullptr, p.wb[2 * b + 1], n.bb[2 * b + 1], h, n.H, h2, n.H, rows, n.H, n.H, 1, 0, 0.f, st));
        f->launches += 2;
        std::swap(h, h2);
    }
    NFB_TRY(launch_linear(h, n.H, nullptr, p.wf, n.bf, nullptr, 0, params, n.out, rows, n.out, n.H, 0, 0, 0.f, st));
    f->launches++;
    return NFB_OK;
}

// ------------------------------------------------------------------------------------------
// fused pack
// ------------------------------------------------------------------------------------------
int build_fused(nfb_flow* f, Layer& L, cudaStream_t st) {
    FusedPack& F = L.fused;
    F.ok = false; F.pair_ok = false;
    const NetDesc& n = L.net;
    const bool ar = (L.kind == L_AR_RQS);
    const int T = ar ? L.D : L.n_tr;
    if (!f->use_tc) return NFB_OK;
    if (L.K != 8 || L.D > 64 || n.H % 64 != 0 || n.H > 256 || n.in > 64 || T > 64 || T < 1) return NFB_OK;
    if (n.out != T * 23) return NFB_OK;
    const int H = n.H, n_hidden = 1 + 2 * n.nb;
    // final layer: fpc features (x24 columns: 23 parameters + 1 pad) per record; a record of N = 48 rows keeps the
    // accumulator of the final layer at 24 registers and its staging tile small (nfb_fused_rqs.cu)
    const int fpc = kFusedFeaturesPerChunk;
    const int n_chunks = ((T + fpc - 1) / fpc + 1) & ~1;   // even: a record carries one chunk per consumer warpgroup
    const int kcs_h = H / 64;
    const int crow = fpc * 24;  // rows (MMA N) per final-layer chunk
    if (n_hidden > 7) return NFB_OK;  // tables inside FusedLayer

    // ---- MADE masks: sort hidden units by degree so that every masked matrix is block-triangular, and
    //      find the all-zero [64 x 64] blocks to drop (nets/made.py:57-76 degree rules) ----
    const bool masked = n.m0 != nullptr;
    std::vector<int> perm(H);
    for (int i = 0; i < H; ++i) perm[i] = i;
    std::vector<float> m_init, m_hid, m_fin;
    if (masked) {
        NFB_TRY(download(n.m0, (size_t)H * n.in, m_init));
        std::vector<int> deg(H, 0);  // row sum of the input mask = number of inputs a unit may see = its degree
        for (int i = 0; i < H; ++i) for (int j = 0; j < n.in; ++j) deg[i] += m_init[(size_t)i * n.in + j] != 0.f;
        std::stable_sort(perm.begin(), perm.end(), [&](int x, int y) { return deg[x] < deg[y]; });
        if (n.nb > 0) NFB_TRY(download(n.mb[0], (size_t)H * H, m_hid));  // all hidden masks share the structure
        NFB_TRY(download(n.mf, (size_t)n.out * H, m_fin));
    }
    F.hperm = perm;
    // does output slice j (rows [64 j, 64 j + 64) in sorted order) of a hidden GEMM have a non-zero in K-chunk kc?
    auto hidden_needs = [&](int j, int kc) -> bool {
        if (!masked || m_hid.empty()) return true;
        for (int i = 64 * j; i < 64 * j + 64; ++i)
            for (int k = kc * 64; k < kc * 64 + 64; ++k)
                if (m_hid[(size_t)perm[i] * H + perm[k]] != 0.f) return true;
        return false;
    };
    // does chunk c of the final layer have a non-zero in K-chunk kc?
    auto final_needs = [&](int c, int kc) -> bool {
        if (!masked) return true;
        for (int i = 0; i < crow; ++i) {
            const int t = fpc * c + i / 24, q = i % 24;
            if (t >= T || q >= 23) continue;
            for (int k = kc * 64; k < kc * 64 + 64; ++k)
                if (m_fin[(size_t)(t * 23 + q) * H + perm[k]] != 0.f) return true;
        }
        return false;
    };

    // ---- GEMM source tables (effective matrices are built in sorted hidden order) ----
    F.gemms.clear();
    auto add_gemm = [&](const float* W, const float* M, int src_cols, int n_pad, int k_pad,
                        const std::vector<int>& sr, const std::vector<int>& sc,
                        const std::vector<float>& rs) -> int {
        FusedPack::Gemm g;
        g.W = W; g.M = M; g.src_cols = src_cols; g.n_pad = n_pad; g.k_pad = k_pad;
        NFB_TRY(g.src_row.upload(sr));
        NFB_TRY(g.src_col.upload(sc));
        if (!rs.empty()) NFB_TRY(g.row_scale.upload(rs));
        F.gemms.push_back(std::move(g));
        return NFB_OK;
    };
    {
        std::vector<int> sc(64);
        for (int k = 0; k < 64; ++k) sc[k] = k < n.in ? k : -1;
        NFB_TRY(add_gemm(n.w0, n.m0, n.in, H, 64, perm, sc, {}));
    }
    for (int i = 0; i < 2 * n.nb; ++i) NFB_TRY(add_gemm(n.wb[i], n.mb[i], H, H, H, perm, perm, {}));
    {
        std::vector<int> fr(n_chunks * crow);
        std::vector<float> fs(n_chunks * crow);
        for (int i = 0; i < n_chunks * crow; ++i) {
            const int t = fpc * (i / crow) + (i % crow) / 24, q = (i % crow) % 24;
            fr[i] = (t < T && q < 23) ? t * 23 + q : -1;
            fs[i] = (q < 16) ? L.wh_scale * kLog2eHost : 1.f;  // softmax logits leave the GEMM in the log2 domain
        }
        NFB_TRY(add_gemm(n.wf, n.mf, H, n_chunks * crow, H, fr, perm, fs));
    }

    // ---- step table + record list (same order).  A record carries the same K-chunk of two output slices, one per
    //      consumer warpgroup of the kernel: hidden GEMMs split their 64-column slices in two halves ([0, half) and
    //      [half, ns)), the final layer deals its chunks alternately.  K-chunks ascend (the accumulation order is part
    //      of the validated numerics); K-chunk 0 is always kept, so that every slice has a first record that initialises
    //      its accumulator; a K-chunk only one of the two slices reaches is skipped by the other warpgroup. ----
    std::vector<FusedStep> steps;
    size_t off = 0;
    // rows [row_a, row_a + nrows) for warpgroup 0 and (row_b >= 0) [row_b, row_b + nrows) for warpgroup 1
    auto add_pair = [&](FusedPack::Gemm& g, int row_a, int row_b, int nrows, const std::vector<bool>& need_a,
                        const std::vector<bool>& need_b, bool onto) {
        const int tot = row_b >= 0 ? 2 * nrows : nrows;
        std::vector<int> kcs;
        for (size_t kc = 0; kc < need_a.size(); ++kc)
            if (kc == 0 || need_a[kc] || (row_b >= 0 && need_b[kc])) kcs.push_back((int)kc);
        for (size_t i = 0; i < kcs.size(); ++i) {
            const int kc = kcs[i];
            FusedStep st{};
            st.bytes16 = (uint16_t)(tot * 16);
            st.n8 = (uint8_t)(nrows / 8);
            st.kc = (uint8_t)kc;
            st.flags = (uint8_t)(((i == 0 && !onto) ? kStepFirst : 0) | (i + 1 == kcs.size() ? kStepLast : 0) |
                                 ((kc > 0 && !need_a[kc]) ? kStepSkip0 : 0) |
                                 ((row_b < 0 || (kc > 0 && !need_b[kc])) ? kStepSkip1 : 0));
            steps.push_back(st);
            g.recs.push_back(FusedPack::Rec{row_a, nrows, kc, off, off + (size_t)tot * 128});
            if (row_b >= 0)
                g.recs.push_back(FusedPack::Rec{row_b, nrows, kc, off + (size_t)nrows * 128, off + (size_t)(tot + nrows) * 128});
            off += (size_t)tot * 256;
        }
    };
    const int half = (kcs_h + 1) / 2;
    for (int ph = 0; ph < n_hidden; ++ph) {
        const bool accum_onto = (ph > 0 && (ph & 1) == 0);  // second GEMM of a residual block: h += ...
        const int kcs = (ph == 0) ? 1 : kcs_h;
        auto need = [&](int j) {
            std::vector<bool> v(kcs);
            for (int kc = 0; kc < kcs; ++kc) v[kc] = ph == 0 || hidden_needs(j, kc);
            return v;
        };
        for (int q = 0; q < half; ++q) {
            const int jb = q + half < kcs_h ? q + half : -1;
            add_pair(F.gemms[ph], 64 * q, jb >= 0 ? 64 * jb : -1, 64, need(q), jb >= 0 ? need(jb) : need(q), accum_onto);
        }
    }
    for (int c = 0; c < n_chunks; c += 2) {
        auto need = [&](int cc) {
            std::vector<bool> v(kcs_h);
            for (int kc = 0; kc < kcs_h; ++kc) v[kc] = final_needs(cc, kc);
            return v;
        };
        add_pair(F.gemms[n_hidden], c * crow, (c + 1) * crow, crow, need(c), need(c + 1), false);
    }
    F.steps_host = steps;
    F.n_steps = (int)steps.size();
    F.D = L.D; F.H = H; F.n_hidden = n_hidden; F.T = T; F.F = fpc; F.n_chunks = n_chunks; F.tail = L.tail;
    F.n_id = ar ? 0 : L.n_id;
    const size_t total = off;
    F.rqs_bytes = total;
    NFB_TRY(F.wstream.reserve(total));
    NFB_TRY(F.steps.upload(steps));

    // ---- index lists ----
    std::vector<int> in_idx(64, -1), tr_idx(T);
    if (ar) {
        for (int k = 0; k < L.D; ++k) in_idx[k] = k;
        for (int t = 0; t < T; ++t) tr_idx[t] = t;
    } else {
        std::vector<int64_t> id64, tr64;
        NFB_TRY(download(L.id64, (size_t)L.n_id, id64));
        NFB_TRY(download(L.tr64, (size_t)L.n_tr, tr64));
        for (int k = 0; k < L.n_id; ++k) in_idx[k] = (int)id64[k];
        for (int t = 0; t < T; ++t) tr_idx[t] = (int)tr64[t];
        F.id_idx.assign(L.n_id, 0);
        for (int k = 0; k < L.n_id; ++k) F.id_idx[k] = (int)id64[k];
    }
    F.in_idx = in_idx;
    F.tr_idx = tr_idx;
    F.ok = true;
    (void)st;
    return NFB_OK;
}

// ------------------------------------------------------------------------------------------
// fp16 operand planning.  The fused kernel multiplies fp16 hi/lo splits (11-bit mantissas: hi + lo carries
// 22-23 bits; the bf16 pairs used before carried 16-17 and cost rows of the 32-layer flagship 3e-4 in log_prob).
// fp16 has a narrow exponent range, so every operand is scaled by a power of two:
//   A operand of GEMM g  = true activation * u_row * 2^pa[g]      (u_row = 2^-e: per-row unit chosen in the kernel
//                                                                  from max |x_row|, so that |x| u_row < 1)
//   weights of GEMM g    = effective weight * 2^pw[g]
//   true GEMM output     = accumulator * 2^-(pa[g]+pw[g]) / u_row  (applied by the epilogue, exact)
// pa[g] comes from a GUARANTEED bound on the activation (infinity-norm chain below: no input can overflow fp16),
// pw[g] from max |w|.  GEMMs 0, 2, 4, ... accumulate onto the residual stream (in registers) and therefore share
// pa + pw.  For inputs that are post-ReLU (>= 0) the bound uses max(sum w+, sum w-) per row instead of sum |w|.
// Values far below the bound lose nothing that matters: fp16 subnormals keep the ABSOLUTE error at 2^-25 of the
// scaled range.  Validated offline against the fp64 oracle by tools/numerics_emul2.py (worst row of the 32-layer
// flagship: 3.1e-4 with bf16 pairs -> 5e-6, the reference's own fp32 error on that row).
// ------------------------------------------------------------------------------------------
int ceil_log2(double v) {
    if (!(v > 1e-30)) return -100;
    return (int)std::ceil(std::log2(v));
}
int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
float pow2f(int e) { return std::ldexp(1.0f, clampi(e, -120, 120)); }

// nm[g] = {inf-norm, non-negative-input norm, max |w|} of GEMM g (g = n_hidden: final layer); bmax[g] = max |bias|
// fold (optional): {inf-norm, -, max |w|} of the folded first matrix G = W0 E_lu (its input is z itself: |z| u_row < 1,
// A scale pinned to 2^14 because the LU stage reads the same operand) and max |b0 + W0 b_lu|.  The folded GEMM also
// accumulates onto the residual stream, so it joins the pa + pw = P constraint; *pw_fold < -100 on return = "do not fold"
// (its weights would have to be scaled down by more than 12 binades to meet P: the lo halves of the LARGEST weights would
// then fall below fp16's normal range and the pair would carry fewer than 22 bits; smaller weights only ever lose absolute
// precision of 2^-25 of the scaled range, like every other operand of this kernel).
void plan_scales(int n_hidden, const std::vector<float>& nm, const std::vector<float>& bmax, double b_in0,
                 int* pa, int* pw, const float* fold_nm = nullptr, float fold_bmax = 0.f, int* pw_fold = nullptr) {
    const int ng = n_hidden + 1;
    std::vector<double> bin(ng);
    auto norm_of = [&](int g) { return (double)((g >= 1 && g < n_hidden) ? nm[3 * g + 1] : nm[3 * g]); };
    bin[0] = b_in0;
    double Bh = norm_of(0) * b_in0 + bmax[0];
    if (fold_nm) Bh = std::max(Bh, (double)fold_nm[0] + fold_bmax);
    for (int g = 1; g + 1 < n_hidden; g += 2) {  // residual blocks: GEMMs (g, g + 1)
        bin[g] = Bh;
        const double Bt = norm_of(g) * Bh + bmax[g];
        bin[g + 1] = Bt;
        Bh += norm_of(g + 1) * Bt + bmax[g + 1];
    }
    bin[n_hidden] = Bh;
    for (int g = 0; g < ng; ++g) {
        pa[g] = clampi(14 - ceil_log2(bin[g]), -60, 14);
        pw[g] = clampi(13 - ceil_log2(nm[3 * g + 2]), -40, 40);
    }
    int P = 1 << 20;
    for (int g = 0; g < n_hidden; g += 2) P = std::min(P, pa[g] + pw[g]);
    int pwf = 0;
    if (fold_nm) {
        pwf = clampi(13 - ceil_log2(fold_nm[2]), -40, 40);
        P = std::min(P, 14 + pwf);
    }
    for (int g = 0; g < n_hidden; g += 2) {
        int d = pa[g] + pw[g] - P;
        const int dw = std::min(d, 8);  // the weight scale has ~10 binades of slack before w_lo goes subnormal
        pw[g] -= dw;
        pa[g] -= d - dw;
    }
    if (fold_nm && pw_fold) *pw_fold = (14 + pwf - P <= 12) ? P - 14 : -1000;
}

// (re)pack the weights/biases of a fused block from the live parameters
// Ufold: the LU layer in front of this block in the density direction (fused pair), or null.  When given (and the
// scale plan allows it) the first conditioner GEMM of the PAIR is packed as G = W0 E_lu[in_idx, :] so that it reads z
// itself: hidden GEMM 0 no longer waits for the LU stage and its epilogue (fused_rqs_kernel, `folded`).
int repack_fused(nfb_flow* f, Layer& L, cudaStream_t st, Layer* Ufold = nullptr) {
    FusedPack& F = L.fused;
    if (!F.ok) return NFB_OK;
    F.fold_ok = false;
    static const bool no_fold = getenv("NFB_NO_FOLD") != nullptr;
    if (no_fold || !F.pair_ok) Ufold = nullptr;
    const NetDesc& n = L.net;
    // every GEMM's effective matrix gets its own region of the scratch buffer: built once, normed, and (after the scale
    // plan) packed from there -- the second build of round 2a is gone
    size_t etot = 0, emax = 0;
    std::vector<size_t> eoff;
    for (auto& g : F.gemms) {
        eoff.push_back(etot);
        etot += (size_t)g.n_pad * g.k_pad;
        emax = std::max(emax, (size_t)g.n_pad * g.k_pad);
    }
    NFB_TRY(f->E.reserve((etot + emax) * sizeof(float)));
    float* const Escratch = f->E.as<float>() + etot;   // (fold: raw first matrix)
    const int ng = (int)F.gemms.size();
    NFB_CHECK(ng == F.n_hidden + 1 && ng <= 9, NFB_ERR_STATE, "fused pack: unexpected GEMM count %d", ng);
    // pass 1: norms of every effective matrix (for the fp16 scale plan)
    NFB_TRY(f->norms.reserve((size_t)(ng + 1) * 3 * sizeof(float)));
    for (int gi = 0; gi < ng; ++gi) {
        auto& g = F.gemms[gi];
        NFB_TRY(launch_build_effective(g.W, g.M, g.src_cols, g.src_row.as<int>(), g.src_col.as<int>(),
                                       g.row_scale.p ? g.row_scale.as<float>() : nullptr, f->E.as<float>() + eoff[gi],
                                       g.n_pad, g.k_pad, acc_gain(3 * g.k_pad / 16), st));
        NFB_TRY(launch_matrix_norms(f->E.as<float>() + eoff[gi], g.n_pad, g.k_pad, f->norms.as<float>() + 3 * gi, st));
    }
    // LU fold, device part (before the one synchronisation of this function): G = gain * E0 E_lu[in_idx, :],
    // delta = E0 b_lu[in_idx] (fp64 accumulation), norms of G
    if (Ufold) {
        auto& g0 = F.gemms[0];
        const int Hf = n.H;
        NFB_TRY(F.fold_lu.reserve(64 * 64 * 4));
        NFB_TRY(F.fold_G.reserve((size_t)Hf * 64 * 4));
        NFB_TRY(F.fold_delta.reserve((size_t)Hf * 4));
        NFB_TRY(launch_build_effective(g0.W, g0.M, g0.src_cols, g0.src_row.as<int>(), g0.src_col.as<int>(), nullptr,
                                       Escratch, Hf, 64, 1.f, st));
        NFB_TRY(launch_build_effective(Ufold->lu_Wd.as<float>(), nullptr, Ufold->D, F.lu_src_row.as<int>(),
                                       F.lu_src_col.as<int>(), nullptr, F.fold_lu.as<float>(), 64, 64, 1.f, st));
        NFB_TRY(launch_fold_lu(Escratch, F.fold_lu.as<float>(), Ufold->lu.bias, F.in_idx_dev.as<int>(), Hf,
                               Ufold->D, acc_gain(3 * 64 / 16), F.fold_G.as<float>(), F.fold_delta.as<float>(), st));
        NFB_TRY(launch_matrix_norms(F.fold_G.as<float>(), Hf, 64, f->norms.as<float>() + 3 * ng, st));
    }
    // every small read of this layer (norms, biases, fold results, final-layer bias, unconditional spline tables) is
    // queued into the pinned staging buffer and waited for ONCE
    const int H = n.H;
    StagedReads& R = f->reads;
    NFB_TRY(R.reserve((size_t)(ng + 1) * 3 + (size_t)(2 + 2 * n.nb) * H + (size_t)n.out + (size_t)L.n_id * 23 + 64));
    R.reset();
    size_t o_nm, o_b0, o_fnm = 0, o_fd = 0, o_bf, o_uw = 0, o_uh = 0, o_ud = 0;
    std::vector<size_t> o_bb(2 * n.nb);
    NFB_TRY(R.add(f->norms.as<float>(), (size_t)ng * 3, st, &o_nm));
    NFB_TRY(R.add(n.b0, (size_t)H, st, &o_b0));
    for (int i = 0; i < 2 * n.nb; ++i) NFB_TRY(R.add(n.bb[i], (size_t)H, st, &o_bb[i]));
    if (Ufold) {
        NFB_TRY(R.add(f->norms.as<float>() + 3 * ng, 3, st, &o_fnm));
        NFB_TRY(R.add(F.fold_delta.as<float>(), (size_t)H, st, &o_fd));
    }
    NFB_TRY(R.add(n.bf, (size_t)n.out, st, &o_bf));
    if (L.kind == L_COUPLED_RQS) {
        NFB_TRY(R.add(L.uw, (size_t)L.n_id * 8, st, &o_uw));
        NFB_TRY(R.add(L.uh, (size_t)L.n_id * 8, st, &o_uh));
        NFB_TRY(R.add(L.ud, (size_t)L.n_id * 7, st, &o_ud));
    }
    NFB_TRY(R.run(st));
    std::vector<float> nm;
    R.get(o_nm, (size_t)ng * 3, nm);
    std::vector<float> bh((size_t)F.n_hidden * 256, 0.f), b0, tmp;
    R.get(o_b0, (size_t)H, b0);
    std::vector<float> bmax(ng, 0.f);
    auto amax = [](const std::vector<float>& v) { float m = 0.f; for (float x : v) m = std::max(m, std::fabs(x)); return m; };
    bmax[0] = amax(b0);
    const std::vector<int>& hp = F.hperm;  // bias index i <-> original hidden unit hp[i]
    std::vector<float> cum = b0;
    for (int j = 0; j < H; ++j) bh[j] = b0[hp[j]];
    for (int b = 0; b < n.nb; ++b) {
        R.get(o_bb[2 * b], (size_t)H, tmp);
        bmax[1 + 2 * b] = amax(tmp);
        for (int j = 0; j < H; ++j) bh[(size_t)(1 + 2 * b) * 256 + j] = tmp[hp[j]];
        R.get(o_bb[2 * b + 1], (size_t)H, tmp);
        bmax[2 + 2 * b] = amax(tmp);
        for (int j = 0; j < H; ++j) cum[j] += tmp[j];
        for (int j = 0; j < H; ++j) bh[(size_t)(2 + 2 * b) * 256 + j] = cum[hp[j]];
    }
    F.bias_h = bh;
    // LU fold, host part: norms of G and the bias shift
    std::vector<float> fold_nm;
    float fold_bmax = 0.f;
    if (Ufold) {
        R.get(o_fnm, 3, fold_nm);
        R.get(o_fd, (size_t)H, F.fold_delta_host);
        for (int j = 0; j < H; ++j) fold_bmax = std::max(fold_bmax, std::fabs(bh[j] + F.fold_delta_host[j]));
    }
    // pass 2: scale plan, then the fp16 records
    plan_scales(F.n_hidden, nm, bmax, F.b_in0, F.pa, F.pw, Ufold ? fold_nm.data() : nullptr, fold_bmax, &F.pw_fold);
    if (getenv("NFB_DEBUG_PACK"))
        fprintf(stderr, "[nfb pack] fold: U=%p pair_ok=%d pw_fold=%d pa0=%d pw0=%d\n", (void*)Ufold, (int)F.pair_ok, F.pw_fold, F.pa[0], F.pw[0]);
    for (auto& g : F.gemms) {
        if (g.recs_dev.p == nullptr && !g.recs.empty()) {   // the record table of a GEMM is static: uploaded once
            std::vector<PackRec> tab;
            for (auto& r : g.recs) {
                tab.push_back(PackRec{r.row0, r.nrows, r.kc, 0, (unsigned long long)r.off_hi, (unsigned long long)r.off_lo});
                g.max_rows = std::max(g.max_rows, r.nrows);
            }
            NFB_TRY(g.recs_dev.upload(tab));
        }
    }
    if (Ufold && F.pw_fold > -100) {   // the folded matrix takes the place of GEMM 0: same records (build_fused)
        auto& g0 = F.gemms[0];
        NFB_TRY(F.fold_recs.reserve((size_t)H * 256));
        NFB_TRY(launch_pack_records(F.fold_G.as<float>(), 64, g0.recs_dev.as<PackRec>(), (int)g0.recs.size(), g0.max_rows,
                                    pow2f(F.pw_fold), F.fold_recs.as<uint8_t>(), st));
        F.fold_ok = true;
    }
    for (int gi = 0; gi < ng; ++gi) {
        auto& g = F.gemms[gi];
        NFB_TRY(launch_pack_records(f->E.as<float>() + eoff[gi], g.k_pad, g.recs_dev.as<PackRec>(), (int)g.recs.size(), g.max_rows,
                                    pow2f(F.pw[gi]), F.wstream.as<uint8_t>(), st));
    }
    const int crow = F.F * 24;
    std::vector<float> bfin, bf((size_t)F.n_chunks * crow, 0.f);
    R.get(o_bf, (size_t)n.out, bfin);
    for (int i = 0; i < F.n_chunks * crow; ++i) {
        const int t = F.F * (i / crow) + (i % crow) / 24, q = (i % crow) % 24;
        if (t < F.T && q < 23) bf[i] = bfin[t * 23 + q] * ((q < 16) ? L.wh_scale * kLog2eHost : 1.f);
    }
    F.bias_f = bf;
    if (L.kind == L_COUPLED_RQS) {
        std::vector<float> w, h, d, tab((size_t)L.n_id * 23);
        R.get(o_uw, (size_t)L.n_id * 8, w);
        R.get(o_uh, (size_t)L.n_id * 8, h);
        R.get(o_ud, (size_t)L.n_id * 7, d);
        for (int i = 0; i < L.n_id; ++i) {
            for (int k = 0; k < 8; ++k) { tab[i * 23 + k] = w[i * 8 + k]; tab[i * 23 + 8 + k] = h[i * 8 + k]; }
            for (int k = 0; k < 7; ++k) tab[i * 23 + 16 + k] = d[i * 7 + k];
        }
        NFB_TRY(F.uncond.upload(tab));
    }
    FusedLayer& Lh = F.host_layer;
    memset(&Lh, 0, sizeof(Lh));
    Lh.D = F.D; Lh.H = F.H; Lh.n_hidden = F.n_hidden; Lh.has_lu = 0; Lh.T = F.T; Lh.F = F.F;
    Lh.n_chunks = F.n_chunks; Lh.n_id = F.n_id; Lh.n_steps = F.n_steps; Lh.tail = F.tail;
    Lh.wstream = F.wstream.as<uint8_t>(); Lh.steps = F.steps.as<FusedStep>();
    Lh.uncond = F.uncond.as<float>();
    for (int k = 0; k < 64; ++k) {
        Lh.in_idx[k] = (signed char)(k < (int)F.in_idx.size() ? F.in_idx[k] : -1);
        Lh.tr_idx[k] = (unsigned char)(k < (int)F.tr_idx.size() ? F.tr_idx[k] : 0);
        Lh.id_idx[k] = (unsigned char)(k < (int)F.id_idx.size() ? F.id_idx[k] : 0);
    }
    Lh.a_sc[0] = 1.f; Lh.a_inv[0] = 1.f;
    for (int gi = 0; gi < ng; ++gi) {
        Lh.a_sc[1 + gi] = pow2f(F.pa[gi]);
        Lh.a_inv[1 + gi] = pow2f(-(F.pa[gi] + F.pw[gi]));
    }
    memcpy(Lh.bias_h, F.bias_h.data(), std::min(sizeof(Lh.bias_h), F.bias_h.size() * sizeof(float)));
    memcpy(Lh.bias_f, F.bias_f.data(), std::min(sizeof(Lh.bias_f), F.bias_f.size() * sizeof(float)));
    // The per-layer device images (layer alone, layer alone in the sampling direction, LU + layer pair) serve single-layer
    // launches only; the whole-stack launches read the arrays nfb_flow_repack uploads.  They are refreshed on first use
    // (upload_layer_images) instead of three blocking 18 KB copies per layer and optimizer step.
    F.ar_passes_fwd = L.kind == L_AR_RQS ? L.D : 0;
    F.images_dirty = true;
    return NFB_OK;
}

int upload_layer_images(FusedPack& F) {
    if (!F.images_dirty) return NFB_OK;
    NFB_TRY(F.layer_dev.reserve(sizeof(FusedLayer)));
    NFB_CUDA(cudaMemcpy(F.layer_dev.p, &F.host_layer, sizeof(FusedLayer), cudaMemcpyHostToDevice));
    FusedLayer Lf = F.host_layer;   // sampling-direction image of the block alone: the autoregressive block iterates D passes
    Lf.ar_passes = F.ar_passes_fwd;
    NFB_TRY(F.layer_fwd_dev.reserve(sizeof(FusedLayer)));
    NFB_CUDA(cudaMemcpy(F.layer_fwd_dev.p, &Lf, sizeof(FusedLayer), cudaMemcpyHostToDevice));
    if (F.pair_ok) {
        NFB_TRY(F.pair_dev.reserve(sizeof(FusedLayer)));
        NFB_CUDA(cudaMemcpy(F.pair_dev.p, &F.host_pair, sizeof(FusedLayer), cudaMemcpyHostToDevice));
    }
    F.images_dirty = false;
    return NFB_OK;
}

// LU layer pack (generic + the pieces the fused pair needs)
int repack_lu(nfb_flow* f, Layer& L, cudaStream_t st, bool packed_already = false) {
    const int n = L.D;
    NFB_TRY(L.lu_Wd.reserve((size_t)n * n * 4));
    NFB_TRY(L.lu_Ws.reserve((size_t)n * n * 4));
    NFB_TRY(L.lu_logdet.reserve(4));
    if (!packed_already)   // (nfb_flow_repack forms W, W^-1 and the log-det of ALL LU layers in one batched launch)
        NFB_TRY(launch_lu_pack(L.lu.lower_entries, L.lu.upper_entries, L.lu.unconstrained_upper_diag,
                               L.lu.eps, n, L.lu_Wd.as<float>(), L.lu_Ws.as<float>(),
                               L.lu_logdet.as<float>(), st));
    // sampling direction: x = (z - b) Winv^T = z Winv^T + bs with bs = -Winv b (tiny; host side).  The norms for the fp16
    // scale plan of the fused units this map is part of (row/column permutations leave them unchanged) are launched
    // first; everything the host needs comes back through the staged reads with ONE synchronisation.
    NFB_TRY(f->norms.reserve(64));
    NFB_TRY(launch_matrix_norms(L.lu_Wd.as<float>(), n, n, f->norms.as<float>(), st));
    NFB_TRY(launch_matrix_norms(L.lu_Ws.as<float>(), n, n, f->norms.as<float>() + 4, st));
    StagedReads& R = f->reads;
    NFB_TRY(R.reserve((size_t)n * n + n + 16));
    R.reset();
    size_t o_w, o_b, o_nm, o_ld;
    NFB_TRY(R.add(L.lu_Ws.as<float>(), (size_t)n * n, st, &o_w));
    NFB_TRY(R.add(L.lu.bias, (size_t)n, st, &o_b));
    NFB_TRY(R.add(f->norms.as<float>(), 8, st, &o_nm));
    NFB_TRY(R.add(L.lu_logdet.as<float>(), 1, st, &o_ld));
    NFB_TRY(R.run(st));
    std::vector<float> winv, b, bs(n), nm, ld;
    R.get(o_w, (size_t)n * n, winv);
    R.get(o_b, (size_t)n, b);
    R.get(o_nm, 8, nm);
    R.get(o_ld, 1, ld);
    for (int i = 0; i < n; ++i) {
        double acc = 0.0;
        for (int k = 0; k < n; ++k) acc += (double)winv[(size_t)i * n + k] * b[k];
        bs[i] = (float)(-acc);
    }
    NFB_TRY(L.lu_bs.upload(bs));
    L.lu_bs_host = bs;
    L.lu_norm_d = nm[0]; L.lu_max_d = nm[2]; L.lu_norm_s = nm[4]; L.lu_max_s = nm[6];
    L.lu_bmax_d = 0.f; L.lu_bmax_s = 0.f;
    for (int i = 0; i < n; ++i) { L.lu_bmax_d = std::max(L.lu_bmax_d, std::fabs(b[i])); L.lu_bmax_s = std::max(L.lu_bmax_s, std::fabs(bs[i])); }
    L.lu_bias_host = b;
    ld[0] = -ld[0];
    NFB_TRY(L.lu_logdet_neg.upload(ld));
    return NFB_OK;
}

// the LU map in front of a block: one 64-row record W_hi | W_lo, all four products (the map transforms z itself, ~2^-22)
FusedStep lu_step() {
    FusedStep s{};
    s.bytes16 = 64 * 16; s.n8 = 8; s.kc = 0; s.flags = kStepFirst | kStepLast | kStepQuad | kStepSkip1;
    return s;
}

int build_pair(nfb_flow* f, Layer& R, Layer& U, cudaStream_t st) {
    FusedPack& F = R.fused;
    F.pair_ok = false;
    if (!F.ok || U.D != R.D || U.D > 64) return NFB_OK;
    std::vector<FusedStep> steps(1, lu_step());
    steps.insert(steps.end(), F.steps_host.begin(), F.steps_host.end());
    F.pair_steps = (int)steps.size();
    NFB_TRY(F.pair_steps_dev.upload(steps));
    NFB_TRY(F.in_idx_dev.upload(F.in_idx));   // (LU fold, repack_fused)
    NFB_TRY(F.pair_wstream.reserve(2 * 8192 + F.rqs_bytes));
    std::vector<int> sr(64), sc(64, -1);
    for (int i = 0; i < 64; ++i) sr[i] = i < U.D ? i : -1;
    for (int j = 0; j < U.D; ++j) sc[U.perm_host[j]] = j;  // E[i, perm[j]] = W[i, j]
    NFB_TRY(F.lu_src_row.upload(sr));
    NFB_TRY(F.lu_src_col.upload(sc));
    F.pair_ok = true;
    (void)f; (void)st;
    return NFB_OK;
}

int repack_pair(nfb_flow* f, Layer& R, Layer& U, cudaStream_t st) {
    FusedPack& F = R.fused;
    if (!F.pair_ok) return NFB_OK;
    NFB_TRY(f->E.reserve(64 * 64 * 4));
    const int pw_lu = clampi(13 - ceil_log2(U.lu_max_d), -40, 40);
    NFB_TRY(launch_build_effective(U.lu_Wd.as<float>(), nullptr, U.D, F.lu_src_row.as<int>(),
                                   F.lu_src_col.as<int>(), nullptr, f->E.as<float>(), 64, 64, acc_gain(4 * 4), st));
    NFB_TRY(launch_swizzle_split(f->E.as<float>(), 64, 64, 64, 2, pow2f(pw_lu), F.pair_wstream.as<uint8_t>(), st));
    NFB_CUDA(cudaMemcpyAsync(F.pair_wstream.as<uint8_t>() + 2 * 8192, F.wstream.p, F.rqs_bytes,
                             cudaMemcpyDeviceToDevice, st));
    std::vector<float> bl(64, 0.f);
    for (int i = 0; i < U.D; ++i) bl[i] = U.lu_bias_host[i];   // (read back by repack_lu in this same repack)
    NFB_TRY(F.bias_lu.upload(bl));
    FusedLayer& Lp = F.host_pair;
    Lp = F.host_layer;
    Lp.has_lu = 1;
    Lp.a_sc[0] = pow2f(14);  // |z| u_row < 1
    Lp.a_inv[0] = pow2f(-(14 + pw_lu));
    Lp.n_steps = F.pair_steps;
    Lp.wstream = F.pair_wstream.as<uint8_t>();
    Lp.steps = F.pair_steps_dev.as<FusedStep>();
    if (F.fold_ok) {
        // the block's first two records (GEMM 0, K-chunk 0, all H rows) are replaced by the folded matrix
        NFB_CUDA(cudaMemcpyAsync(F.pair_wstream.as<uint8_t>() + 2 * 8192, F.fold_recs.p, (size_t)F.H * 256,
                                 cudaMemcpyDeviceToDevice, st));   // (stream-ordered after the copy of the block's records)
        Lp.fold_lu = 1;
        for (int ph = 0; ph < F.n_hidden; ph += 2)   // b0 (+ W0 b_lu) is part of every pre-summed residual bias
            for (int j = 0; j < F.H; ++j) Lp.bias_h[ph * 256 + j] += F.fold_delta_host[j];
    }
    Lp.bias_lu = F.bias_lu.as<float>();
    Lp.lu_logdet = U.lu_logdet.as<float>();
    F.images_dirty = true;   // (pair_dev is refreshed by upload_layer_images on first single-pair launch)
    return NFB_OK;
}

// Sampling direction.  Unit = [inverse LU map of layer U (or none) + coupling block R with its splines inverted].
// x = ((z - b) Winv^T)[:, inv_perm]  (LULinearPermute.forward, flows/mixing.py:551-556: linear.inverse, then
// permutation.inverse), i.e. one dense map E z + e with E[i, :] = Winv[inv_perm[i], :], e[i] = bs[inv_perm[i]];
// Winv = (L U)^-1 is formed in fp64 by lu_pack_kernel (the reference solves two triangular systems in fp32).
int build_fwd_unit(nfb_flow* f, Layer& R, Layer* U) {
    FusedPack& F = R.fused;
    F.fwd_ok = false;
    if (!F.ok || (R.kind != L_COUPLED_RQS && R.kind != L_AR_RQS)) return NFB_OK;
    if (!U) { F.fwd_ok = true; return NFB_OK; }  // first block of the stack: no LU in front of it
    if (U->D != R.D || U->D > 64) return NFB_OK;
    std::vector<FusedStep> steps(1, lu_step());
    steps.insert(steps.end(), F.steps_host.begin(), F.steps_host.end());
    NFB_TRY(F.fwd_steps_dev.upload(steps));
    NFB_TRY(F.fwd_wstream.reserve(2 * 8192 + F.rqs_bytes));
    std::vector<int> sr(64, -1), sc(64, -1);
    for (int i = 0; i < U->D; ++i) { sr[i] = U->inv_perm_host[i]; sc[i] = i; }
    NFB_TRY(F.fwd_src_row.upload(sr));
    NFB_TRY(F.fwd_src_col.upload(sc));
    F.fwd_ok = true;
    (void)f;
    return NFB_OK;
}

int repack_fwd_unit(nfb_flow* f, Layer& R, Layer* U, cudaStream_t st) {
    FusedPack& F = R.fused;
    FusedLayer& Lp = F.host_fwd;
    Lp = F.host_layer;
    Lp.ar_passes = R.kind == L_AR_RQS ? R.D : 0;  // autoregressive block: D conditioner passes inside the unit
    if (!U) return NFB_OK;  // spline block alone: the density descriptor (+ ar_passes) serves
    NFB_TRY(f->E.reserve(64 * 64 * 4));
    const int pw_lu = clampi(13 - ceil_log2(U->lu_max_s), -40, 40);
    NFB_TRY(launch_build_effective(U->lu_Ws.as<float>(), nullptr, U->D, F.fwd_src_row.as<int>(),
                                   F.fwd_src_col.as<int>(), nullptr, f->E.as<float>(), 64, 64, acc_gain(4 * 4), st));
    NFB_TRY(launch_swizzle_split(f->E.as<float>(), 64, 64, 64, 2, pow2f(pw_lu), F.fwd_wstream.as<uint8_t>(), st));
    NFB_CUDA(cudaMemcpyAsync(F.fwd_wstream.as<uint8_t>() + 2 * 8192, F.wstream.p, F.rqs_bytes,
                             cudaMemcpyDeviceToDevice, st));
    std::vector<float> bl(64, 0.f);
    for (int i = 0; i < U->D; ++i) bl[i] = U->lu_bs_host[U->inv_perm_host[i]];
    NFB_TRY(F.fwd_bias_lu.upload(bl));
    Lp.has_lu = 1;
    Lp.a_sc[0] = pow2f(14);
    Lp.a_inv[0] = pow2f(-(14 + pw_lu));
    Lp.n_steps = F.n_steps + 1;
    Lp.wstream = F.fwd_wstream.as<uint8_t>();
    Lp.steps = F.fwd_steps_dev.as<FusedStep>();
    Lp.bias_lu = F.fwd_bias_lu.as<float>();
    Lp.lu_logdet = U->lu_logdet_neg.as<float>();
    return NFB_OK;
}

int launch_fused_layer(nfb_flow* f, Layer& R, Layer* U, const float* zin, float* zout, float* logq,
                       long long rows, int accumulate, cudaStream_t st, int sample = 0) {
    FusedPack& F = R.fused;
    NFB_TRY(upload_layer_images(F));
    FusedParams p{};
    p.layers = U ? F.pair_dev.as<FusedLayer>() : (sample ? F.layer_fwd_dev.as<FusedLayer>() : F.layer_dev.as<FusedLayer>());
    p.n_layers = 1;
    p.zin = zin; p.zout = zout; p.logq = logq; p.rows = rows; p.accumulate = accumulate;
    p.progress = nullptr;
    p.err = f->err.as<int>();
    NFB_TRY(launch_fused_rqs(p, f->sm_count, sample, st));
    f->launches++;
    return NFB_OK;
}

// Whole stack in ONE persistent launch: (layer, tile) work units with per-tile progress flags.  logq must be
// pre-filled (accumulate semantics); zout may alias zin.
int launch_fused_stack(nfb_flow* f, const float* zin, float* zout, float* logq, long long rows, cudaStream_t st,
                       int sample = 0, long long z_stride = 0) {
    const long long n_tiles = (rows + kFusedTileRows - 1) / kFusedTileRows;
    NFB_TRY(f->progress.reserve((size_t)(n_tiles + 1) * sizeof(int)));   // + the unit ticket counter
    NFB_CUDA(cudaMemsetAsync(f->progress.p, 0, (size_t)(n_tiles + 1) * sizeof(int), st));
    FusedParams p{};
    p.layers = sample ? f->fwd_layers.as<FusedLayer>() : f->stack_layers.as<FusedLayer>();
    p.n_layers = sample ? f->fwd_n : f->stack_n;
    p.zin = zin; p.zout = zout; p.logq = logq; p.rows = rows; p.accumulate = 1; p.z_stride = z_stride;
    p.progress = f->progress.as<int>();
    p.ticket = getenv("NFB_STATIC_UNITS") ? nullptr : f->progress.as<int>() + n_tiles;
    p.in_ready = sample ? nullptr : f->cur_in_ready;
    f->cur_in_ready = nullptr;  // consumed (or not applicable): later launches must not wait on it
    if (p.in_ready && p.ticket && p.n_layers > 1 && p.n_layers <= 255 && n_tiles >= 64 && z_stride == 0 &&
        getenv("NFB_NO_WAVE_ORDER") == nullptr) {
        // host batch in flight: diagonal (layer, tile group) order, groups in arrival order (fused_rqs_kernel `decode`)
        const int tpg = (int)((n_tiles + 7) / 8);
        const int G = (int)((n_tiles + tpg - 1) / tpg);   // (<= 8 groups, the last one possibly short, none empty)
        if (f->wave_layers != p.n_layers || f->wave_tiles != n_tiles) {
            std::vector<unsigned int> tab;
            unsigned int start = 0;
            for (int d = 0; d < p.n_layers + G - 1; ++d)
                for (int g = 0; g < G; ++g) {
                    const int l = d - g;
                    if (l < 0 || l >= p.n_layers) continue;
                    tab.push_back((unsigned int)(l | (g << 8)));
                    tab.push_back(start);
                    start += (unsigned int)std::min<long long>(tpg, n_tiles - (long long)g * tpg);
                }
            NFB_TRY(f->wave_order.upload(tab));
            f->wave_layers = p.n_layers;
            f->wave_tiles = n_tiles;
        }
        p.wave_order = f->wave_order.as<unsigned int>();
        p.wave_elems = p.n_layers * G;
        p.wave_tpg = tpg;
    }
    p.err = f->err.as<int>();
    NFB_TRY(launch_fused_rqs(p, f->sm_count, sample, st));
    f->launches += 2;  // memset + kernel
    return NFB_OK;
}

// ------------------------------------------------------------------------------------------
// per-layer generic application.  zin != zout.  logdet: [rows], accumulate semantic.
// ------------------------------------------------------------------------------------------
int zero_if(nfb_flow* f, float* logdet, long long rows, int accumulate, cudaStream_t st) {
    if (logdet && !accumulate) { NFB_TRY(launch_fill(logdet, rows, 0.f, st)); f->launches++; }
    return NFB_OK;
}

int apply_layer_generic(nfb_flow* f, Layer& L, int direction, const float* zin, float* zout,
                        float* logdet, long long rows, int accumulate, cudaStream_t st) {
    const int D = L.D;
    switch (L.kind) {
    case L_AR_RQS: {
        const int P = 3 * L.K - 1;
        NFB_TRY(f->params.reserve((size_t)rows * D * P * 4));
        NFB_TRY(zero_if(f, logdet, rows, accumulate, st));
        if (direction == NFB_INVERSE) {  // affine/autoregressive.py:24-27: one MADE pass
            NFB_TRY(run_net_generic(f, L.net, L.pack, zin, D, nullptr, rows, f->params.as<float>(), st));
            NFB_TRY(launch_rqs_rows(zin, f->params.as<float>(), zout, logdet, rows, D, D, nullptr, L.K,
                                    L.tail, 1.f, 0, st));
            f->launches++;
        } else {  // affine/autoregressive.py:29-38: D MADE passes, spline inverse
            NFB_TRY(f->ar_tmp.reserve((size_t)rows * D * 4));
            float* out = f->ar_tmp.as<float>();
            NFB_TRY(launch_fill(out, rows * D, 0.f, st));
            f->launches++;
            for (int i = 0; i < D; ++i) {
                NFB_TRY(run_net_generic(f, L.net, L.pack, out, D, nullptr, rows, f->params.as<float>(), st));
                const bool last = (i == D - 1);
                NFB_TRY(launch_rqs_rows(zin, f->params.as<float>(), last ? zout : out, last ? logdet : nullptr,
                                        rows, D, D, nullptr, L.K, L.tail, 1.f, 1, st));
                f->launches++;
            }
        }
        return NFB_OK;
    }
    case L_COUPLED_RQS: {
        const int P = 3 * L.K - 1;
        NFB_TRY(f->params.reserve((size_t)rows * L.n_tr * P * 4));
        NFB_TRY(zero_if(f, logdet, rows, accumulate, st));
        if (direction == NFB_INVERSE) {  // Coupling.forward, neural_spline/coupling.py:71-98
            NFB_TRY(run_net_generic(f, L.net, L.pack, zin, D, L.id_idx.as<int>(), rows, f->params.as<float>(), st));
            NFB_TRY(launch_rqs_rows(zin, f->params.as<float>(), zout, logdet, rows, L.n_tr, D,
                                    L.tr_idx.as<int>(), L.K, L.tail, L.wh_scale, 0, st));
            NFB_TRY(launch_rqs_shared(zin, L.uncond.as<float>(), zout, logdet, rows, L.n_id, D,
                                      L.id_idx.as<int>(), L.K, L.tail, 0, st));
            f->launches += 2;
        } else {  // Coupling.inverse, :100-128: unconditional inverse first, net sees its output
            NFB_TRY(launch_rqs_shared(zin, L.uncond.as<float>(), zout, logdet, rows, L.n_id, D,
                                      L.id_idx.as<int>(), L.K, L.tail, 1, st));
            NFB_TRY(run_net_generic(f, L.net, L.pack, zout, D, L.id_idx.as<int>(), rows, f->params.as<float>(), st));
            NFB_TRY(launch_rqs_rows(zin, f->params.as<float>(), zout, logdet, rows, L.n_tr, D,
                                    L.tr_idx.as<int>(), L.K, L.tail, L.wh_scale, 1, st));
            f->launches += 2;
        }
        return NFB_OK;
    }
    case L_LU: {
        if (direction == NFB_INVERSE) {  // mixing.py:560-563 -> :414-434
            NFB_TRY(launch_linear(zin, D, L.lu_perm.as<int>(), L.lu_Wd.as<float>(), L.lu.bias, nullptr, 0,
                                  zout, D, rows, D, D, 0, 0, 0.f, st));
        } else {  // mixing.py:555-558 -> :436-473 : (z - b) (LU)^-T, then inverse permutation
            NFB_TRY(f->hT.reserve((size_t)rows * D * 4));
            // t = z W^-T - (W^-1 b) == (z - b) W^-T ; bias term applied via a second tiny pass below
            NFB_TRY(launch_linear(zin, D, nullptr, L.lu_Ws.as<float>(), L.lu_bs.as<float>(), nullptr, 0,
                                  f->hT.as<float>(), D, rows, D, D, 0, 0, 0.f, st));
            NFB_TRY(launch_gather_cols(f->hT.as<float>(), zout, L.lu_tmp.as<int>(), rows, D, 1, st));
            f->launches++;
        }
        f->launches++;
        if (logdet) {
            NFB_TRY(zero_if(f, logdet, rows, accumulate, st));
            NFB_TRY(launch_add_scalar(logdet, rows, L.lu_logdet.as<float>(), direction == NFB_INVERSE ? 1.f : -1.f, st));
            f->launches++;
        }
        return NFB_OK;
    }
    default:
        break;
    }
    nfb_set_error("apply_layer_generic: layer kind %d not handled here", (int)L.kind);
    return NFB_ERR_STATE;
}

bool is_affine_kind(const Layer& L) {
    return L.kind == L_MASKED_AFFINE || L.kind == L_AFFINE_COUPLING || L.kind == L_AFFINE_CONST ||
           L.kind == L_PERMUTE;
}

int copy_mlp(const nfb_mlp_desc_t& d, AffMlp& m, float* slope) {
    NFB_CHECK(d.num_layers >= 0 && d.num_layers <= kAffMaxLayers, NFB_ERR_UNSUPPORTED, "MLP: %d layers > %d", d.num_layers, kAffMaxLayers);
    m.n_layers = d.num_layers;
    for (int i = 0; i <= d.num_layers; ++i) {
        NFB_CHECK(d.sizes[i] >= 1 && d.sizes[i] <= kAffMaxW, NFB_ERR_UNSUPPORTED, "MLP: layer width %d > %d", d.sizes[i], kAffMaxW);
        m.sizes[i] = d.sizes[i];
    }
    for (int i = 0; i < d.num_layers; ++i) {
        NFB_CHECK(d.w[i] && d.b[i], NFB_ERR_ARG, "MLP: null weight");
        m.w[i] = d.w[i]; m.b[i] = d.b[i];
    }
    if (d.num_layers) *slope = d.leaky;
    return NFB_OK;
}

cudaStream_t S(void* s) { return static_cast<cudaStream_t>(s); }

int ensure_ws(nfb_flow* f, long long rows) {
    NFB_TRY(f->zA.reserve((size_t)rows * f->D * 4));
    NFB_TRY(f->zB.reserve((size_t)rows * f->D * 4));
    NFB_TRY(f->logq.reserve((size_t)rows * 4));
    NFB_TRY(f->scratch_sum.reserve(1024 * 8));
    NFB_TRY(f->loss.reserve(16));
    return NFB_OK;
}

// Apply execution group g.  in/out must differ.  logdet accumulates (+=) -- caller zeroes first.
int run_group(nfb_flow* f, Group& g, int direction, const float* zin, float* zout, float* logdet,
              long long rows, cudaStream_t st) {
    switch (g.kind) {
    case G_FUSED_PAIR:
        if (direction == NFB_INVERSE)
            return launch_fused_layer(f, *f->layers[g.first], f->layers[g.last].get(), zin, zout, logdet, rows, 1, st);
        break;
    case G_FUSED:
        if (direction == NFB_INVERSE)
            return launch_fused_layer(f, *f->layers[g.first], nullptr, zin, zout, logdet, rows, 1, st);
        break;
    case G_AFFINE:
        NFB_TRY(launch_affine_stack(g.ops.p, g.last - g.first + 1, zin, zout, logdet, rows, f->D, 1, direction, st));
        f->launches++;
        return NFB_OK;
    case G_SINGLE:
        return apply_layer_generic(f, *f->layers[g.first], direction, zin, zout, logdet, rows, 1, st);
    }
    // fused groups in the sampling direction, layer by layer: a coupling block runs the fused kernel with its
    // splines inverted; the autoregressive block needs D sequential conditioner passes (generic kernels)
    auto fwd_block = [&](Layer& R, const float* in, float* out) -> int {
        if ((R.kind == L_COUPLED_RQS || R.kind == L_AR_RQS) && R.fused.ok)
            return launch_fused_layer(f, R, nullptr, in, out, logdet, rows, 1, st, 1);
        return apply_layer_generic(f, R, direction, in, out, logdet, rows, 1, st);
    };
    if (g.first == g.last) return fwd_block(*f->layers[g.first], zin, zout);
    // pair = [spline block (first), LU (last)] in list order; forward applies first then last
    NFB_TRY(f->pair_tmp.reserve((size_t)rows * f->D * 4));
    NFB_TRY(fwd_block(*f->layers[g.first], zin, f->pair_tmp.as<float>()));
    return apply_layer_generic(f, *f->layers[g.last], direction, f->pair_tmp.as<float>(), zout, logdet, rows, 1, st);
}

}  // namespace

// ==========================================================================================
// extern "C"
// ==========================================================================================
extern "C" {

int nfb_abi_version(void) { return NFB_ABI_VERSION; }
const char* nfb_last_error(void) { return g_err.c_str(); }

int nfb_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int dev = 0;
    NFB_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    NFB_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (sm_count) *sm_count = prop.multiProcessorCount;
    if (cc_major) *cc_major = prop.major;
    if (cc_minor) *cc_minor = prop.minor;
    return NFB_OK;
}

int nfb_rqs_spline(const float* x, const float* params, float* y, float* log_det, int64_t rows,
                   int32_t feats, int32_t num_bins, float tail_bound, float wh_scale, int32_t inverse,
                   int32_t accumulate, void* stream) {
    NFB_CHECK(x && params && y, NFB_ERR_ARG, "nfb_rqs_spline: null pointer");
    NFB_CHECK(rows >= 0 && feats >= 0, NFB_ERR_ARG, "nfb_rqs_spline: negative size");
    if (log_det && !accumulate) NFB_TRY(launch_fill(log_det, rows, 0.f, S(stream)));
    return launch_rqs_rows(x, params, y, log_det, rows, feats, feats, nullptr, num_bins, tail_bound,
                           wh_scale, inverse, S(stream));
}

int nfb_rqs_spline_tails(const float* x, const float* params, float* y, float* log_det, int64_t rows, int32_t feats,
                         int32_t num_bins, int32_t num_derivatives, const float* tail_bound, const int32_t* circular,
                         float wh_scale, int32_t inverse, int32_t accumulate, void* stream) {
    NFB_CHECK(x && params && y && tail_bound && circular, NFB_ERR_ARG, "nfb_rqs_spline_tails: null pointer");
    NFB_CHECK(rows >= 0 && feats >= 0, NFB_ERR_ARG, "nfb_rqs_spline_tails: negative size");
    if (log_det && !accumulate) NFB_TRY(launch_fill(log_det, rows, 0.f, S(stream)));
    return launch_rqs_rows_tails(x, params, y, log_det, rows, feats, num_bins, num_derivatives, tail_bound, circular,
                                 wh_scale, inverse, S(stream));
}
int nfb_periodic_features(const float* x, float* y, int64_t rows, int32_t dim, const int32_t* slot, const float* weights,
                          const float* scale, const float* bias, void* stream) {
    NFB_CHECK(x && y && slot && weights && scale, NFB_ERR_ARG, "nfb_periodic_features: null pointer");
    NFB_CHECK(rows >= 0 && dim >= 0, NFB_ERR_ARG, "nfb_periodic_features: negative size");
    return launch_periodic_features(x, y, rows, dim, slot, weights, scale, bias, S(stream));
}

int nfb_diag_gaussian_log_prob(const float* z, const float* loc, const float* log_scale, float* log_q,
                               int64_t rows, int32_t dim, int32_t accumulate, void* stream) {
    NFB_CHECK(z && loc && log_scale && log_q, NFB_ERR_ARG, "nfb_diag_gaussian_log_prob: null pointer");
    return launch_diag_gauss(z, loc, log_scale, log_q, rows, dim, accumulate, S(stream));
}

int nfb_conv2d(const float* x, int32_t x_channels, int32_t c0, const float* w, const float* b, float* y,
               int64_t batch, int32_t cin, int32_t height, int32_t width, int32_t cout, int32_t ksize,
               float leaky, void* stream) {
    NFB_CHECK(x && w && y, NFB_ERR_ARG, "nfb_conv2d: null pointer");
    return launch_conv2d(x, x_channels, c0, w, b, y, batch, cin, height, width, cout, ksize, leaky, S(stream));
}
static float glow_gain() {
    static const float gain = [] { const char* e = getenv("NFB_ACC_COMP_STEP"); return e ? (float)atof(e) : nfb::kAccStepGain; }();
    return gain;
}
static int glow_err_buf(int** out) {
    static thread_local int* err_dev = nullptr;
    if (!err_dev) { NFB_CUDA(cudaMalloc(reinterpret_cast<void**>(&err_dev), 16)); NFB_CUDA(cudaMemset(err_dev, 0, 16)); }
    *out = err_dev;
    return NFB_OK;
}
int nfb_glow_conditioner(const float* x, int32_t x_channels, int32_t c0, int32_t cin, const float* w1, const float* b1,
                         const float* w2, const float* b2, const float* w3_taps, float* y_taps, int64_t batch,
                         int32_t height, int32_t width, int32_t hidden, int32_t cout, float leaky, void* stream) {
    NFB_CHECK(x && w1 && b1 && w2 && b2 && w3_taps && y_taps, NFB_ERR_ARG, "nfb_glow_conditioner: null pointer");
    NFB_CHECK(glow_cond_supported(cin, hidden, cout, 3, 1, 3), NFB_ERR_UNSUPPORTED,
              "nfb_glow_conditioner: needs hidden %% 64 == 0 (<= 256), 9 cin <= 256, 9 cout <= 512");
    int* err_dev = nullptr;
    NFB_TRY(glow_err_buf(&err_dev));
    return launch_glow_conditioner(x, x_channels, c0, cin, w1, b1, w2, b2, w3_taps, nullptr, y_taps, batch, height, width,
                                   hidden, cout, leaky, glow_gain(), err_dev, S(stream));
}
int64_t nfb_glow_conditioner_packed_bytes(int32_t cin, int32_t hidden, int32_t cout) {
    if (!glow_cond_supported(cin, hidden, cout, 3, 1, 3)) return -1;
    return (int64_t)glow_cond_packed_bytes(cin, hidden, cout);
}
int nfb_glow_conditioner_pack(const float* w1, const float* w2, const float* w3_taps, int32_t cin, int32_t hidden,
                              int32_t cout, void* packed, void* stream) {
    NFB_CHECK(w1 && w2 && w3_taps && packed, NFB_ERR_ARG, "nfb_glow_conditioner_pack: null pointer");
    return launch_glow_cond_pack(w1, w2, w3_taps, cin, hidden, cout, glow_gain(), static_cast<uint8_t*>(packed), S(stream));
}
int nfb_glow_conditioner_packed(const float* x, int32_t x_channels, int32_t c0, int32_t cin, const void* packed,
                                const float* b1, const float* b2, float* y_taps, int64_t batch, int32_t height,
                                int32_t width, int32_t hidden, int32_t cout, float leaky, void* stream) {
    NFB_CHECK(x && packed && b1 && b2 && y_taps, NFB_ERR_ARG, "nfb_glow_conditioner_packed: null pointer");
    NFB_CHECK(glow_cond_supported(cin, hidden, cout, 3, 1, 3), NFB_ERR_UNSUPPORTED,
              "nfb_glow_conditioner_packed: needs hidden %% 64 == 0 (<= 256), 9 cin <= 256, 9 cout <= 512");
    int* err_dev = nullptr;
    NFB_TRY(glow_err_buf(&err_dev));
    return launch_glow_conditioner(x, x_channels, c0, cin, nullptr, b1, nullptr, b2, nullptr,
                                   static_cast<const uint8_t*>(packed), y_taps, batch, height, width, hidden, cout, leaky,
                                   glow_gain(), err_dev, S(stream));
}
// One GlowBlock in one call (flows/affine/glow.py:72-84), parameters prepared by the caller once per parameter version:
//   density  (NFB_INVERSE): z_out = conv1x1(z_in; w, b)   [ActNorm.inverse folded into Invertible1x1Conv.inverse], then the
//                            affine coupling in place on z_out, conditioner reading z_out's other half;
//   sampling (NFB_FORWARD): coupling on a copy of z_in (conditioner reads z_in), then z_out = conv1x1(copy; w, b).
int nfb_glow_block(const float* z_in, float* z_out, float* scratch, float* y_taps, float* log_det, const float* w1x1,
                   const float* b1x1, const float* logdet_const, const void* cond_packed, const float* cond_b1,
                   const float* cond_b2, const float* cond_b3, int64_t batch, int32_t channels, int32_t height,
                   int32_t width, int32_t hidden, int32_t scale, int32_t scale_map, int32_t split_mode, float leaky,
                   int32_t direction, void* stream) {
    NFB_CHECK(z_in && z_out && y_taps && log_det && w1x1 && b1x1 && cond_packed && cond_b1 && cond_b2, NFB_ERR_ARG,
              "nfb_glow_block: null pointer");
    NFB_CHECK(direction == NFB_INVERSE || scratch, NFB_ERR_ARG, "nfb_glow_block: the sampling direction needs a scratch tensor");
    NFB_CHECK(scale_map >= 0 && scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(split_mode == 0 || split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    const int C = channels, h = (C + 1) / 2;
    const int c0 = split_mode == 0 ? 0 : h, cin = split_mode == 0 ? h : C - h;   // conditioner input chunk
    const int n2 = C - cin, cout = (scale ? 2 : 1) * n2;
    NFB_CHECK(glow_cond_supported(cin, hidden, cout, 3, 1, 3) && coupling_taps_supported(C, height, width, scale),
              NFB_ERR_UNSUPPORTED, "nfb_glow_block: conditioner shape outside the fused kernels");
    cudaStream_t st = S(stream);
    int* err_dev = nullptr;
    NFB_TRY(glow_err_buf(&err_dev));
    const uint8_t* packed = static_cast<const uint8_t*>(cond_packed);
    if (direction == NFB_INVERSE) {
        NFB_TRY(launch_conv2d(z_in, C, 0, w1x1, b1x1, z_out, batch, C, height, width, C, 1, -1.f, st));
        NFB_TRY(launch_glow_conditioner(z_out, C, c0, cin, nullptr, cond_b1, nullptr, cond_b2, nullptr, packed, y_taps, batch,
                                        height, width, hidden, cout, leaky, glow_gain(), err_dev, st));
        return launch_coupling_taps(z_out, y_taps, cond_b3, log_det, logdet_const, batch, C, height, width, scale, scale_map,
                                    split_mode, direction, 0, st);
    }
    NFB_CUDA(cudaMemcpyAsync(scratch, z_in, (size_t)batch * C * height * width * sizeof(float), cudaMemcpyDeviceToDevice, st));
    NFB_TRY(launch_glow_conditioner(z_in, C, c0, cin, nullptr, cond_b1, nullptr, cond_b2, nullptr, packed, y_taps, batch,
                                    height, width, hidden, cout, leaky, glow_gain(), err_dev, st));
    NFB_TRY(launch_coupling_taps(scratch, y_taps, cond_b3, log_det, logdet_const, batch, C, height, width, scale, scale_map,
                                 split_mode, direction, 0, st));
    return launch_conv2d(scratch, C, 0, w1x1, b1x1, z_out, batch, C, height, width, C, 1, -1.f, st);
}
int nfb_tap_shift_add(const float* y_taps, const float* bias, float* out, int64_t batch, int32_t cout, int32_t height,
                      int32_t width, int32_t ksize, void* stream) {
    NFB_CHECK(y_taps && out, NFB_ERR_ARG, "nfb_tap_shift_add: null pointer");
    NFB_CHECK(ksize >= 1 && (ksize & 1), NFB_ERR_ARG, "nfb_tap_shift_add: odd kernel sizes only");
    return launch_tap_shift_add(y_taps, bias, out, batch, cout, height, width, ksize, S(stream));
}
int nfb_glow_fold_actnorm_conv1x1(const float* P, const float* L, const float* U, const float* sign_S,
                                  const float* log_S, const float* s, const float* t, int32_t channels,
                                  int32_t hw, float* w_out, float* b_out, float* logdet_out, void* stream) {
    NFB_CHECK(P && L && U && sign_S && log_S && s && t && w_out && b_out && logdet_out, NFB_ERR_ARG,
              "nfb_glow_fold_actnorm_conv1x1: null pointer");
    return launch_glow_fold(P, L, U, sign_S, log_S, s, t, channels, hw, w_out, b_out, logdet_out, S(stream));
}
int nfb_glow_fold_conv1x1_actnorm_forward(const float* P, const float* L, const float* U, const float* sign_S,
                                          const float* log_S, const float* s, const float* t, int32_t channels,
                                          int32_t hw, float* w_out, float* b_out, float* logdet_out, void* stream) {
    NFB_CHECK(P && L && U && sign_S && log_S && s && t && w_out && b_out && logdet_out, NFB_ERR_ARG,
              "nfb_glow_fold_conv1x1_actnorm_forward: null pointer");
    return launch_glow_fold_fwd(P, L, U, sign_S, log_S, s, t, channels, hw, w_out, b_out, logdet_out, S(stream));
}
int nfb_paste_channels(const float* in, float* out, int64_t batch, int32_t channels, int32_t c0, int32_t n,
                       int32_t hw, void* stream) {
    NFB_CHECK(in && out, NFB_ERR_ARG, "nfb_paste_channels: null pointer");
    return launch_paste_channels(in, out, batch, channels, c0, n, hw, S(stream));
}
int nfb_affine_coupling_image(float* z, const float* param, float* log_det, const float* logdet_const,
                              int64_t batch, int32_t channels, int32_t hw, int32_t scale, int32_t scale_map,
                              int32_t split_mode, int32_t direction, int32_t accumulate, void* stream) {
    NFB_CHECK(z && param, NFB_ERR_ARG, "nfb_affine_coupling_image: null pointer");
    NFB_CHECK(scale_map >= 0 && scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(split_mode == 0 || split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    return launch_coupling_image(z, param, log_det, logdet_const, batch, channels, hw, scale, scale_map,
                                 split_mode, direction, accumulate, S(stream));
}
int nfb_affine_coupling_image_taps(float* z, const float* y_taps, const float* bias, float* log_det,
                                   const float* logdet_const, int64_t batch, int32_t channels, int32_t height,
                                   int32_t width, int32_t scale, int32_t scale_map, int32_t split_mode, int32_t direction,
                                   int32_t accumulate, void* stream) {
    NFB_CHECK(z && y_taps, NFB_ERR_ARG, "nfb_affine_coupling_image_taps: null pointer");
    NFB_CHECK(scale_map >= 0 && scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(split_mode == 0 || split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    return launch_coupling_taps(z, y_taps, bias, log_det, logdet_const, batch, channels, height, width, scale, scale_map,
                                split_mode, direction, accumulate, S(stream));
}
int32_t nfb_affine_coupling_image_taps_supported(int32_t channels, int32_t height, int32_t width, int32_t scale) {
    return coupling_taps_supported(channels, height, width, scale) ? 1 : 0;
}
int nfb_squeeze(const float* in, float* out, int64_t batch, int32_t channels, int32_t height, int32_t width,
                int32_t direction, void* stream) {
    NFB_CHECK(in && out, NFB_ERR_ARG, "nfb_squeeze: null pointer");
    return launch_squeeze(in, out, batch, channels, height, width, direction, S(stream));
}
int nfb_copy_channels(const float* in, float* out, int64_t batch, int32_t channels, int32_t c0, int32_t n,
                      int32_t hw, void* stream) {
    NFB_CHECK(in && out, NFB_ERR_ARG, "nfb_copy_channels: null pointer");
    return launch_copy_channels(in, out, batch, channels, c0, n, hw, S(stream));
}
int nfb_class_cond_diag_gaussian_log_prob(const float* z, const int64_t* y, const float* loc,
                                          const float* log_scale, float* log_q, int64_t batch, int32_t dim,
                                          int32_t num_classes, int32_t accumulate, void* stream) {
    NFB_CHECK(z && y && loc && log_scale && log_q, NFB_ERR_ARG, "nfb_class_cond_diag_gaussian_log_prob: null pointer");
    return launch_class_cond_gauss(z, reinterpret_cast<const long long*>(y), loc, log_scale, log_q, batch, dim,
                                   num_classes, accumulate, S(stream));
}

int nfb_swish(const float* x, float beta_softplus, int64_t n, float* a, float* da, void* stream) {
    NFB_CHECK(x && a, NFB_ERR_ARG, "nfb_swish: null pointer");
    return launch_swish(x, beta_softplus, n, a, da, S(stream));
}
int nfb_mul_rows(const float* src, const float* m, int64_t n, int32_t nt, float* dst, void* stream) {
    NFB_CHECK(src && m && dst, NFB_ERR_ARG, "nfb_mul_rows: null pointer");
    return launch_mul_rows(src, m, n, nt, dst, S(stream));
}
int nfb_logabsdet_i_plus_j_2x2(const float* jt, int64_t batch, float* out, void* stream) {
    NFB_CHECK(jt && out, NFB_ERR_ARG, "nfb_logabsdet_i_plus_j_2x2: null pointer");
    return launch_logdet2(jt, batch, out, S(stream));
}
int nfb_glu_residual(const float* h, const float* t, const float* c, int64_t n, float* out, void* stream) {
    NFB_CHECK(h && t && c && out, NFB_ERR_ARG, "nfb_glu_residual: null pointer");
    return launch_glu_residual(h, t, c, n, out, S(stream));
}
int nfb_rowdot(const float* a, const float* b, int64_t rows, int32_t d, float c, int32_t accumulate, float* out,
               void* stream) {
    NFB_CHECK(a && b && out, NFB_ERR_ARG, "nfb_rowdot: null pointer");
    return launch_rowdot(a, b, rows, d, c, accumulate, out, S(stream));
}

int nfb_maf_affine(const float* x, const float* params, float* y, float* log_det, int64_t rows, int32_t features,
                   int32_t inverse, int32_t accumulate, void* stream) {
    NFB_CHECK(x && params && y, NFB_ERR_ARG, "nfb_maf_affine: null pointer");
    NFB_CHECK(features >= 1, NFB_ERR_ARG, "nfb_maf_affine: bad feature count");
    return launch_maf_affine(x, params, y, log_det, rows, features, inverse, accumulate, S(stream));
}

int nfb_logit_transform(const float* in, float* out, float* log_det, int64_t batch, int64_t inner, float alpha,
                        int32_t direction, int32_t accumulate, void* stream) {
    NFB_CHECK(in && out, NFB_ERR_ARG, "nfb_logit_transform: null pointer");
    NFB_CHECK(direction == NFB_INVERSE || direction == NFB_FORWARD, NFB_ERR_ARG, "bad direction");
    NFB_CHECK(alpha >= 0.f && alpha < 0.5f, NFB_ERR_ARG, "Logit: alpha must be in [0, 0.5)");
    return launch_logit(in, out, log_det, batch, inner, alpha, direction, accumulate, S(stream));
}

int nfb_gemm_f32(const nfb_gemm_desc_t* d, void* stream) {
    NFB_CHECK(d && d->A && d->B && d->C, NFB_ERR_ARG, "nfb_gemm_f32: null pointer");
    NFB_CHECK(d->M >= 0 && d->N >= 0 && d->K > 0 && d->N < (1ll << 30), NFB_ERR_ARG, "nfb_gemm_f32: bad shape");
    GemmTcArgs a{};
    a.A = d->A; a.B = d->B; a.C = d->C; a.lda = d->lda; a.ldb = d->ldb; a.ldc = d->ldc; a.M = d->M; a.N = d->N; a.K = d->K;
    a.a_mn = d->a_mn; a.b_mn = d->b_mn; a.a_relu = d->a_relu; a.b_relu = d->b_relu; a.relu_out = d->relu_out;
    a.accumulate = d->accumulate; a.bias = d->bias; a.mask = d->mask; a.mulm = d->mulm; a.ldmask = d->ldmask;
    a.resid = d->resid; a.ldres = d->ldres;
    static thread_local int* err_dev = nullptr;  // per-thread device word for the kernel's barrier-timeout tag
    if (!err_dev) { NFB_CUDA(cudaMalloc(reinterpret_cast<void**>(&err_dev), 16)); NFB_CUDA(cudaMemset(err_dev, 0, 16)); }
    return launch_gemm_tc(a, err_dev, S(stream));
}

int nfb_flow_create(nfb_flow_t** out, int32_t features) {
    NFB_CHECK(out, NFB_ERR_ARG, "nfb_flow_create: null out");
    NFB_CHECK(features >= 1, NFB_ERR_ARG, "nfb_flow_create: features must be >= 1");
    int n = 0;
    NFB_CUDA(cudaGetDeviceCount(&n));
    NFB_CHECK(n > 0, NFB_ERR_CUDA, "nfb_flow_create: no CUDA device (this library has no CPU path)");
    nfb_flow* f = new nfb_flow();
    f->D = features;
    int sm = 132;
    if (nfb_device_info(&sm, nullptr, nullptr) == NFB_OK) f->sm_count = sm;
    int rc = f->err.reserve(16);
    if (rc) { delete f; return rc; }
    cudaMemset(f->err.p, 0, 16);
    *out = f;
    return NFB_OK;
}

int nfb_flow_destroy(nfb_flow_t* f) {
    delete f;
    return NFB_OK;
}

#define NFB_NEW_LAYER(kind_)                                                             \
    NFB_CHECK(f && d, NFB_ERR_ARG, "null argument");                                     \
    NFB_CHECK(!f->finalized, NFB_ERR_STATE, "flow already finalized");                   \
    NFB_CHECK(d->features == f->D, NFB_ERR_ARG, "Expected features = %d, got %d.", f->D, d->features); \
    std::unique_ptr<Layer> L(new Layer());                                               \
    L->kind = kind_;                                                                     \
    L->D = f->D

int nfb_flow_add_ar_rqs(nfb_flow_t* f, const nfb_ar_rqs_desc_t* d) {
    NFB_NEW_LAYER(L_AR_RQS);
    L->K = d->num_bins; L->tail = d->tail_bound; L->wh_scale = 1.f;  // MADE has no hidden_features attr
    NFB_CHECK(L->K >= 1 && L->K <= 32, NFB_ERR_ARG, "num_bins out of range");
    NFB_CHECK(kMinBinWidth * L->K <= 1.0f, NFB_ERR_ARG, "Minimal bin width too large for the number of bins");
    NFB_TRY(copy_net(d->net, L->net));
    NFB_CHECK(L->net.in == f->D && L->net.out == f->D * (3 * L->K - 1), NFB_ERR_ARG, "AR net shape mismatch");
    L->n_tr = f->D;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_coupled_rqs(nfb_flow_t* f, const nfb_coupled_rqs_desc_t* d) {
    NFB_NEW_LAYER(L_COUPLED_RQS);
    L->K = d->num_bins; L->tail = d->tail_bound;
    NFB_CHECK(L->K >= 1 && L->K <= 32, NFB_ERR_ARG, "num_bins out of range");
    NFB_CHECK(kMinBinWidth * L->K <= 1.0f, NFB_ERR_ARG, "Minimal bin width too large for the number of bins");
    NFB_CHECK(d->num_identity + d->num_transform == f->D && d->num_identity > 0 && d->num_transform > 0,
              NFB_ERR_ARG, "coupled: identity + transform features must cover the input");
    NFB_CHECK(d->identity_features && d->transform_features && d->uncond_widths && d->uncond_heights && d->uncond_derivatives,
              NFB_ERR_ARG, "coupled: null pointer");
    NFB_TRY(copy_net(d->net, L->net));
    NFB_CHECK(L->net.in == d->num_identity && L->net.out == d->num_transform * (3 * L->K - 1), NFB_ERR_ARG, "coupled net shape mismatch");
    L->wh_scale = 1.0f / sqrtf((float)L->net.H);  // neural_spline/coupling.py:334-336
    L->n_id = d->num_identity; L->n_tr = d->num_transform;
    L->id64 = d->identity_features; L->tr64 = d->transform_features;
    L->uw = d->uncond_widths; L->uh = d->uncond_heights; L->ud = d->uncond_derivatives;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_lu_linear_permute(nfb_flow_t* f, const nfb_lu_desc_t* d) {
    NFB_NEW_LAYER(L_LU);
    NFB_CHECK(d->permutation && d->lower_entries && d->upper_entries && d->unconstrained_upper_diag && d->bias,
              NFB_ERR_ARG, "LULinearPermute: null pointer");
    NFB_CHECK(f->D <= 64, NFB_ERR_UNSUPPORTED, "LULinearPermute: features %d > 64", f->D);
    L->lu = *d;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_masked_affine(nfb_flow_t* f, const nfb_masked_affine_desc_t* d) {
    NFB_NEW_LAYER(L_MASKED_AFFINE);
    NFB_CHECK(f->D <= kAffMaxD, NFB_ERR_UNSUPPORTED, "MaskedAffineFlow: features %d > %d", f->D, kAffMaxD);
    NFB_CHECK(d->b, NFB_ERR_ARG, "MaskedAffineFlow: null mask");
    L->op.type = kOpMasked; L->op.p0 = d->b; L->op.slope = 0.f;
    NFB_TRY(copy_mlp(d->s, L->op.s, &L->op.slope));
    NFB_TRY(copy_mlp(d->t, L->op.t, &L->op.slope));
    if (d->s.num_layers) NFB_CHECK(d->s.sizes[0] == f->D && d->s.sizes[d->s.num_layers] == f->D, NFB_ERR_ARG, "s-net must map D -> D");
    if (d->t.num_layers) NFB_CHECK(d->t.sizes[0] == f->D && d->t.sizes[d->t.num_layers] == f->D, NFB_ERR_ARG, "t-net must map D -> D");
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_affine_coupling(nfb_flow_t* f, const nfb_affine_coupling_desc_t* d) {
    NFB_NEW_LAYER(L_AFFINE_COUPLING);
    NFB_CHECK(f->D <= kAffMaxD, NFB_ERR_UNSUPPORTED, "AffineCouplingBlock: features %d > %d", f->D, kAffMaxD);
    NFB_CHECK(d->scale_map >= 0 && d->scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(d->split_mode == 0 || d->split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    L->op.type = kOpCoupling;
    L->op.flags = (d->scale ? 1 : 0) | (d->scale_map << 1) | (d->split_mode << 3);
    NFB_TRY(copy_mlp(d->param_map, L->op.s, &L->op.slope));
    const int h = (f->D + 1) / 2;
    const int n1 = d->split_mode ? f->D - h : h, n2 = f->D - n1;
    NFB_CHECK(d->param_map.num_layers >= 1 && d->param_map.sizes[0] == n1 &&
              d->param_map.sizes[d->param_map.num_layers] == (d->scale ? 2 : 1) * n2,
              NFB_ERR_ARG, "param_map must map %d -> %d", n1, (d->scale ? 2 : 1) * n2);
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_affine_const(nfb_flow_t* f, const nfb_affine_const_desc_t* d) {
    NFB_NEW_LAYER(L_AFFINE_CONST);
    NFB_CHECK(f->D <= kAffMaxD, NFB_ERR_UNSUPPORTED, "AffineConstFlow: features %d > %d", f->D, kAffMaxD);
    NFB_CHECK(d->s && d->t, NFB_ERR_ARG, "AffineConstFlow: null s/t");
    L->op.type = kOpConst; L->op.p0 = d->s; L->op.p1 = d->t;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_permute(nfb_flow_t* f, const nfb_permute_desc_t* d) {
    NFB_NEW_LAYER(L_PERMUTE);
    NFB_CHECK(f->D <= kAffMaxD, NFB_ERR_UNSUPPORTED, "Permute: features %d > %d", f->D, kAffMaxD);
    NFB_CHECK(d->perm && d->inv_perm, NFB_ERR_ARG, "Permute: null index list");
    L->perm_fwd.assign(d->perm, d->perm + f->D);
    L->perm_inv.assign(d->inv_perm, d->inv_perm + f->D);
    for (int j = 0; j < f->D; ++j)
        NFB_CHECK(L->perm_fwd[j] >= 0 && L->perm_fwd[j] < f->D && L->perm_inv[j] >= 0 && L->perm_inv[j] < f->D,
                  NFB_ERR_ARG, "Permute: index out of range");
    NFB_TRY(L->perm_fwd_dev.upload(L->perm_fwd));
    NFB_TRY(L->perm_inv_dev.upload(L->perm_inv));
    L->op.type = kOpPermute; L->op.fwd_idx = L->perm_fwd_dev.as<int>(); L->op.inv_idx = L->perm_inv_dev.as<int>();
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_set_base_diag_gaussian(nfb_flow_t* f, const float* loc, const float* log_scale) {
    NFB_CHECK(f && loc && log_scale, NFB_ERR_ARG, "null argument");
    f->base_loc = loc; f->base_log_scale = log_scale;
    return NFB_OK;
}

int nfb_flow_repack(nfb_flow_t* f, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "nfb_flow_repack: flow not finalized");
    cudaStream_t st = S(stream);
    // LU maps first: the fused blocks' fp16 scale plans need the norms of the maps in front of them
    {
        std::vector<LuPackArgs> args;
        int n_max = 1;
        for (auto& Lp : f->layers)
            if (Lp->kind == L_LU) {
                Layer& L = *Lp;
                const int n = L.D;
                NFB_TRY(L.lu_Wd.reserve((size_t)n * n * 4));
                NFB_TRY(L.lu_Ws.reserve((size_t)n * n * 4));
                NFB_TRY(L.lu_logdet.reserve(4));
                args.push_back(LuPackArgs{L.lu.lower_entries, L.lu.upper_entries, L.lu.unconstrained_upper_diag, L.lu.eps, n,
                                          L.lu_Wd.as<float>(), L.lu_Ws.as<float>(), L.lu_logdet.as<float>()});
                n_max = std::max(n_max, n);
            }
        if (!args.empty()) {
            NFB_TRY(f->lu_args.upload(args));
            NFB_TRY(launch_lu_pack_batched(f->lu_args.as<LuPackArgs>(), (int)args.size(), n_max, st));
        }
    }
    for (auto& Lp : f->layers)
        if (Lp->kind == L_LU) NFB_TRY(repack_lu(f, *Lp, st, true));
    for (auto& Lp : f->layers) {
        Layer& L = *Lp;
        // |input| u_row < 1.  Coupled block, sampling direction: the conditioner sees the inverse unconditional
        // spline's output, bounded by max(|x|, tail); the autoregressive block folds the tail into u_row itself.
        if (L.kind == L_AR_RQS || L.kind == L_COUPLED_RQS) L.fused.b_in0 = L.kind == L_COUPLED_RQS ? std::max(1.f, L.tail) : 1.f;
    }
    for (auto& g : f->groups)
        if (g.kind == G_FUSED_PAIR) {
            Layer& R = *f->layers[g.first];
            Layer& U = *f->layers[g.last];
            R.fused.b_in0 = std::max(R.fused.b_in0, U.lu_norm_d + U.lu_bmax_d);
        }
    for (auto& u : f->fwd_units)
        if (u.first >= 0) {
            Layer& R = *f->layers[u.second];
            Layer& U = *f->layers[u.first];
            R.fused.b_in0 = std::max(R.fused.b_in0, U.lu_norm_s + U.lu_bmax_s);
        }
    for (auto& Lp : f->layers) {
        Layer& L = *Lp;
        if (L.kind == L_AR_RQS || L.kind == L_COUPLED_RQS) {
            NFB_TRY(pack_net_generic(L.net, L.pack, st));
            if (L.kind == L_COUPLED_RQS) {
                const int P = 3 * L.K - 1, K = L.K;
                std::vector<float> w, h, d, tab((size_t)L.n_id * P);
                NFB_CUDA(cudaStreamSynchronize(st));
                NFB_TRY(download(L.uw, (size_t)L.n_id * K, w));
                NFB_TRY(download(L.uh, (size_t)L.n_id * K, h));
                NFB_TRY(download(L.ud, (size_t)L.n_id * (K - 1), d));
                for (int i = 0; i < L.n_id; ++i) {
                    for (int k = 0; k < K; ++k) { tab[i * P + k] = w[i * K + k]; tab[i * P + K + k] = h[i * K + k]; }
                    for (int k = 0; k < K - 1; ++k) tab[i * P + 2 * K + k] = d[i * (K - 1) + k];
                }
                NFB_TRY(L.uncond.upload(tab));
            }
            Layer* Ufold = nullptr;
            for (auto& g : f->groups)
                if (g.kind == G_FUSED_PAIR && f->layers[g.first].get() == &L) Ufold = f->layers[g.last].get();
            NFB_TRY(repack_fused(f, L, st, Ufold));
        }
    }
    for (auto& g : f->groups)
        if (g.kind == G_FUSED_PAIR) NFB_TRY(repack_pair(f, *f->layers[g.first], *f->layers[g.last], st));
    // whole-stack launch plan (density direction applies the groups last-to-first)
    f->stack_n = 0;
    bool all_fused = !f->groups.empty() && getenv("NFB_NO_STACK") == nullptr;
    for (auto& g : f->groups) all_fused = all_fused && (g.kind == G_FUSED_PAIR || g.kind == G_FUSED);
    if (all_fused) {
        std::vector<FusedLayer> arr;
        for (int k = (int)f->groups.size() - 1; k >= 0; --k) {
            Group& g = f->groups[k];
            FusedPack& F = f->layers[g.first]->fused;
            arr.push_back(g.kind == G_FUSED_PAIR ? F.host_pair : F.host_layer);
        }
        NFB_TRY(f->stack_layers.reserve(arr.size() * sizeof(FusedLayer)));
        NFB_CUDA(cudaMemcpy(f->stack_layers.p, arr.data(), arr.size() * sizeof(FusedLayer), cudaMemcpyHostToDevice));
        f->stack_n = (int)arr.size();
    }
    // sampling-direction plan (list order); same persistent kernel, SAMPLE instantiation
    f->fwd_n = 0;
    if (!f->fwd_units.empty() && getenv("NFB_NO_STACK") == nullptr) {
        std::vector<FusedLayer> arr;
        for (auto& u : f->fwd_units) {
            Layer& R = *f->layers[u.second];
            NFB_TRY(repack_fwd_unit(f, R, u.first >= 0 ? f->layers[u.first].get() : nullptr, st));
            arr.push_back(R.fused.host_fwd);
        }
        NFB_TRY(f->fwd_layers.reserve(arr.size() * sizeof(FusedLayer)));
        NFB_CUDA(cudaMemcpy(f->fwd_layers.p, arr.data(), arr.size() * sizeof(FusedLayer), cudaMemcpyHostToDevice));
        f->fwd_n = (int)arr.size();
    }
    NFB_CUDA(cudaStreamSynchronize(st));
    return NFB_OK;
}

int nfb_flow_finalize(nfb_flow_t* f, int32_t use_tensor_cores, void* stream) {
    NFB_CHECK(f, NFB_ERR_ARG, "null flow");
    NFB_CHECK(!f->finalized, NFB_ERR_STATE, "flow already finalized");
    cudaStream_t st = S(stream);
    f->use_tc = use_tensor_cores != 0;
    int major = 0;
    NFB_TRY(nfb_device_info(nullptr, &major, nullptr));
    if (major != 9) f->use_tc = false;  // wgmma exists on sm_90 only; the fp32 kernels still run
    const int n = (int)f->layers.size();
    // per-layer static prep
    for (auto& Lp : f->layers) {
        Layer& L = *Lp;
        if (L.kind == L_COUPLED_RQS) {
            std::vector<int64_t> id64, tr64;
            NFB_TRY(download(L.id64, (size_t)L.n_id, id64));
            NFB_TRY(download(L.tr64, (size_t)L.n_tr, tr64));
            std::vector<int> a(id64.begin(), id64.end()), b(tr64.begin(), tr64.end());
            for (int v : a) NFB_CHECK(v >= 0 && v < L.D, NFB_ERR_ARG, "identity feature index out of range");
            for (int v : b) NFB_CHECK(v >= 0 && v < L.D, NFB_ERR_ARG, "transform feature index out of range");
            NFB_TRY(L.id_idx.upload(a));
            NFB_TRY(L.tr_idx.upload(b));
        }
        if (L.kind == L_AR_RQS || L.kind == L_COUPLED_RQS) NFB_TRY(build_fused(f, L, st));
        if (L.kind == L_LU) {
            std::vector<int64_t> p64;
            NFB_TRY(download(L.lu.permutation, (size_t)L.D, p64));
            L.perm_host.assign(p64.begin(), p64.end());
            std::vector<int> inv(L.D);
            for (int j = 0; j < L.D; ++j) {
                NFB_CHECK(L.perm_host[j] >= 0 && L.perm_host[j] < L.D, NFB_ERR_ARG, "permutation out of range");
                inv[L.perm_host[j]] = j;
            }
            NFB_TRY(L.lu_perm.upload(L.perm_host));
            NFB_TRY(L.lu_tmp.upload(inv));
            L.inv_perm_host = inv;
        }
    }
    // execution groups (list order)
    f->groups.clear();
    for (int i = 0; i < n;) {
        Layer& L = *f->layers[i];
        if ((L.kind == L_AR_RQS || L.kind == L_COUPLED_RQS) && L.fused.ok) {
            if (i + 1 < n && f->layers[i + 1]->kind == L_LU) {
                NFB_TRY(build_pair(f, L, *f->layers[i + 1], st));
                if (L.fused.pair_ok) {
                    Group g; g.kind = G_FUSED_PAIR; g.first = i; g.last = i + 1;
                    f->groups.push_back(std::move(g));
                    i += 2;
                    continue;
                }
            }
            Group g; g.kind = G_FUSED; g.first = g.last = i;
            f->groups.push_back(std::move(g));
            ++i;
        } else if (is_affine_kind(L)) {
            int j = i;
            while (j + 1 < n && is_affine_kind(*f->layers[j + 1])) ++j;
            Group g; g.kind = G_AFFINE; g.first = i; g.last = j;
            std::vector<AffineOp> ops;
            for (int k = i; k <= j; ++k) ops.push_back(f->layers[k]->op);
            NFB_TRY(g.ops.upload(ops));
            f->groups.push_back(std::move(g));
            i = j + 1;
        } else {
            Group g; g.kind = G_SINGLE; g.first = g.last = i;
            f->groups.push_back(std::move(g));
            ++i;
        }
    }
    // sampling-direction units: every layer must be a fused coupling block or an LU map that directly
    // precedes one (or closes the list); anything else keeps the group-by-group path
    f->fwd_units.clear();
    f->fwd_trailing_lu = -1;
    {
        bool ok = f->use_tc && n > 0;
        int pending = -1;
        for (int i = 0; i < n && ok; ++i) {
            Layer& L = *f->layers[i];
            if (L.kind == L_LU) {
                ok = pending < 0;
                pending = i;
            } else if ((L.kind == L_COUPLED_RQS || L.kind == L_AR_RQS) && L.fused.ok) {
                NFB_TRY(build_fwd_unit(f, L, pending >= 0 ? f->layers[pending].get() : nullptr));
                ok = L.fused.fwd_ok;
                f->fwd_units.push_back({pending, i});
                pending = -1;
            } else {
                ok = false;
            }
        }
        if (ok) f->fwd_trailing_lu = pending;
        else f->fwd_units.clear();
    }
    f->finalized = true;
    return nfb_flow_repack(f, stream);
}

int nfb_flow_num_layers(const nfb_flow_t* f) { return f ? (int)f->layers.size() : 0; }
int64_t nfb_flow_last_launch_count(const nfb_flow_t* f) { return f ? f->launches : 0; }
int nfb_flow_layer_is_fused(const nfb_flow_t* f, int32_t index) {
    if (!f || index < 0 || index >= (int)f->layers.size()) return 0;
    for (auto& g : f->groups)
        if ((g.kind == G_FUSED || g.kind == G_FUSED_PAIR) && index >= g.first && index <= g.last) return 1;
    return 0;
}

int nfb_flow_layer_apply(nfb_flow_t* f, int32_t index, int32_t direction, const float* z_in, float* z_out,
                         float* log_det, int64_t rows, int32_t accumulate, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(index >= 0 && index < (int)f->layers.size(), NFB_ERR_ARG, "layer index out of range");
    NFB_CHECK(z_in && z_out, NFB_ERR_ARG, "null pointer");
    NFB_CHECK(direction == NFB_INVERSE || direction == NFB_FORWARD, NFB_ERR_ARG, "bad direction");
    cudaStream_t st = S(stream);
    if (rows == 0) return NFB_OK;
    Layer& L = *f->layers[index];
    float* out = z_out;
    if (z_in == z_out) {
        NFB_TRY(f->zA.reserve((size_t)rows * f->D * 4));
        out = f->zA.as<float>();
    }
    if (log_det && !accumulate) NFB_TRY(launch_fill(log_det, rows, 0.f, st));
    int rc;
    if (is_affine_kind(L)) {
        DevBuf ops;
        std::vector<AffineOp> v{L.op};
        NFB_TRY(ops.upload(v));
        rc = launch_affine_stack(ops.p, 1, z_in, out, log_det, rows, f->D, 1, direction, st);
        NFB_CUDA(cudaStreamSynchronize(st));  // ops buffer is freed on return
    } else if ((L.kind == L_AR_RQS || L.kind == L_COUPLED_RQS) && L.fused.ok) {
        // (the autoregressive block's sampling direction runs its D conditioner passes inside the fused unit)
        if (!log_det) { NFB_TRY(f->logq.reserve((size_t)rows * 4)); }
        rc = launch_fused_layer(f, L, nullptr, z_in, out, log_det ? log_det : f->logq.as<float>(), rows, 1, st,
                                direction == NFB_FORWARD);
    } else {
        rc = apply_layer_generic(f, L, direction, z_in, out, log_det, rows, 1, st);
    }
    if (rc) return rc;
    if (out != z_out) NFB_CUDA(cudaMemcpyAsync(z_out, out, (size_t)rows * f->D * 4, cudaMemcpyDeviceToDevice, st));
    return NFB_OK;
}

int nfb_flow_transform(nfb_flow_t* f, int32_t direction, const float* z_in, float* z_out, float* log_det,
                       int64_t rows, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(z_in && z_out, NFB_ERR_ARG, "null pointer");
    NFB_CHECK(direction == NFB_INVERSE || direction == NFB_FORWARD, NFB_ERR_ARG, "bad direction");
    cudaStream_t st = S(stream);
    f->launches = 0;
    if (rows == 0) return NFB_OK;
    NFB_TRY(ensure_ws(f, rows));
    float* ld = log_det ? log_det : f->logq.as<float>();
    NFB_TRY(launch_fill(ld, rows, 0.f, st));
    f->launches++;
    if (direction == NFB_INVERSE && f->stack_n > 0)
        return launch_fused_stack(f, z_in, z_out, ld, rows, st);
    if (direction == NFB_FORWARD && f->fwd_n > 0) {
        if (f->fwd_trailing_lu < 0) return launch_fused_stack(f, z_in, z_out, ld, rows, st, 1);
        float* tmp = f->zA.as<float>();
        NFB_TRY(launch_fused_stack(f, z_in, tmp, ld, rows, st, 1));
        return apply_layer_generic(f, *f->layers[f->fwd_trailing_lu], NFB_FORWARD, tmp, z_out, ld, rows, 1, st);
    }
    const int ng = (int)f->groups.size();
    const float* cur = z_in;
    float* bufs[2] = {f->zA.as<float>(), f->zB.as<float>()};
    int flip = 0;
    for (int k = 0; k < ng; ++k) {
        Group& g = f->groups[direction == NFB_FORWARD ? k : ng - 1 - k];
        float* out = (k == ng - 1 && z_out != z_in) ? z_out : bufs[flip];
        NFB_TRY(run_group(f, g, direction, cur, out, ld, rows, st));
        cur = out;
        flip ^= 1;
    }
    if (cur != z_out) NFB_CUDA(cudaMemcpyAsync(z_out, cur, (size_t)rows * f->D * 4, cudaMemcpyDeviceToDevice, st));
    return NFB_OK;
}

int nfb_flow_log_prob(nfb_flow_t* f, const float* x, float* log_q, int64_t rows, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(f->base_loc && f->base_log_scale, NFB_ERR_STATE, "no base distribution set");
    NFB_CHECK(x && log_q, NFB_ERR_ARG, "null pointer");
    if (rows == 0) return NFB_OK;
    NFB_TRY(ensure_ws(f, rows));
    NFB_TRY(f->zfinal.reserve((size_t)rows * f->D * 4));
    float* z = f->zfinal.as<float>();
    NFB_TRY(nfb_flow_transform(f, NFB_INVERSE, x, z, log_q, rows, stream));
    NFB_TRY(launch_diag_gauss(z, f->base_loc, f->base_log_scale, log_q, rows, f->D, 1, S(stream)));
    f->launches++;
    return NFB_OK;
}

int nfb_flow_forward_kld(nfb_flow_t* f, const float* x, int64_t rows, float* loss, double* sum, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(x && (loss || sum), NFB_ERR_ARG, "null pointer");
    NFB_CHECK(rows > 0, NFB_ERR_ARG, "forward_kld needs at least one row");
    NFB_TRY(ensure_ws(f, rows));
    NFB_TRY(f->loss.reserve(16 + (size_t)rows * 4));
    float* logq = reinterpret_cast<float*>(static_cast<char*>(f->loss.p) + 16);
    NFB_TRY(nfb_flow_log_prob(f, x, logq, rows, stream));
    NFB_TRY(launch_sum(logq, rows, -1.0 / (double)rows, f->scratch_sum.as<double>(), loss, sum, S(stream)));
    f->launches += 2;
    return NFB_OK;
}

namespace {
constexpr int kH2dChunks = 16;
// Start the host->device copy of a [rows x D] batch in kH2dChunks pieces on the flow's copy stream; after each
// piece a 4-byte copy publishes the number of resident rows in f->in_ready.  When the density pass runs as ONE
// whole-stack launch, that kernel starts immediately on the compute stream and gates its layer-0 tiles on the
// counter (FusedParams::in_ready), so the transfer overlaps the first layers; any other execution plan simply
// waits for the last piece (event).  Copy engines do not need SMs, so a resident spinning kernel cannot starve
// them.  Returns with *gated = 1 if the kernel-side gate is armed.
// Host batch -> device in kH2dChunks pieces on a copy stream; after every piece a 4-byte copy publishes the number of
// resident rows, and the whole-stack kernel's layer-0 tiles wait for their rows (fused_rqs_kernel, in_ready).
// h2d_prepare resets the counter and decides whether the pass is gated; h2d_copies enqueues the pieces.
int h2d_prepare(nfb_flow* f, int64_t rows, int* gated) {
    if (!f->copy_stream) {
        NFB_CUDA(cudaStreamCreateWithFlags(&f->copy_stream, cudaStreamNonBlocking));
        NFB_CUDA(cudaEventCreateWithFlags(&f->ev_reset, cudaEventDisableTiming));
        NFB_CUDA(cudaEventCreateWithFlags(&f->ev_copied, cudaEventDisableTiming));
        NFB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&f->h_seq), kH2dChunks * sizeof(int), cudaHostAllocDefault));
        NFB_TRY(f->in_ready.reserve(16));
    }
    const bool gate = f->stack_n > 0 && rows >= 8192 && rows < (1ll << 31) && getenv("NFB_NO_H2D_OVERLAP") == nullptr;
    NFB_CUDA(cudaMemsetAsync(f->in_ready.p, 0, 4, 0));
    NFB_CUDA(cudaEventRecord(f->ev_reset, 0));
    NFB_CUDA(cudaStreamWaitEvent(f->copy_stream, f->ev_reset, 0));  // previous pass has finished with xd / the counter
    if (gate) f->cur_in_ready = f->in_ready.as<int>();
    *gated = gate ? 1 : 0;
    return NFB_OK;
}
int h2d_copies(nfb_flow* f, const float* x_host, float* xd, int64_t rows, int gate) {
    const int64_t per = ((rows + kH2dChunks - 1) / kH2dChunks + kFusedTileRows - 1) / kFusedTileRows * kFusedTileRows;  // whole tiles
    int64_t done = 0;
    for (int c = 0; c < kH2dChunks && done < rows; ++c) {
        const int64_t n = std::min(per, rows - done);
        NFB_CUDA(cudaMemcpyAsync(xd + done * f->D, x_host + done * f->D, (size_t)n * f->D * 4, cudaMemcpyHostToDevice,
                                 f->copy_stream));
        done += n;
        if (gate) {
            f->h_seq[c] = (int)done;
            NFB_CUDA(cudaMemcpyAsync(f->in_ready.p, &f->h_seq[c], 4, cudaMemcpyHostToDevice, f->copy_stream));
        }
    }
    NFB_CUDA(cudaEventRecord(f->ev_copied, f->copy_stream));
    if (!gate) NFB_CUDA(cudaStreamWaitEvent(0, f->ev_copied, 0));
    return NFB_OK;
}
}  // namespace

int nfb_flow_log_prob_host(nfb_flow_t* f, const float* x_host, float* log_q_host, int64_t rows) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(x_host && log_q_host, NFB_ERR_ARG, "null pointer");
    if (rows == 0) return NFB_OK;
    NFB_TRY(f->host_x.reserve((size_t)rows * f->D * 4 + (size_t)rows * 4));
    float* xd = f->host_x.as<float>();
    float* lq = xd + (size_t)rows * f->D;
    int gated = 0;
    NFB_TRY(h2d_prepare(f, rows, &gated));
    // Copies are enqueued BEFORE the compute launches: a launch that blocks the host until the kernel has finished
    // (CUDA_LAUNCH_BLOCKING, ncu, compute-sanitizer) must find its input already on its way -- the kernel waits for it.
    // (Kernels-first was measured: no e2e gain; the gap to the device-resident pass is PCIe time, not enqueue time.)
    NFB_TRY(h2d_copies(f, x_host, xd, rows, gated));
    const int rc = nfb_flow_log_prob(f, xd, lq, rows, nullptr);
    f->cur_in_ready = nullptr;
    if (rc) return rc;
    NFB_CUDA(cudaMemcpyAsync(log_q_host, lq, (size_t)rows * 4, cudaMemcpyDeviceToHost, 0));
    NFB_CUDA(cudaStreamSynchronize(0));
    return NFB_OK;
}

int nfb_flow_forward_kld_host(nfb_flow_t* f, const float* x_host, int64_t rows, float* loss_host) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(x_host && loss_host, NFB_ERR_ARG, "null pointer");
    NFB_CHECK(rows > 0, NFB_ERR_ARG, "forward_kld needs at least one row");
    NFB_TRY(f->host_x.reserve((size_t)rows * f->D * 4));
    NFB_TRY(f->loss.reserve(16 + (size_t)rows * 4));
    float* xd = f->host_x.as<float>();
    int gated = 0;
    NFB_TRY(h2d_prepare(f, rows, &gated));
    // Copies are enqueued BEFORE the compute launches: a launch that blocks the host until the kernel has finished
    // (CUDA_LAUNCH_BLOCKING, ncu, compute-sanitizer) must find its input already on its way -- the kernel waits for it.
    // (Kernels-first was measured: no e2e gain; the gap to the device-resident pass is PCIe time, not enqueue time.)
    NFB_TRY(h2d_copies(f, x_host, xd, rows, gated));
    const int rc = nfb_flow_forward_kld(f, xd, rows, f->loss.as<float>(), nullptr, nullptr);
    f->cur_in_ready = nullptr;
    if (rc) return rc;
    NFB_CUDA(cudaMemcpyAsync(loss_host, f->loss.p, 4, cudaMemcpyDeviceToHost, 0));
    NFB_CUDA(cudaStreamSynchronize(0));
    return NFB_OK;
}

}  // extern "C"

// ==========================================================================================
// training pass: gradients of log_prob w.r.t. every parameter and the input (SURVEY 8f-1)
// ==========================================================================================
namespace {

int grad_slots_of(const Layer& L) {
    switch (L.kind) {
    case L_AR_RQS: return 4 + 4 * L.net.nb;
    case L_COUPLED_RQS: return 4 + 4 * L.net.nb + 3;
    case L_LU: return 4;
    default: return -1;
    }
}
long long grad_slot_numel(const Layer& L, int s) {
    const NetDesc& n = L.net;
    if (L.kind == L_LU) {
        const long long d = L.D;
        return s == 0 ? d * (d - 1) / 2 : s == 1 ? d * (d - 1) / 2 : d;
    }
    const int nlin = 2 + 2 * n.nb;  // linears: initial, blocks..., final
    if (s < 2 * nlin) {
        const int lin = s / 2, isb = s & 1;
        const long long out = lin == 0 ? n.H : (lin == nlin - 1 ? n.out : n.H);
        const long long in = lin == 0 ? n.in : n.H;
        return isb ? out : out * in;
    }
    const int u = s - 2 * nlin;  // coupled: unconditional widths, heights, derivatives
    return (long long)L.n_id * (u == 2 ? L.K - 1 : L.K);
}

struct Gemm {
    nfb_flow* f; cudaStream_t st;
    int run(GemmTcArgs a) { f->launches++; return launch_gemm_tc(a, f->err.as<int>(), st); }
    // B is a WEIGHT matrix (reused by every 128-row tile of the batch): split it to bf16 hi | lo records once
    // (launch_gemm_pack_b) and let the GEMM stream them by TMA instead of converting them per tile.
    int run_w(GemmTcArgs a) {
        const size_t bytes = gemm_tc_packed_b_bytes(a.N, a.K, a.b_mn);
        NFB_TRY(f->tr_wpack.reserve(bytes));
        NFB_TRY(launch_gemm_pack_b(a.B, a.ldb, a.b_mn, a.N, a.K, f->tr_wpack.as<uint8_t>(), st));
        a.b_packed = f->tr_wpack.as<uint8_t>();
        f->launches += 2;
        return launch_gemm_tc(a, f->err.as<int>(), st);
    }
};

// conditioner forward (recompute) into h[0..n_hidden-1] ([rows x H] each) and P ([rows x out])
int net_recompute(nfb_flow* f, const NetDesc& n, const NetPack& p, const float* in, int ld_in, long long rows, float* hbuf,
                  float* P, cudaStream_t st) {
    Gemm g{f, st};
    const long long HS = rows * n.H;
    GemmTcArgs a{};
    a.A = in; a.lda = ld_in; a.B = p.w0; a.ldb = n.in; a.C = hbuf; a.ldc = n.H; a.M = rows; a.N = n.H; a.K = n.in; a.bias = n.b0;
    NFB_TRY(g.run_w(a));
    for (int b = 0; b < n.nb; ++b) {
        float* hprev = hbuf + (size_t)(2 * b) * HS;
        float* t = hbuf + (size_t)(2 * b + 1) * HS;
        float* hnext = hbuf + (size_t)(2 * b + 2) * HS;
        GemmTcArgs t1{};
        t1.A = hprev; t1.lda = n.H; t1.a_relu = 1; t1.B = p.wb[2 * b]; t1.ldb = n.H; t1.C = t; t1.ldc = n.H;
        t1.M = rows; t1.N = n.H; t1.K = n.H; t1.bias = n.bb[2 * b];
        NFB_TRY(g.run_w(t1));
        GemmTcArgs t2{};
        t2.A = t; t2.lda = n.H; t2.a_relu = 1; t2.B = p.wb[2 * b + 1]; t2.ldb = n.H; t2.C = hnext; t2.ldc = n.H;
        t2.M = rows; t2.N = n.H; t2.K = n.H; t2.bias = n.bb[2 * b + 1]; t2.resid = hprev; t2.ldres = n.H;
        NFB_TRY(g.run_w(t2));
    }
    GemmTcArgs fl{};
    fl.A = hbuf + (size_t)(2 * n.nb) * HS; fl.lda = n.H; fl.B = p.wf; fl.ldb = n.H; fl.C = P; fl.ldc = n.out;
    fl.M = rows; fl.N = n.out; fl.K = n.H; fl.bias = n.bf;
    return g.run_w(fl);
}

// one Linear's parameter gradients: dW = gY^T act(X) (* mask), db = colsum(gY)
int linear_wgrad(nfb_flow* f, const float* gY, int n_out, const float* X, int ldx, int n_in, int x_relu, const float* mask,
                 long long rows, float* dW, float* db, cudaStream_t st) {
    if (dW) {
        Gemm g{f, st};
        GemmTcArgs a{};
        a.A = gY; a.lda = n_out; a.a_mn = 1; a.B = X; a.ldb = ldx; a.b_mn = 1; a.b_relu = x_relu;
        a.C = dW; a.ldc = n_in; a.M = n_out; a.N = n_in; a.K = rows; a.mulm = mask; a.ldmask = n_in;
        NFB_TRY(g.run(a));
    }
    if (db) {
        NFB_CUDA(cudaMemsetAsync(db, 0, (size_t)n_out * 4, st));
        NFB_TRY(launch_colsum(gY, n_out, rows, n_out, db, st));
        f->launches += 2;
    }
    return NFB_OK;
}

// backward of one spline layer: xp = the layer's input [rows x D], gy = gradient w.r.t. its output; writes the
// gradient w.r.t. its input into gxp ([rows x D]) and the parameter gradients into `slots`.
int rqs_layer_backward(nfb_flow* f, Layer& L, const float* xp, const float* gy, const float* glq, long long rows,
                       float* gxp, float* const* slots, cudaStream_t st) {
    const NetDesc& n = L.net;
    const NetPack& p = L.pack;
    const int D = L.D, H = n.H, T = L.n_tr, P = 3 * L.K - 1;
    const bool coupled = L.kind == L_COUPLED_RQS;
    const int n_hidden = 1 + 2 * n.nb;
    const long long HS = rows * H;
    NFB_CHECK(L.K == 8, NFB_ERR_UNSUPPORTED, "native backward: num_bins %d != 8", L.K);
    NFB_TRY(f->tr_h.reserve((size_t)n_hidden * HS * 4));
    NFB_TRY(f->tr_P.reserve((size_t)rows * n.out * 4));
    NFB_TRY(f->tr_gP.reserve((size_t)rows * n.out * 4));
    NFB_TRY(f->tr_ga.reserve((size_t)HS * 4));
    NFB_TRY(f->tr_gb.reserve((size_t)HS * 4));
    float* hb = f->tr_h.as<float>();
    float* Pm = f->tr_P.as<float>();
    float* gP = f->tr_gP.as<float>();
    float* ga = f->tr_ga.as<float>();
    float* gb = f->tr_gb.as<float>();
    // conditioner input: all columns (autoregressive) or the gathered identity columns (coupling)
    const float* in = xp;
    int ld_in = D;
    if (coupled) {
        NFB_TRY(f->tr_in.reserve((size_t)rows * L.n_id * 4));
        NFB_TRY(f->tr_gin.reserve((size_t)rows * L.n_id * 4));
        NFB_TRY(launch_gather_cols_ld(xp, D, f->tr_in.as<float>(), L.n_id, L.id_idx.as<int>(), rows, st));
        in = f->tr_in.as<float>();
        ld_in = L.n_id;
    }
    NFB_TRY(net_recompute(f, n, p, in, ld_in, rows, hb, Pm, st));
    // spline element backward -> gP, gxp (transformed columns)
    NFB_TRY(launch_spline_bwd_rows(xp, D, Pm, gy, glq, coupled ? L.tr_idx.as<int>() : nullptr, rows, T, L.K, L.tail,
                                   L.wh_scale, gP, gxp, st));
    f->launches++;
    const int nlin = 2 + 2 * n.nb;
    if (coupled) {
        NFB_TRY(f->tr_small.reserve((size_t)(64 * 64 + 64 * 23 + 64) * 4));
        float* gtab = f->tr_small.as<float>();
        NFB_CUDA(cudaMemsetAsync(gtab, 0, (size_t)L.n_id * P * 4, st));
        NFB_TRY(launch_spline_bwd_shared(xp, D, L.uncond.as<float>(), gy, glq, L.id_idx.as<int>(), rows, L.n_id, L.K, L.tail,
                                         gtab, gxp, st));
        NFB_TRY(launch_split_table(gtab, L.n_id, slots[2 * nlin], slots[2 * nlin + 1], slots[2 * nlin + 2], st));
        f->launches += 3;
    }
    Gemm g{f, st};
    // final layer
    float* hlast = hb + (size_t)(2 * n.nb) * HS;
    NFB_TRY(linear_wgrad(f, gP, n.out, hlast, H, H, 0, n.mf, rows, slots[2 * (nlin - 1)], slots[2 * (nlin - 1) + 1], st));
    {
        GemmTcArgs a{};
        a.A = gP; a.lda = n.out; a.B = p.wf; a.ldb = H; a.b_mn = 1; a.C = ga; a.ldc = H; a.M = rows; a.N = H; a.K = n.out;
        NFB_TRY(g.run_w(a));  // g_h(last)
    }
    for (int b = n.nb - 1; b >= 0; --b) {
        float* hprev = hb + (size_t)(2 * b) * HS;
        float* t = hb + (size_t)(2 * b + 1) * HS;
        const int l1 = 1 + 2 * b, l2 = 2 + 2 * b;  // linear indices of the block's two layers
        // h_next = h_prev + W2 relu(t) + b2
        NFB_TRY(linear_wgrad(f, ga, H, t, H, H, 1, n.mb[2 * b + 1], rows, slots[2 * l2], slots[2 * l2 + 1], st));
        GemmTcArgs a{};
        a.A = ga; a.lda = H; a.B = p.wb[2 * b + 1]; a.ldb = H; a.b_mn = 1; a.C = gb; a.ldc = H; a.M = rows; a.N = H; a.K = H;
        a.mask = t; a.ldmask = H;
        NFB_TRY(g.run_w(a));  // g_t = (g_h W2) * (t > 0)
        // t = W1 relu(h_prev) + b1
        NFB_TRY(linear_wgrad(f, gb, H, hprev, H, H, 1, n.mb[2 * b], rows, slots[2 * l1], slots[2 * l1 + 1], st));
        GemmTcArgs c{};
        c.A = gb; c.lda = H; c.B = p.wb[2 * b]; c.ldb = H; c.b_mn = 1; c.C = ga; c.ldc = H; c.M = rows; c.N = H; c.K = H;
        c.mask = hprev; c.ldmask = H; c.resid = ga; c.ldres = H;
        NFB_TRY(g.run_w(c));  // g_h_prev = g_h + (g_t W1) * (h_prev > 0)     (in place)
    }
    // initial layer
    NFB_TRY(linear_wgrad(f, ga, H, in, ld_in, n.in, 0, n.m0, rows, slots[0], slots[1], st));
    if (!coupled) {
        GemmTcArgs a{};
        a.A = ga; a.lda = H; a.B = p.w0; a.ldb = n.in; a.b_mn = 1; a.C = gxp; a.ldc = D; a.M = rows; a.N = D; a.K = H;
        a.resid = gxp; a.ldres = D;
        NFB_TRY(g.run_w(a));  // + conditioner path (in place)
    } else {
        GemmTcArgs a{};
        a.A = ga; a.lda = H; a.B = p.w0; a.ldb = n.in; a.b_mn = 1; a.C = f->tr_gin.as<float>(); a.ldc = L.n_id;
        a.M = rows; a.N = L.n_id; a.K = H;
        NFB_TRY(g.run(a));
        NFB_TRY(launch_scatter_cols(f->tr_gin.as<float>(), gxp, L.id_idx.as<int>(), rows, L.n_id, D, 1, st));
        f->launches++;
    }
    return NFB_OK;
}

// backward of LULinearPermute (density direction x' = W z[:, perm] + b): gxp = gradient w.r.t. x'; writes gradient
// w.r.t. z into gz.  glq_sum: device scalar sum of the upstream gradients on log_q (for logabsdet).
int lu_layer_backward(nfb_flow* f, Layer& L, const float* zin, const float* gxp, const float* glq_sum, long long rows,
                      float* gz, float* const* slots, cudaStream_t st) {
    const int D = L.D;
    NFB_TRY(f->tr_zp.reserve((size_t)rows * D * 4));
    NFB_TRY(f->tr_gzp.reserve((size_t)rows * D * 4));
    NFB_TRY(f->tr_small.reserve((size_t)(64 * 64 + 64 * 23 + 64) * 4));
    float* zp = f->tr_zp.as<float>();
    float* gzp = f->tr_gzp.as<float>();
    float* dW = f->tr_small.as<float>() + 64 * 23 + 64;
    Gemm g{f, st};
    NFB_TRY(launch_gather_cols(zin, zp, L.lu_perm.as<int>(), rows, D, 1, st));
    f->launches++;
    if (slots[0] || slots[1] || slots[2]) {
        GemmTcArgs a{};
        a.A = gxp; a.lda = D; a.a_mn = 1; a.B = zp; a.ldb = D; a.b_mn = 1; a.C = dW; a.ldc = D; a.M = D; a.N = D; a.K = rows;
        NFB_TRY(g.run(a));
        NFB_TRY(launch_lu_param_bwd(dW, L.lu.lower_entries, L.lu.upper_entries, L.lu.unconstrained_upper_diag, L.lu.eps, D,
                                    glq_sum, slots[0], slots[1], slots[2], st));
        f->launches++;
    }
    if (slots[3]) {
        NFB_CUDA(cudaMemsetAsync(slots[3], 0, (size_t)D * 4, st));
        NFB_TRY(launch_colsum(gxp, D, rows, D, slots[3], st));
        f->launches += 2;
    }
    GemmTcArgs a{};
    a.A = gxp; a.lda = D; a.B = L.lu_Wd.as<float>(); a.ldb = D; a.b_mn = 1; a.C = gzp; a.ldc = D; a.M = rows; a.N = D; a.K = D;
    NFB_TRY(g.run(a));
    NFB_TRY(launch_scatter_cols(gzp, gz, L.lu_perm.as<int>(), rows, D, D, 0, st));
    f->launches++;
    return NFB_OK;
}

}  // namespace

extern "C" {

int nfb_flow_num_grad_slots(const nfb_flow_t* f) {
    if (!f) return -1;
    int n = 0;
    for (auto& L : f->layers) {
        const int k = grad_slots_of(*L);
        if (k < 0) return -1;  // a layer kind without a native backward
        n += k;
    }
    return n + (f->base_loc ? 2 : 0);
}

int64_t nfb_flow_grad_slot_numel(const nfb_flow_t* f, int32_t slot) {
    if (!f || slot < 0) return -1;
    for (auto& L : f->layers) {
        const int k = grad_slots_of(*L);
        if (k < 0) return -1;
        if (slot < k) return grad_slot_numel(*L, slot);
        slot -= k;
    }
    return (f->base_loc && slot < 2) ? f->D : -1;
}

int nfb_flow_log_prob_backward(nfb_flow_t* f, const float* x, const float* g_logq, int64_t rows, float* log_q_out,
                               float* gx_out, float* const* grad_slots, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(f->base_loc && f->base_log_scale, NFB_ERR_STATE, "no base distribution set");
    NFB_CHECK(x && g_logq && grad_slots, NFB_ERR_ARG, "null pointer");
    const int n_slots = nfb_flow_num_grad_slots(f);
    NFB_CHECK(n_slots >= 0, NFB_ERR_UNSUPPORTED, "native backward covers spline blocks + LULinearPermute + DiagGaussian");
    if (rows == 0) return NFB_OK;
    cudaStream_t st = S(stream);
    const int D = f->D;
    const int ng = (int)f->groups.size();
    const size_t ZS = (size_t)rows * D;
    f->launches = 0;
    NFB_TRY(ensure_ws(f, rows));
    NFB_TRY(f->tr_store.reserve((size_t)(ng + 1) * ZS * 4));
    NFB_TRY(f->tr_glq.reserve((size_t)rows * 4 + 64));
    NFB_TRY(f->tr_g0.reserve(ZS * 4));
    NFB_TRY(f->tr_g1.reserve(ZS * 4));
    NFB_TRY(f->tr_xp.reserve(ZS * 4));
    NFB_TRY(f->tr_gxp.reserve(ZS * 4));
    float* store = f->tr_store.as<float>();
    float* lq = f->tr_glq.as<float>();  // scratch log_q when the caller does not want it
    float* glq_sum = lq + rows;          // (64-byte tail of the buffer)
    float* logq = log_q_out ? log_q_out : lq;
    // ---- forward, keeping every group's input (density order: groups last-to-first) ----
    NFB_CUDA(cudaMemcpyAsync(store, x, ZS * 4, cudaMemcpyDeviceToDevice, st));
    NFB_TRY(launch_fill(logq, rows, 0.f, st));
    if (f->stack_n == ng && ng > 0) {
        // all groups fused: ONE persistent launch, layer l writing its output to store[l + 1]
        NFB_TRY(launch_fused_stack(f, store, store + ZS, logq, rows, st, 0, (long long)ZS));
    } else {
        for (int k = 0; k < ng; ++k)
            NFB_TRY(run_group(f, f->groups[ng - 1 - k], NFB_INVERSE, store + (size_t)k * ZS, store + (size_t)(k + 1) * ZS,
                              logq, rows, st));
    }
    const float* zfin = store + (size_t)ng * ZS;
    NFB_TRY(launch_diag_gauss(zfin, f->base_loc, f->base_log_scale, logq, rows, D, 1, st));
    // ---- backward ----
    // slot offsets per layer
    std::vector<int> off(f->layers.size() + 1, 0);
    for (size_t i = 0; i < f->layers.size(); ++i) off[i + 1] = off[i] + grad_slots_of(*f->layers[i]);
    float* const* base_slots = grad_slots + off[f->layers.size()];
    NFB_CUDA(cudaMemsetAsync(glq_sum, 0, 4, st));
    NFB_TRY(launch_colsum(g_logq, 1, rows, 1, glq_sum, st));
    float* g = f->tr_g0.as<float>();
    float* g2 = f->tr_g1.as<float>();
    {
        float *t0 = nullptr, *t1 = nullptr;
        if (base_slots[0] || base_slots[1]) {
            NFB_TRY(f->tr_t0.reserve(ZS * 4));
            NFB_TRY(f->tr_t1.reserve(ZS * 4));
            t0 = f->tr_t0.as<float>(); t1 = f->tr_t1.as<float>();
        }
        NFB_TRY(launch_diag_gauss_bwd(zfin, f->base_loc, f->base_log_scale, g_logq, rows, D, g, t0, t1, st));
        for (int j = 0; j < 2; ++j)
            if (base_slots[j]) {
                NFB_CUDA(cudaMemsetAsync(base_slots[j], 0, (size_t)D * 4, st));
                NFB_TRY(launch_colsum(j == 0 ? t0 : t1, D, rows, D, base_slots[j], st));
            }
    }
    for (int k = ng - 1; k >= 0; --k) {
        Group& grp = f->groups[ng - 1 - k];
        const float* zin = store + (size_t)k * ZS;
        NFB_CHECK(grp.kind != G_AFFINE, NFB_ERR_UNSUPPORTED, "native backward: affine-family group");
        Layer& A = *f->layers[grp.first];
        Layer* Bl = grp.last != grp.first ? f->layers[grp.last].get() : nullptr;  // pair: first = spline block, last = LU
        Layer* R = (A.kind == L_AR_RQS || A.kind == L_COUPLED_RQS) ? &A : nullptr;
        Layer* U = A.kind == L_LU ? &A : Bl;
        NFB_CHECK(R || U, NFB_ERR_UNSUPPORTED, "native backward: unsupported layer in group");
        const float* xp = zin;
        if (R && U) {  // recompute the LU output (the spline block's input)
            NFB_TRY(launch_linear(zin, D, U->lu_perm.as<int>(), U->lu_Wd.as<float>(), U->lu.bias, nullptr, 0,
                                  f->tr_xp.as<float>(), D, rows, D, D, 0, 0, 0.f, st));
            xp = f->tr_xp.as<float>();
        }
        const float* gcur = g;
        if (R) {
            NFB_TRY(rqs_layer_backward(f, *R, xp, g, g_logq, rows, f->tr_gxp.as<float>(), grad_slots + off[grp.first], st));
            gcur = f->tr_gxp.as<float>();
        }
        if (U) {
            const int ui = (U == &A) ? grp.first : grp.last;
            NFB_TRY(lu_layer_backward(f, *U, zin, gcur, glq_sum, rows, g2, grad_slots + off[ui], st));
            std::swap(g, g2);
        } else {
            NFB_CUDA(cudaMemcpyAsync(g, gcur, ZS * 4, cudaMemcpyDeviceToDevice, st));
        }
    }
    if (gx_out) NFB_CUDA(cudaMemcpyAsync(gx_out, g, ZS * 4, cudaMemcpyDeviceToDevice, st));
    return NFB_OK;
}

}  // extern "C"
