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
#include "nfb_affine_wide.cuh"
#include "nfb_planar_bwd.cuh"

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

// Bump allocator over a caller's workspace, every piece 256-byte aligned; with base == nullptr it only sizes it.
struct Carver {
    char* base = nullptr;
    size_t off = 0;
    template <typename T> T* take(size_t count) {
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += (count * sizeof(T) + 255) / 256 * 256;
        return p;
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

enum LayerKind { L_AR_RQS, L_COUPLED_RQS, L_LU, L_MASKED_AFFINE, L_AFFINE_COUPLING, L_AFFINE_CONST, L_PERMUTE, L_PLANAR,
                 L_RADIAL };

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
    struct Gemm { DevBuf src_row, src_col, row_scale, recs_dev; const float* W; const float* M; int src_cols, n_pad, k_pad;
                  int max_rows = 0; std::vector<FusedRec> recs; };
    std::vector<int> hperm;  // sorted-by-degree order of the hidden units (identity for unmasked nets)
    int own[2][2] = {{-1, -1}, {-1, -1}};  // hidden output slices of each consumer warpgroup (FusedLayer::own)
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
    // planar / radial
    PlanarOp pop{};
};

enum GroupKind { G_FUSED_PAIR, G_FUSED, G_AFFINE, G_PLANAR, G_SINGLE };
struct Group {
    GroupKind kind; int first, last; DevBuf ops;
    // affine group, sampling-direction backward: workspace plan (units per row), per-op unit table and the weight
    // reduction's items (output pointers filled per call)
    bool bwd_planned = false;
    int units = 0;
    long long n_elem = 0;
    DevBuf bops;
    std::vector<AffRedItem> items;
    // planar group: the layers' descriptors (with their workspace plan), the reduction's items (outputs relative to the
    // sums, rebased per call), workspace units per row, and whether every layer has a density direction
    std::vector<PlanarOp> pops;
    bool invertible = true;
    // affine group over affine_stack_kernel's limits (kAffMaxD features, kAffMaxW net width): runs layer by layer on the
    // wide path, with scratch widths per row: wo the nets' outputs (at least D), hs / ht the hidden activations of the s
    // (param_map) / t nets, wy the widest Linear
    bool wide = false;
    int wo = 0, hs = 0, ht = 0, wy = 1;
};

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
    const float* base_weight_scores = nullptr;   // set: the base is a Gaussian mixture of base_modes modes
    int base_modes = 0;
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
    DevBuf tr_store, tr_net, tr_P, tr_gP, tr_xp, tr_gxp, tr_zp, tr_gzp, tr_in, tr_gin, tr_g0, tr_g1, tr_small, tr_glq,
        tr_t0, tr_t1, tr_wpack, tr_aff, tr_mix, aw_fwd;
    const int* cur_in_ready = nullptr;
    // affine sampling backward: the reduction items with this call's gradient pointers, staged through pinned memory
    AffRedItem* afb_host = nullptr;
    size_t afb_cap = 0;
    cudaEvent_t afb_ev = nullptr;
    DevBuf afb_items;
    // planar sampling backward: reduction items and per-layer gradient outputs of this call, staged the same way
    char* plb_host = nullptr;
    size_t plb_cap = 0;
    cudaEvent_t plb_ev = nullptr;
    DevBuf plb_dev;
    ~nfb_flow() {
        if (plb_ev) cudaEventDestroy(plb_ev);
        if (plb_host) cudaFreeHost(plb_host);
        if (afb_ev) cudaEventDestroy(afb_ev);
        if (afb_host) cudaFreeHost(afb_host);
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
    const int crow = fpc * 24;  // rows (MMA N) per final-layer chunk
    if (n_hidden > 7) return NFB_OK;  // tables inside FusedLayer

    // ---- MADE masks: sort hidden units by degree so that every masked matrix is block-triangular, and
    //      find the all-zero [64 x 64] blocks to drop (nfb_fused_plan.h) ----
    const bool masked = n.m0 != nullptr;
    std::vector<float> m_init, m_hid, m_fin;
    if (masked) {
        NFB_TRY(download(n.m0, (size_t)H * n.in, m_init));
        if (n.nb > 0) NFB_TRY(download(n.mb[0], (size_t)H * H, m_hid));  // all hidden masks share the structure
        NFB_TRY(download(n.mf, (size_t)n.out * H, m_fin));
    }
    const FusedNeeds needs = fused_needs(H, n.in, T, fpc, n_chunks, masked ? m_init.data() : nullptr,
                                         m_hid.empty() ? nullptr : m_hid.data(), masked ? m_fin.data() : nullptr);
    const std::vector<int>& perm = needs.perm;
    F.hperm = perm;

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

    // ---- slice ownership, step table and record list (nfb_fused_plan.h) ----
    FusedPlan plan = plan_fused(needs, n_hidden, crow);
    for (int g = 0; g <= n_hidden; ++g) F.gemms[g].recs = std::move(plan.recs[g]);
    std::copy(&plan.own[0][0], &plan.own[0][0] + 4, &F.own[0][0]);
    F.steps_host = plan.steps;
    F.n_steps = (int)plan.steps.size();
    F.D = L.D; F.H = H; F.n_hidden = n_hidden; F.T = T; F.F = fpc; F.n_chunks = n_chunks; F.tail = L.tail;
    F.n_id = ar ? 0 : L.n_id;
    F.rqs_bytes = plan.bytes;
    NFB_TRY(F.wstream.reserve(plan.bytes));
    NFB_TRY(F.steps.upload(plan.steps));

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
    for (int w = 0; w < 2; ++w)
        for (int q = 0; q < 2; ++q) Lh.own[w][q] = (signed char)F.own[w][q];
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

// the LU map in front of a block: one 64-row record W_hi | W_lo for warpgroup 0, all four products (the map transforms
// z itself, ~2^-22)
FusedStep lu_step() {
    FusedStep s{};
    s.bytes16 = 64 * 16; s.n8 = 8;
    s.kc = 0; s.flags = kStepFirst | kStepLast | kStepQuad | kStepHalf;
    s.kc1 = 0; s.flags1 = kStepFirst | kStepLast | kStepQuad | kStepHalf | kStepSkip;
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

bool is_planar_kind(const Layer& L) { return L.kind == L_PLANAR || L.kind == L_RADIAL; }

int copy_mlp(const nfb_mlp_desc_t& d, AffMlp& m, float* slope) {
    NFB_CHECK(d.num_layers >= 0 && d.num_layers <= kAffMaxLayers, NFB_ERR_UNSUPPORTED, "MLP: %d layers > %d", d.num_layers, kAffMaxLayers);
    m.n_layers = d.num_layers;
    if (d.num_layers == 0) return NFB_OK;   // absent net (MaskedAffineFlow with s or t = None)
    for (int i = 0; i <= d.num_layers; ++i) {
        NFB_CHECK(d.sizes[i] >= 1, NFB_ERR_ARG, "MLP: layer width %d < 1", d.sizes[i]);
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

int affine_wide_apply(nfb_flow* f, const Group& g, int first, int last, int dir, const float* zin, float* zout,
                      float* logdet, long long rows, cudaStream_t st);

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
        if (g.wide) return affine_wide_apply(f, g, g.first, g.last, direction, zin, zout, logdet, rows, st);
        NFB_TRY(launch_affine_stack(g.ops.p, g.last - g.first + 1, zin, zout, logdet, rows, f->D, 1, direction, st));
        f->launches++;
        return NFB_OK;
    case G_PLANAR:
        NFB_CHECK(direction == NFB_FORWARD || g.invertible, NFB_ERR_UNSUPPORTED, "This flow has no algebraic inverse.");
        NFB_TRY(launch_planar_stack(g.ops.p, g.last - g.first + 1, zin, zout, logdet, rows, f->D, 1, direction, st));
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

int nfb_gaussian_mixture_log_prob(const float* z, const float* loc, const float* log_scale, const float* weight_scores,
                                  float* log_q, int64_t rows, int32_t n_modes, int32_t dim, int32_t accumulate,
                                  void* stream) {
    NFB_CHECK(rows >= 0, NFB_ERR_ARG, "nfb_gaussian_mixture_log_prob: negative size");
    NFB_CHECK(rows == 0 || (z && loc && log_scale && weight_scores && log_q), NFB_ERR_ARG,
              "nfb_gaussian_mixture_log_prob: null pointer");
    return launch_mixture_log_prob(z, loc, log_scale, weight_scores, log_q, rows, n_modes, dim, accumulate, S(stream));
}

int64_t nfb_gaussian_mixture_log_prob_backward_workspace_bytes(int64_t rows, int32_t n_modes, int32_t dim) {
    if (rows < 0 || n_modes < 1 || dim < 1) return -1;
    return mixture_bwd_ws_bytes(rows, n_modes, dim);
}

int nfb_gaussian_mixture_log_prob_backward(const float* z, const float* loc, const float* log_scale,
                                           const float* weight_scores, const float* g_log_q, int64_t rows,
                                           int32_t n_modes, int32_t dim, void* ws, int64_t ws_bytes, float* g_z,
                                           float* g_loc, float* g_log_scale, float* g_weight_scores, void* stream) {
    NFB_CHECK(rows >= 0, NFB_ERR_ARG, "nfb_gaussian_mixture_log_prob_backward: negative size");
    NFB_CHECK(weight_scores && (rows == 0 || (z && loc && log_scale && g_log_q)), NFB_ERR_ARG,
              "nfb_gaussian_mixture_log_prob_backward: null pointer");
    return launch_mixture_bwd(z, loc, log_scale, weight_scores, g_log_q, rows, n_modes, dim, ws, ws_bytes, g_z, g_loc,
                              g_log_scale, g_weight_scores, S(stream));
}

int nfb_hmc_chain(const nfb_density_t* density, int64_t rows, int32_t transitions, int32_t leapfrog, float max_abs_grad,
                  const float* coef, const float* log_step_size, const float* log_mass, const float* noise,
                  const float* uniforms, const float* z, float* z_out, float* log_w, uint8_t* accept, void* stream) {
    NFB_CHECK(density, NFB_ERR_ARG, "nfb_hmc_chain: null density");
    return launch_hmc_chain(*density, rows, transitions, leapfrog, max_abs_grad, coef, log_step_size, log_mass, noise,
                            uniforms, z, z_out, log_w, accept, S(stream));
}

int64_t nfb_hmc_backward_workspace_bytes(int64_t rows, int32_t dim) {
    if (rows < 0 || dim < 1) return -1;
    return hmc_bwd_ws_bytes(rows, dim);
}

int nfb_hmc_backward(const nfb_density_t* density, int64_t rows, int32_t leapfrog, float max_abs_grad, const float* coef,
                     const float* log_step_size, const float* log_mass, const float* noise, const float* z,
                     const uint8_t* accept, const float* g_z_out, void* ws, int64_t ws_bytes, float* g_log_step_size,
                     float* g_log_mass, void* stream) {
    NFB_CHECK(density, NFB_ERR_ARG, "nfb_hmc_backward: null density");
    return launch_hmc_bwd(*density, rows, leapfrog, max_abs_grad, coef, log_step_size, log_mass, noise, z, accept,
                          g_z_out, ws, ws_bytes, g_log_step_size, g_log_mass, S(stream));
}

int nfb_mh_chain(const nfb_density_t* density, int64_t rows, int32_t steps, const float* coef, const float* scale,
                 const float* noise, const float* uniforms, const float* z, float* z_out, float* log_det, uint8_t* moved,
                 void* stream) {
    NFB_CHECK(density, NFB_ERR_ARG, "nfb_mh_chain: null density");
    return launch_mh_chain(*density, rows, steps, coef, scale, noise, uniforms, z, z_out, log_det, moved, S(stream));
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

int nfb_conv2d_wgrad(const float* x, int32_t x_channels, int32_t c0, const float* gy, float* gw, float* gb, int64_t batch,
                     int32_t cin, int32_t height, int32_t width, int32_t cout, int32_t ksize, int32_t accumulate,
                     void* stream) {
    NFB_CHECK(x && gy, NFB_ERR_ARG, "nfb_conv2d_wgrad: null pointer");
    return launch_conv2d_wgrad(x, x_channels, c0, gy, gw, gb, batch, cin, height, width, cout, ksize, accumulate, 0,
                               S(stream));
}
int nfb_conv2d_dgrad(const float* gy, const float* w, float* gx, int64_t batch, int32_t cin, int32_t height, int32_t width,
                     int32_t cout, int32_t ksize, const float* mask_act, float mask_slope, int32_t accumulate,
                     void* stream) {
    NFB_CHECK(gy && w && gx, NFB_ERR_ARG, "nfb_conv2d_dgrad: null pointer");
    return launch_conv2d_dgrad(gy, w, gx, batch, cin, height, width, cout, ksize, mask_act, mask_slope, accumulate,
                               S(stream));
}
int nfb_affine_coupling_image_backward(const float* z, const float* param, const float* g_out, const float* g_log_det,
                                       float* g_z, float* g_param, int64_t batch, int32_t channels, int32_t hw,
                                       int32_t scale, int32_t scale_map, int32_t split_mode, void* stream) {
    NFB_CHECK(z && param && g_out && g_z && g_param, NFB_ERR_ARG, "nfb_affine_coupling_image_backward: null pointer");
    NFB_CHECK(scale_map >= 0 && scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(split_mode == 0 || split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    return launch_coupling_image_bwd(z, param, g_out, g_log_det, g_z, g_param, batch, channels, hw, scale, scale_map,
                                     split_mode, S(stream));
}
int nfb_gaussian_table_log_prob_backward(const float* z, const int64_t* y, const float* loc, const float* log_scale,
                                         const float* g_log_q, float* g_z, float* g_loc, float* g_log_scale, int64_t batch,
                                         int32_t dim, int32_t group, int32_t num_classes, void* stream) {
    NFB_CHECK(z && loc && log_scale && g_log_q, NFB_ERR_ARG, "nfb_gaussian_table_log_prob_backward: null pointer");
    NFB_CHECK(y || num_classes == 1, NFB_ERR_ARG, "nfb_gaussian_table_log_prob_backward: labels needed for num_classes > 1");
    return launch_gauss_table_bwd(z, reinterpret_cast<const long long*>(y), loc, log_scale, g_log_q, g_z, g_loc,
                                  g_log_scale, batch, dim, group, num_classes, S(stream));
}
int nfb_logit_transform_backward(const float* in, const float* g_out, const float* g_log_det, float* g_in, int64_t batch,
                                 int64_t inner, float alpha, void* stream) {
    NFB_CHECK(in && g_in, NFB_ERR_ARG, "nfb_logit_transform_backward: null pointer");
    NFB_CHECK(alpha >= 0.f && alpha < 0.5f, NFB_ERR_ARG, "Logit: alpha must be in [0, 0.5)");
    return launch_logit_bwd(in, g_out, g_log_det, g_in, batch, inner, alpha, S(stream));
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

// ---- training pass of the residual block ----
int nfb_swish_dual(const float* H, const float* bias, float b, int64_t rows, int32_t width, int32_t nt, float* A,
                   void* stream) {
    NFB_CHECK(rows == 0 || (H && A), NFB_ERR_ARG, "nfb_swish_dual: null pointer");
    NFB_CHECK(rows >= 0 && width >= 1 && nt >= 0, NFB_ERR_ARG, "nfb_swish_dual: bad shape");
    return launch_swish_dual(H, bias, b, rows, width, nt, A, S(stream));
}
int nfb_swish_dual_adjoint(const float* H, const float* bias, float b, int64_t rows, int32_t width, int32_t nt,
                           const float* Abar, float* out_primal, float* out_tangent, double* partials, float* g_b,
                           void* stream) {
    NFB_CHECK(partials && (rows == 0 || (H && Abar)), NFB_ERR_ARG, "nfb_swish_dual_adjoint: null pointer");
    NFB_CHECK(rows >= 0 && width >= 1 && nt >= 0, NFB_ERR_ARG, "nfb_swish_dual_adjoint: bad shape");
    return launch_swish_dual_adjoint(H, bias, b, rows, width, nt, Abar, out_primal, out_tangent, partials, g_b, S(stream));
}
int nfb_logabsdet_i_plus_j_2x2_backward(const float* jt, const float* g_ld, int64_t batch, float* seeds, void* stream) {
    NFB_CHECK(batch == 0 || (jt && g_ld && seeds), NFB_ERR_ARG, "nfb_logabsdet_i_plus_j_2x2_backward: null pointer");
    return launch_logdet2_backward(jt, g_ld, batch, seeds, S(stream));
}

namespace {
// Scratch of the dual backward, carved from the caller's workspace:
//   H[l], l < L      stacked input of Swish l (= output of Linear l-1 without bias; H[0] = [x; tangents0])
//   A[l], l < L      stacked output of Swish l (the A operand of Linear l)      both [(1 + nt) rows, widths[l]]
//   Y0, Y1           cotangent ping-pong buffers                              [(1 + nt) rows, max width]
//   partials         per-CTA fp64 partial sums of the b gradient              [NFB_SWISH_DUAL_PARTIALS]
struct MlpDualWs {
    float* H[NFB_LIPSCHITZ_MLP_MAX_LAYERS]; float* A[NFB_LIPSCHITZ_MLP_MAX_LAYERS];
    float* Y[2]; double* partials;
};
int64_t mlp_dual_layout(const nfb_lipschitz_mlp_desc_t* d, int nt, long long rows, char* base, MlpDualWs* ws) {
    if (!d || d->num_layers < 1 || d->num_layers > NFB_LIPSCHITZ_MLP_MAX_LAYERS || nt < 0 || rows < 0) return -1;
    const long long rows2 = (1 + nt) * rows;
    Carver c{base};
    int wmax = 0;
    for (int l = 0; l <= d->num_layers; ++l) {
        if (d->widths[l] < 1) return -1;
        wmax = std::max(wmax, (int)d->widths[l]);
    }
    for (int l = 0; l < d->num_layers; ++l) {
        float* h = c.take<float>((size_t)rows2 * d->widths[l]);
        float* a = c.take<float>((size_t)rows2 * d->widths[l]);
        if (ws) { ws->H[l] = h; ws->A[l] = a; }
    }
    for (int i = 0; i < 2; ++i) {
        float* y = c.take<float>((size_t)rows2 * wmax);
        if (ws) ws->Y[i] = y;
    }
    double* p = c.take<double>(NFB_SWISH_DUAL_PARTIALS);
    if (ws) ws->partials = p;
    return (int64_t)c.off;
}
}  // namespace

int64_t nfb_lipschitz_mlp_dual_backward_workspace_bytes(const nfb_lipschitz_mlp_desc_t* d, int32_t nt, int64_t rows) {
    return mlp_dual_layout(d, nt, rows, nullptr, nullptr);
}

int nfb_lipschitz_mlp_dual_backward(const nfb_lipschitz_mlp_desc_t* d, const float* x, const float* tangents0, int32_t nt,
                                    const float* g_seed, const float* t_seeds, int64_t rows, void* workspace,
                                    int64_t workspace_bytes, float* gx, float* const* gW, float* const* gbias, float* gb,
                                    void* stream) {
    NFB_CHECK(d && workspace && (rows == 0 || x), NFB_ERR_ARG, "nfb_lipschitz_mlp_dual_backward: null pointer");
    NFB_CHECK(nt == 0 || rows == 0 || tangents0, NFB_ERR_ARG, "nfb_lipschitz_mlp_dual_backward: nt > 0 needs tangents0");
    const int64_t need = mlp_dual_layout(d, nt, rows, nullptr, nullptr);
    NFB_CHECK(need >= 0, NFB_ERR_ARG, "nfb_lipschitz_mlp_dual_backward: bad descriptor or shape");
    NFB_CHECK(workspace_bytes >= need, NFB_ERR_ARG, "nfb_lipschitz_mlp_dual_backward: workspace of %lld bytes, needs %lld",
              (long long)workspace_bytes, (long long)need);
    const int L = d->num_layers;
    for (int l = 0; l < L; ++l)
        NFB_CHECK(d->w[l] && d->bias[l], NFB_ERR_ARG, "nfb_lipschitz_mlp_dual_backward: null weight or bias");
    MlpDualWs ws{};
    mlp_dual_layout(d, nt, rows, static_cast<char*>(workspace), &ws);
    cudaStream_t st = S(stream);
    const int* w = d->widths;
    const long long rows2 = (1 + nt) * rows;
    const int D = w[0], out = w[L];
    if (rows == 0) {   // empty batch: every gradient is zero
        for (int l = 0; l < L; ++l) {
            if (gW && gW[l]) NFB_CUDA(cudaMemsetAsync(gW[l], 0, (size_t)w[l + 1] * w[l] * 4, st));
            if (gbias && gbias[l]) NFB_CUDA(cudaMemsetAsync(gbias[l], 0, (size_t)w[l + 1] * 4, st));
        }
        if (gb) NFB_CUDA(cudaMemsetAsync(gb, 0, (size_t)L * 4, st));
        return NFB_OK;
    }
    int* err_dev = nullptr;
    NFB_TRY(glow_err_buf(&err_dev));
    // dual forward (recompute): H[0] = [x; tangents0]; A[l] = swish_dual(H[l]); H[l+1] = A[l] W~_l^T (no bias)
    NFB_CUDA(cudaMemcpyAsync(ws.H[0], x, (size_t)rows * D * 4, cudaMemcpyDeviceToDevice, st));
    if (nt) NFB_CUDA(cudaMemcpyAsync(ws.H[0] + (size_t)rows * D, tangents0, (size_t)nt * rows * D * 4,
                                     cudaMemcpyDeviceToDevice, st));
    for (int l = 0; l < L; ++l) {
        NFB_TRY(launch_swish_dual(ws.H[l], l ? d->bias[l - 1] : nullptr, d->b[l], rows, w[l], nt, ws.A[l], st));
        if (l + 1 == L) break;   // the network's output is not needed by the adjoint
        GemmTcArgs a{};
        a.A = ws.A[l]; a.lda = w[l]; a.B = d->w[l]; a.ldb = w[l]; a.C = ws.H[l + 1]; a.ldc = w[l + 1];
        a.M = rows2; a.N = w[l + 1]; a.K = w[l];
        NFB_TRY(launch_gemm_tc(a, err_dev, st));
    }
    // seeds: Y = [g_seed; t_seeds] (zero where absent)
    float* Y = ws.Y[0];
    if (g_seed) NFB_CUDA(cudaMemcpyAsync(Y, g_seed, (size_t)rows * out * 4, cudaMemcpyDeviceToDevice, st));
    else NFB_CUDA(cudaMemsetAsync(Y, 0, (size_t)rows * out * 4, st));
    if (nt) {
        float* ty = Y + (size_t)rows * out;
        if (t_seeds) NFB_CUDA(cudaMemcpyAsync(ty, t_seeds, (size_t)nt * rows * out * 4, cudaMemcpyDeviceToDevice, st));
        else NFB_CUDA(cudaMemsetAsync(ty, 0, (size_t)nt * rows * out * 4, st));
    }
    // adjoint, Linear l and Swish l from the output back to the input
    for (int l = L - 1; l >= 0; --l) {
        const int n_out = w[l + 1], n_in = w[l];
        if (gW && gW[l]) {   // gW~_l = Y^T A[l], reduced over all (1 + nt) rows stacks
            GemmTcArgs a{};
            a.A = Y; a.lda = n_out; a.a_mn = 1; a.B = ws.A[l]; a.ldb = n_in; a.b_mn = 1;
            a.C = gW[l]; a.ldc = n_in; a.M = n_out; a.N = n_in; a.K = rows2;
            NFB_TRY(launch_gemm_tc(a, err_dev, st));
        }
        if (gbias && gbias[l]) {   // primal rows only
            NFB_CUDA(cudaMemsetAsync(gbias[l], 0, (size_t)n_out * 4, st));
            NFB_TRY(launch_colsum(Y, n_out, rows, n_out, gbias[l], st));
        }
        float* Abar = ws.Y[(L - l) & 1];   // the other buffer
        GemmTcArgs a{};   // [abar; tabar] = Y W~_l
        a.A = Y; a.lda = n_out; a.B = d->w[l]; a.ldb = n_in; a.b_mn = 1; a.C = Abar; a.ldc = n_in;
        a.M = rows2; a.N = n_in; a.K = n_out;
        NFB_TRY(launch_gemm_tc(a, err_dev, st));
        float* outp = l ? Abar : gx;
        float* outt = l ? Abar + (size_t)rows * n_in : nullptr;
        NFB_TRY(launch_swish_dual_adjoint(ws.H[l], l ? d->bias[l - 1] : nullptr, d->b[l], rows, n_in, nt, Abar, outp, outt,
                                          ws.partials, gb ? gb + l : nullptr, st));
        Y = Abar;
    }
    return NFB_OK;
}

// ---- training pass of the stand-alone layers (splines, conditioners called as modules, periodic features) ----
static int spline_backward(const char* who, const float* x, const float* params, int64_t stride, const float* gy,
                           const float* gld, float* gx, float* gp, int64_t rows, int32_t feats, int32_t K, int32_t nd,
                           const float* tail, const int32_t* circ, float tail0, float wh_scale, void* stream,
                           bool inverse = false) {
    NFB_CHECK(rows >= 0 && feats >= 0, NFB_ERR_ARG, "%s: negative size", who);
    NFB_CHECK(K >= 1 && K <= 32 && (nd == K - 1 || nd == K || nd == K + 1), NFB_ERR_ARG, "%s: bad bins / derivatives",
              who);
    const int64_t P = 2 * (int64_t)K + nd;
    NFB_CHECK(stride == 0 || stride == feats * P, NFB_ERR_ARG,
              "%s: params_row_stride must be 0 (shared table) or feats * (2 num_bins + num_derivatives)", who);
    NFB_CHECK(params && (rows == 0 || feats == 0 || x), NFB_ERR_ARG, "%s: null pointer", who);
    if (inverse)
        return launch_spline_inverse_adjoint(x, params, stride == 0, gy, nullptr, gld, rows, feats, K, nd, tail, circ,
                                             tail0, wh_scale, gp, gx, S(stream));
    return launch_spline_adjoint(x, params, stride == 0, gy, gld, rows, feats, K, nd, tail, circ, tail0, wh_scale, gp, gx,
                                 S(stream));
}
int nfb_rqs_spline_backward(const float* x, const float* params, int64_t params_row_stride, const float* g_y,
                            const float* g_log_det, float* g_x, float* g_params, int64_t rows, int32_t feats,
                            int32_t num_bins, float tail_bound, float wh_scale, void* stream) {
    return spline_backward("nfb_rqs_spline_backward", x, params, params_row_stride, g_y, g_log_det, g_x, g_params, rows,
                           feats, num_bins, num_bins - 1, nullptr, nullptr, tail_bound, wh_scale, stream);
}
int nfb_rqs_spline_tails_backward(const float* x, const float* params, int64_t params_row_stride, const float* g_y,
                                  const float* g_log_det, float* g_x, float* g_params, int64_t rows, int32_t feats,
                                  int32_t num_bins, int32_t num_derivatives, const float* tail_bound,
                                  const int32_t* circular, float wh_scale, void* stream) {
    NFB_CHECK(tail_bound && circular, NFB_ERR_ARG, "nfb_rqs_spline_tails_backward: null pointer");
    NFB_CHECK(num_derivatives != num_bins - 1, NFB_ERR_ARG,
              "nfb_rqs_spline_tails_backward: %d derivative parameters for %d bins", num_derivatives, num_bins);
    return spline_backward("nfb_rqs_spline_tails_backward", x, params, params_row_stride, g_y, g_log_det, g_x, g_params,
                           rows, feats, num_bins, num_derivatives, tail_bound, circular, 0.f, wh_scale, stream);
}
int nfb_rqs_spline_inverse_backward(const float* z, const float* params, int64_t params_row_stride, const float* g_x,
                                    const float* g_log_det, float* g_z, float* g_params, int64_t rows, int32_t feats,
                                    int32_t num_bins, float tail_bound, float wh_scale, void* stream) {
    return spline_backward("nfb_rqs_spline_inverse_backward", z, params, params_row_stride, g_x, g_log_det, g_z, g_params,
                           rows, feats, num_bins, num_bins - 1, nullptr, nullptr, tail_bound, wh_scale, stream, true);
}
int nfb_rqs_spline_tails_inverse_backward(const float* z, const float* params, int64_t params_row_stride,
                                          const float* g_x, const float* g_log_det, float* g_z, float* g_params,
                                          int64_t rows, int32_t feats, int32_t num_bins, int32_t num_derivatives,
                                          const float* tail_bound, const int32_t* circular, float wh_scale,
                                          void* stream) {
    NFB_CHECK(tail_bound && circular, NFB_ERR_ARG, "nfb_rqs_spline_tails_inverse_backward: null pointer");
    NFB_CHECK(num_derivatives != num_bins - 1, NFB_ERR_ARG,
              "nfb_rqs_spline_tails_inverse_backward: %d derivative parameters for %d bins", num_derivatives, num_bins);
    return spline_backward("nfb_rqs_spline_tails_inverse_backward", z, params, params_row_stride, g_x, g_log_det, g_z,
                           g_params, rows, feats, num_bins, num_derivatives, tail_bound, circular, 0.f, wh_scale, stream,
                           true);
}
int nfb_periodic_features_backward(const float* x, const float* g_y, int64_t rows, int32_t dim, const int32_t* slot,
                                   const float* weights, const float* scale, int32_t n_periodic, float* g_x,
                                   float* g_weights, float* g_bias, void* stream) {
    NFB_CHECK(rows >= 0 && dim >= 0 && n_periodic >= 0, NFB_ERR_ARG, "nfb_periodic_features_backward: negative size");
    NFB_CHECK(slot && weights && scale && (rows == 0 || dim == 0 || (x && g_y)), NFB_ERR_ARG,
              "nfb_periodic_features_backward: null pointer");
    return launch_periodic_features_bwd(x, g_y, rows, dim, slot, weights, scale, n_periodic, g_x, g_weights, g_bias,
                                        S(stream));
}
int nfb_glu_residual_backward(const float* g_out, const float* t, const float* c, int64_t n, float* g_h, float* g_t,
                              float* g_c, void* stream) {
    NFB_CHECK(n >= 0 && (n == 0 || (g_out && t && c)), NFB_ERR_ARG, "nfb_glu_residual_backward: null pointer");
    return launch_glu_residual_bwd(g_out, t, c, n, g_h, g_t, g_c, S(stream));
}

namespace {
// Scratch of the ResidualNet / MADE backward.  H = hidden, nb = blocks, C = context features:
//   in0   [rows, in]  ResidualNet with a context: cat(x, context), the initial layer's input; later its data gradient
//   weff  masked effective weights W * mask of every Linear (MADE whose caller brings no effective weights)
//   h[b]  [rows, H], b <= nb: input of block b (h[nb] = the final layer's input)
//   t1[b], t2[b], c[b] [rows, H]: block b's first / second Linear output and its context gate logits (t2, c: context)
//   ga, gt, gt1 [rows, H]: cotangents (gt: context);  gc0 [rows, C]: context columns of in0's gradient (ResidualNet
//   with a context)
struct ResnetWs {
    float* in0; float* gc0; float* w0e; float* wfe;
    std::vector<float*> wbe, h, t1, t2, c;
    float* ga; float* gt; float* gt1;
};
int64_t resnet_layout(const nfb_resnet_ctx_desc_t* d, long long rows, Carver& c, ResnetWs& ws, bool weff = true) {
    if (!d || rows < 0) return -1;
    const nfb_resnet_desc_t& n = d->net;
    const int nb = n.num_blocks, H = n.hidden_features, C = d->context_features;
    if (nb < 0 || H < 1 || n.in_features < 1 || n.out_features < 1 || C < 0) return -1;
    const bool concat = C > 0 && !d->w_context;
    if (concat && n.in_features <= C) return -1;
    const size_t RH = (size_t)rows * H;
    ws = ResnetWs{};
    ws.in0 = concat ? c.take<float>((size_t)rows * n.in_features) : nullptr;
    ws.gc0 = concat ? c.take<float>((size_t)rows * C) : nullptr;
    if (weff && n.m_initial) {
        ws.w0e = c.take<float>((size_t)H * n.in_features);
        for (int i = 0; i < 2 * nb; ++i) ws.wbe.push_back(c.take<float>((size_t)H * H));
        ws.wfe = c.take<float>((size_t)n.out_features * H);
    }
    for (int b = 0; b <= nb; ++b) ws.h.push_back(c.take<float>(RH));
    for (int b = 0; b < nb; ++b) {
        ws.t1.push_back(c.take<float>(RH));
        if (C > 0) { ws.t2.push_back(c.take<float>(RH)); ws.c.push_back(c.take<float>(RH)); }
    }
    ws.ga = c.take<float>(RH);
    if (C > 0) ws.gt = c.take<float>(RH);
    ws.gt1 = c.take<float>(RH);
    return (int64_t)c.off;
}

// Launches the tensor-core GEMMs of a backward.  Optional: wpack, a buffer into which a GEMM whose B is a weight
// (reused by every 128-row tile of the batch) splits B to bf16 hi | lo records once (launch_gemm_pack_b), so that
// the GEMM streams them by TMA instead of converting them per tile; launches, a counter of the kernels and memsets
// issued.
struct GemmRun {
    int* err; cudaStream_t st;
    DevBuf* wpack = nullptr;
    long long* launches = nullptr;
    void count(int k) const { if (launches) *launches += k; }
    int operator()(const GemmTcArgs& a) const { count(1); return launch_gemm_tc(a, err, st); }
    int w(GemmTcArgs a) const {   // B is a weight
        if (!wpack) return (*this)(a);
        NFB_TRY(wpack->reserve(gemm_tc_packed_b_bytes(a.N, a.K, a.b_mn)));
        NFB_TRY(launch_gemm_pack_b(a.B, a.ldb, a.b_mn, a.N, a.K, wpack->as<uint8_t>(), st));
        a.b_packed = wpack->as<uint8_t>();
        count(2);
        return launch_gemm_tc(a, err, st);
    }
};
// Y = act(X) W^T (+ bias) (+ resid) (the forward of one Linear)
GemmTcArgs fwd_args(const float* X, long long ldx, int relu_x, const float* W, const float* bias, float* Y, long long M,
                    int N, int K) {
    GemmTcArgs a{};
    a.A = X; a.lda = ldx; a.a_relu = relu_x; a.B = W; a.ldb = K; a.C = Y; a.ldc = N; a.M = M; a.N = N; a.K = K; a.bias = bias;
    return a;
}
// gX = gY W  (dgrad)
GemmTcArgs dgrad_args(const float* gY, const float* W, float* gX, long long M, int n_in, int n_out) {
    GemmTcArgs a{};
    a.A = gY; a.lda = n_out; a.B = W; a.ldb = n_in; a.b_mn = 1; a.C = gX; a.ldc = n_in; a.M = M; a.N = n_in; a.K = n_out;
    return a;
}
// dW = gY^T act(X) (* mask), db = colsum(gY); accumulate: added to dW and db
int wgrad(const GemmRun& g, const float* gY, int n_out, const float* X, long long ldx, int n_in, int relu_x,
          const float* mask, long long rows, float* dW, float* db, int accumulate = 0) {
    if (dW) {
        GemmTcArgs a{};
        a.A = gY; a.lda = n_out; a.a_mn = 1; a.B = X; a.ldb = ldx; a.b_mn = 1; a.b_relu = relu_x;
        a.C = dW; a.ldc = n_in; a.M = n_out; a.N = n_in; a.K = rows; a.mulm = mask; a.ldmask = n_in;
        a.accumulate = accumulate;
        NFB_TRY(g(a));
    }
    if (db) {
        if (!accumulate) { NFB_CUDA(cudaMemsetAsync(db, 0, (size_t)n_out * 4, g.st)); g.count(1); }
        NFB_TRY(launch_colsum(gY, n_out, rows, n_out, db, g.st));
        g.count(1);
    }
    return NFB_OK;
}
}  // namespace

namespace {
// One backward of a ResidualNet / MADE: the effective weights, the recomputed activations (ws, laid out by the caller)
// and the initial layer's input, shared by every adjoint run on them (nfb_maf_inverse_backward runs several on one
// recompute).  A caller that keeps its own effective weights sets w0 / wb / wf before resnet_recompute.
struct ResnetPass {
    const nfb_resnet_ctx_desc_t* d;
    long long rows;
    GemmRun g;
    ResnetWs ws;
    const float* w0; const float* wf; std::vector<const float*> wb;
    const float* in; long long ld_in;   // x, or cat(x, context) in ws.in0
};

// Gradient pointers of Linear i at p[i * stride]; p == nullptr: none wanted.
struct Slots {
    float* const* p = nullptr;
    int stride = 1;
    Slots(float* const* p_ = nullptr, int stride_ = 1) : p(p_), stride(stride_) {}
    float* operator[](int i) const { return p ? p[(size_t)i * stride] : nullptr; }
};

int resnet_validate(const char* who, const nfb_resnet_ctx_desc_t* d, int64_t rows, const float* x, const float* context,
                    const float* g_out, void* workspace, int64_t workspace_bytes, int64_t need) {
    NFB_CHECK(need >= 0, NFB_ERR_ARG, "%s: bad descriptor or shape", who);
    NFB_CHECK(workspace_bytes >= need && (need == 0 || workspace), NFB_ERR_ARG, "%s: workspace of %lld bytes, needs %lld",
              who, (long long)workspace_bytes, (long long)need);
    const nfb_resnet_desc_t& n = d->net;
    const int nb = n.num_blocks;
    const bool ctx = d->context_features > 0, masked = n.m_initial != nullptr;
    NFB_CHECK(n.w_initial && n.b_initial && n.w_final && n.b_final && (nb == 0 || (n.w_blocks && n.b_blocks)),
              NFB_ERR_ARG, "%s: null weight or bias", who);
    NFB_CHECK(!masked || (n.m_final && (nb == 0 || n.m_blocks)), NFB_ERR_ARG, "%s: missing masks", who);
    NFB_CHECK(!ctx || ((d->w_context ? d->b_context != nullptr : true) &&
                       (nb == 0 || (d->w_block_context && d->b_block_context))),
              NFB_ERR_ARG, "%s: null context layer", who);
    NFB_CHECK(rows == 0 || (x && g_out && (!ctx || context)), NFB_ERR_ARG, "%s: null input", who);
    return NFB_OK;
}

// empty batch: every parameter gradient is zero
int resnet_zero_grads(const nfb_resnet_ctx_desc_t* d, Slots g_w, Slots g_b, Slots g_wc, Slots g_bc, cudaStream_t st) {
    const nfb_resnet_desc_t& n = d->net;
    const int nb = n.num_blocks, H = n.hidden_features, C = d->context_features, out = n.out_features, nin = n.in_features;
    auto zero = [&](float* p, size_t numel) { return p ? (int)cudaMemsetAsync(p, 0, numel * 4, st) : 0; };
    auto wsz = [&](int i) { return (size_t)H * (i == 0 ? nin : H); };  // weights of linear i < 1 + 2 nb
    for (int i = 0; i < 1 + 2 * nb; ++i) {
        NFB_CUDA((cudaError_t)zero(g_w[i], wsz(i)));
        NFB_CUDA((cudaError_t)zero(g_b[i], H));
    }
    NFB_CUDA((cudaError_t)zero(g_w[1 + 2 * nb], (size_t)out * H));
    NFB_CUDA((cudaError_t)zero(g_b[1 + 2 * nb], out));
    if (C > 0)
        for (int i = 0; i <= nb; ++i) {
            NFB_CUDA((cudaError_t)zero(g_wc[i], (size_t)H * C));
            NFB_CUDA((cudaError_t)zero(g_bc[i], H));
        }
    return NFB_OK;
}

// Effective weights (unless the caller set them) and the activations of the forward at x / context (the same GEMMs
// as the forward, nets/*.forward through nfb_gemm_f32).  rows > 0.
int resnet_recompute(ResnetPass& r, const float* x, const float* context) {
    const nfb_resnet_ctx_desc_t* d = r.d;
    const nfb_resnet_desc_t& n = d->net;
    const long long rows = r.rows;
    const int nb = n.num_blocks, H = n.hidden_features, C = d->context_features, out = n.out_features;
    const bool ctx = C > 0, concat = ctx && !d->w_context, masked = n.m_initial != nullptr;
    const int nin = n.in_features, nx = concat ? nin - C : nin;
    const ResnetWs& ws = r.ws;
    const GemmRun& g = r.g;
    cudaStream_t st = g.st;
    if (!r.w0) {
        r.w0 = n.w_initial; r.wf = n.w_final;
        r.wb.assign(n.w_blocks, n.w_blocks + 2 * nb);
        if (masked) {
            NFB_TRY(launch_mask_mul(n.w_initial, n.m_initial, ws.w0e, (long long)H * nin, st));
            for (int i = 0; i < 2 * nb; ++i)
                NFB_TRY(launch_mask_mul(n.w_blocks[i], n.m_blocks[i], ws.wbe[i], (long long)H * H, st));
            NFB_TRY(launch_mask_mul(n.w_final, n.m_final, ws.wfe, (long long)out * H, st));
            r.w0 = ws.w0e; r.wf = ws.wfe;
            r.wb.assign(ws.wbe.begin(), ws.wbe.end());
        }
    }
    r.in = x;
    r.ld_in = nin;
    if (concat) {
        NFB_CUDA(cudaMemcpy2DAsync(ws.in0, (size_t)nin * 4, x, (size_t)nx * 4, (size_t)nx * 4, rows,
                                   cudaMemcpyDeviceToDevice, st));
        NFB_CUDA(cudaMemcpy2DAsync(ws.in0 + nx, (size_t)nin * 4, context, (size_t)C * 4, (size_t)C * 4, rows,
                                   cudaMemcpyDeviceToDevice, st));
        r.in = ws.in0;
    }
    NFB_TRY(g.w(fwd_args(r.in, r.ld_in, 0, r.w0, n.b_initial, ws.h[0], rows, H, nin)));
    if (ctx && !concat) {
        GemmTcArgs a = fwd_args(context, C, 0, d->w_context, d->b_context, ws.h[0], rows, H, C);
        a.resid = ws.h[0]; a.ldres = H;
        NFB_TRY(g.w(a));
    }
    for (int b = 0; b < nb; ++b) {
        NFB_TRY(g.w(fwd_args(ws.h[b], H, 1, r.wb[2 * b], n.b_blocks[2 * b], ws.t1[b], rows, H, H)));
        if (!ctx) {
            GemmTcArgs a = fwd_args(ws.t1[b], H, 1, r.wb[2 * b + 1], n.b_blocks[2 * b + 1], ws.h[b + 1], rows, H, H);
            a.resid = ws.h[b]; a.ldres = H;
            NFB_TRY(g.w(a));
        } else {
            NFB_TRY(g.w(fwd_args(ws.t1[b], H, 1, r.wb[2 * b + 1], n.b_blocks[2 * b + 1], ws.t2[b], rows, H, H)));
            NFB_TRY(g.w(fwd_args(context, C, 0, d->w_block_context[b], d->b_block_context[b], ws.c[b], rows, H, C)));
            NFB_TRY(launch_glu_residual(ws.h[b], ws.t2[b], ws.c[b], (long long)rows * H, ws.h[b + 1], st));
        }
    }
    return NFB_OK;
}

// Adjoint of the recomputed net for the output cotangent g_out.  data_only: the data gradient g_x alone -- no weight
// gradient, no bias column sum, no context GEMM, no context gradient (g_context and the g_* arrays are ignored).
// g_x_add (no concatenated context): g_x += the data gradient, through the GEMM's resid epilogue.
int resnet_adjoint(const ResnetPass& r, const float* context, const float* g_out, bool data_only, float* g_x,
                   float* g_context, Slots g_w, Slots g_b, Slots g_wc, Slots g_bc, bool g_x_add = false) {
    if (data_only) { g_context = nullptr; g_w = g_b = g_wc = g_bc = Slots(); }
    const nfb_resnet_ctx_desc_t* d = r.d;
    const nfb_resnet_desc_t& n = d->net;
    const long long rows = r.rows;
    const int nb = n.num_blocks, H = n.hidden_features, C = d->context_features, out = n.out_features;
    const bool ctx = C > 0, concat = ctx && !d->w_context, masked = n.m_initial != nullptr;
    const int nin = n.in_features, nx = concat ? nin - C : nin;
    const ResnetWs& ws = r.ws;
    const GemmRun& g = r.g;
    cudaStream_t st = g.st;
    auto mask_of = [&](int i) -> const float* {   // linear i: 0 initial, 1 + j block linear j, 1 + 2 nb final
        if (!masked) return nullptr;
        return i == 0 ? n.m_initial : (i == 1 + 2 * nb ? n.m_final : n.m_blocks[i - 1]);
    };
    if (g_context) NFB_CUDA(cudaMemsetAsync(g_context, 0, (size_t)rows * C * 4, st));
    auto ctx_layer = [&](const float* gY, const float* W, int slot) -> int {   // a Linear of the context
        NFB_TRY(wgrad(g, gY, H, context, C, C, 0, nullptr, rows, g_wc[slot], g_bc[slot]));
        if (g_context) {
            GemmTcArgs a = dgrad_args(gY, W, g_context, rows, C, H);
            a.accumulate = 1;
            NFB_TRY(g.w(a));
        }
        return NFB_OK;
    };
    const int fl = 1 + 2 * nb;
    NFB_TRY(wgrad(g, g_out, out, ws.h[nb], H, H, 0, mask_of(fl), rows, g_w[fl], g_b[fl]));
    NFB_TRY(g.w(dgrad_args(g_out, r.wf, ws.ga, rows, H, out)));
    for (int b = nb - 1; b >= 0; --b) {
        const int l1 = 1 + 2 * b, l2 = 2 + 2 * b;
        const float* gt2 = ws.ga;  // h_{b+1} = h_b + t2 (no context)
        if (ctx) {                 // h_{b+1} = h_b + t2 * sigmoid(c)
            NFB_TRY(launch_glu_residual_bwd(ws.ga, ws.t2[b], ws.c[b], (long long)rows * H, nullptr, ws.gt,
                                            data_only ? nullptr : ws.gt1, st));
            if (!data_only) NFB_TRY(ctx_layer(ws.gt1, d->w_block_context[b], 1 + b));
            gt2 = ws.gt;
        }
        // t2 = W2 relu(t1) + b2
        NFB_TRY(wgrad(g, gt2, H, ws.t1[b], H, H, 1, mask_of(l2), rows, g_w[l2], g_b[l2]));
        GemmTcArgs a = dgrad_args(gt2, r.wb[2 * b + 1], ws.gt1, rows, H, H);
        a.mask = ws.t1[b]; a.ldmask = H;
        NFB_TRY(g.w(a));   // g_t1 = (g_t2 W2) * (t1 > 0)
        // t1 = W1 relu(h_b) + b1
        NFB_TRY(wgrad(g, ws.gt1, H, ws.h[b], H, H, 1, mask_of(l1), rows, g_w[l1], g_b[l1]));
        GemmTcArgs c = dgrad_args(ws.gt1, r.wb[2 * b], ws.ga, rows, H, H);
        c.mask = ws.h[b]; c.ldmask = H; c.resid = ws.ga; c.ldres = H;
        NFB_TRY(g.w(c));   // g_h_b = g_h_{b+1} + (g_t1 W1) * (h_b > 0)     (in place)
    }
    NFB_TRY(wgrad(g, ws.ga, H, r.in, r.ld_in, nin, 0, mask_of(0), rows, g_w[0], g_b[0]));
    if (ctx && !concat && !data_only) NFB_TRY(ctx_layer(ws.ga, d->w_context, 0));
    if (concat) {
        if (g_x || g_context) {
            NFB_TRY(g.w(dgrad_args(ws.ga, r.w0, ws.in0, rows, nin, H)));   // [g_x | g_context] of cat(x, context)
            if (g_x)
                NFB_CUDA(cudaMemcpy2DAsync(g_x, (size_t)nx * 4, ws.in0, (size_t)nin * 4, (size_t)nx * 4, rows,
                                           cudaMemcpyDeviceToDevice, st));
            if (g_context) {   // += the context columns (g_context holds the block context layers' share)
                NFB_CUDA(cudaMemcpy2DAsync(ws.gc0, (size_t)C * 4, ws.in0 + nx, (size_t)nin * 4, (size_t)C * 4, rows,
                                           cudaMemcpyDeviceToDevice, st));
                NFB_TRY(launch_axpy(ws.gc0, 1.f, g_context, (long long)rows * C, 1, st));
            }
        }
    } else if (g_x) {
        GemmTcArgs a = dgrad_args(ws.ga, r.w0, g_x, rows, nin, H);
        if (g_x_add) { a.resid = g_x; a.ldres = nin; }
        NFB_TRY(g.w(a));
    }
    return NFB_OK;
}

// Scratch of nfb_maf_inverse_backward: the conditioner's (resnet_layout), then
//   P    [rows, 2 D]  MADE(y, context), the conditioner output at the layer's output
//   pbar [rows, 2 D]  its cotangent
//   gin  [rows, D]    MADE data gradient of the latest fixed-point pass
int64_t maf_layout(const nfb_resnet_ctx_desc_t* d, int32_t features, long long rows, char* base, ResnetWs& ws, float** P,
                   float** pbar, float** gin) {
    Carver c{base};
    if (resnet_layout(d, rows, c, ws) < 0 || features < 1) return -1;
    float* p = c.take<float>((size_t)rows * 2 * features); if (P) *P = p;
    p = c.take<float>((size_t)rows * 2 * features); if (pbar) *pbar = p;
    p = c.take<float>((size_t)rows * features); if (gin) *gin = p;
    return (int64_t)c.off;
}
}  // namespace

int64_t nfb_resnet_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* d, int64_t rows) {
    Carver c;
    ResnetWs ws;
    return resnet_layout(d, rows, c, ws);
}

int nfb_resnet_backward(const nfb_resnet_ctx_desc_t* d, const float* x, const float* context, const float* g_out,
                        int64_t rows, void* workspace, int64_t workspace_bytes, float* g_x, float* g_context,
                        float* const* g_w, float* const* g_b, float* const* g_wc, float* const* g_bc, void* stream) {
    NFB_TRY(resnet_validate("nfb_resnet_backward", d, rows, x, context, g_out, workspace, workspace_bytes,
                            nfb_resnet_backward_workspace_bytes(d, rows)));
    cudaStream_t st = S(stream);
    if (rows == 0) return resnet_zero_grads(d, g_w, g_b, g_wc, g_bc, st);
    ResnetPass r{d, rows, {nullptr, st}};
    NFB_TRY(glow_err_buf(&r.g.err));
    Carver c{static_cast<char*>(workspace)};
    resnet_layout(d, rows, c, r.ws);
    NFB_TRY(resnet_recompute(r, x, context));
    return resnet_adjoint(r, context, g_out, false, g_x, g_context, g_w, g_b, g_wc, g_bc);
}

int64_t nfb_maf_inverse_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* d, int32_t features, int64_t rows) {
    ResnetWs ws;
    return maf_layout(d, features, rows, nullptr, ws, nullptr, nullptr, nullptr);
}

int nfb_maf_inverse_backward(const nfb_resnet_ctx_desc_t* d, int32_t features, const float* x, const float* y,
                             const float* context, const float* g_y, const float* g_log_det, int64_t rows,
                             void* workspace, int64_t workspace_bytes, float* g_x, float* g_context, float* const* g_w,
                             float* const* g_b, float* const* g_wc, float* const* g_bc, void* stream) {
    const char* who = "nfb_maf_inverse_backward";
    NFB_CHECK(d && d->net.m_initial, NFB_ERR_ARG, "%s: the descriptor must be a MADE (mask pointers set)", who);
    NFB_CHECK(features >= 1 && d->net.in_features == features && d->net.out_features == 2 * features, NFB_ERR_ARG,
              "%s: a MADE of %d -> %d features does not parameterise %d features", who, d->net.in_features,
              d->net.out_features, features);
    NFB_CHECK(d->context_features == 0 || d->w_context, NFB_ERR_ARG, "%s: a MADE takes its context through w_context",
              who);
    NFB_TRY(resnet_validate(who, d, rows, y, context, x /* g_y and g_log_det may be NULL: zero */, workspace,
                            workspace_bytes, nfb_maf_inverse_backward_workspace_bytes(d, features, rows)));
    cudaStream_t st = S(stream);
    if (rows == 0) return resnet_zero_grads(d, g_w, g_b, g_wc, g_bc, st);
    ResnetPass r{d, rows, {nullptr, st}};
    NFB_TRY(glow_err_buf(&r.g.err));
    float *P = nullptr, *pbar = nullptr, *gin = nullptr;
    maf_layout(d, features, rows, static_cast<char*>(workspace), r.ws, &P, &pbar, &gin);
    // one recompute at the layer's output y; its ReLU masks and gate logits serve every pass below
    NFB_TRY(resnet_recompute(r, y, context));
    const int H = d->net.hidden_features, nb = d->net.num_blocks;
    NFB_TRY(r.g.w(fwd_args(r.ws.h[nb], H, 0, r.wf, d->net.b_final, P, rows, 2 * features, H)));
    // lam = g_y + MADE_dgrad_x(A(lam)), D - 1 times: exact, as MADE's Jacobian in y is strictly lower triangular
    for (int it = 0; it + 1 < features; ++it) {
        NFB_TRY(launch_maf_affine_adjoint(x, P, g_y, g_log_det, it ? gin : nullptr, rows, features, pbar, nullptr, st));
        NFB_TRY(resnet_adjoint(r, context, pbar, true, gin, nullptr, {}, {}, {}, {}));
    }
    NFB_TRY(launch_maf_affine_adjoint(x, P, g_y, g_log_det, features > 1 ? gin : nullptr, rows, features, pbar, g_x, st));
    return resnet_adjoint(r, context, pbar, false, nullptr, g_context, g_w, g_b, g_wc, g_bc);
}

namespace {
// Scratch of nfb_ar_rqs_sampling_backward: the conditioner's (resnet_layout), then
//   P    [rows, D, 2K + nd]  MADE(pre(x), context), the spline parameters at the layer's output
//   pbar [rows, D, 2K + nd]  their cotangent
//   gin  [rows, D]           data gradient of the latest fixed-point pass (through pre)
//   gxin [rows, D]           MADE data gradient at pre(x)
//   xin  [rows, D]           pre(x), the MADE's input (periodic features)
int64_t ar_rqs_layout(const nfb_resnet_ctx_desc_t* d, int32_t features, int32_t K, int32_t nd, long long rows,
                      char* base, ResnetWs& ws, float** P, float** pbar, float** gin, float** gxin, float** xin) {
    Carver c{base};
    if (resnet_layout(d, rows, c, ws) < 0 || features < 1 || K < 1 || K > 32 || (nd != K - 1 && nd != K && nd != K + 1))
        return -1;
    const size_t np = (size_t)rows * features * (2 * K + nd);
    float* p = c.take<float>(np); if (P) *P = p;
    p = c.take<float>(np); if (pbar) *pbar = p;
    p = c.take<float>((size_t)rows * features); if (gin) *gin = p;
    p = c.take<float>((size_t)rows * features); if (gxin) *gxin = p;
    p = c.take<float>((size_t)rows * features); if (xin) *xin = p;
    return (int64_t)c.off;
}
}  // namespace

int64_t nfb_ar_rqs_sampling_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* d, int32_t features, int32_t num_bins,
                                                     int32_t num_derivatives, int64_t rows) {
    ResnetWs ws;
    return ar_rqs_layout(d, features, num_bins, num_derivatives, rows, nullptr, ws, nullptr, nullptr, nullptr, nullptr,
                         nullptr);
}

int nfb_ar_rqs_sampling_backward(const nfb_resnet_ctx_desc_t* d, int32_t features, int32_t num_bins,
                                 int32_t num_derivatives, float tail_bound, const float* tails, const int32_t* circular,
                                 const int32_t* pf_slot, const float* pf_weights, const float* pf_scale,
                                 const float* pf_bias, int32_t pf_n_periodic, const float* z, const float* x,
                                 const float* context, const float* g_x, const float* g_log_det, int64_t rows,
                                 void* workspace, int64_t workspace_bytes, float* g_z, float* g_context,
                                 float* const* g_w, float* const* g_b, float* const* g_wc, float* const* g_bc,
                                 float* g_pf_weights, float* g_pf_bias, void* stream) {
    const char* who = "nfb_ar_rqs_sampling_backward";
    const int D = features, K = num_bins, nd = num_derivatives, P = 2 * K + nd;
    NFB_CHECK(d && d->net.m_initial, NFB_ERR_ARG, "%s: the descriptor must be a MADE (mask pointers set)", who);
    NFB_CHECK(K >= 1 && K <= 32 && (nd == K - 1 || nd == K || nd == K + 1), NFB_ERR_ARG,
              "%s: %d derivative parameters for %d bins", who, nd, K);
    NFB_CHECK(D >= 1 && d->net.in_features == D && d->net.out_features == D * P, NFB_ERR_ARG,
              "%s: a MADE of %d -> %d features does not parameterise %d features of %d spline parameters", who,
              d->net.in_features, d->net.out_features, D, P);
    NFB_CHECK(d->context_features == 0 || d->w_context, NFB_ERR_ARG, "%s: a MADE takes its context through w_context",
              who);
    NFB_CHECK(nd == K - 1 ? (!tails && !circular) : (tails && circular), NFB_ERR_ARG,
              "%s: per-feature tail bounds and circular flags go with num_derivatives = K or K + 1, and only there", who);
    const bool pf = pf_slot != nullptr;
    NFB_CHECK(!pf || (pf_weights && pf_scale && pf_n_periodic >= 0), NFB_ERR_ARG, "%s: incomplete periodic tables", who);
    NFB_TRY(resnet_validate(who, d, rows, x, context, z /* g_x and g_log_det may be NULL: zero */, workspace,
                            workspace_bytes, nfb_ar_rqs_sampling_backward_workspace_bytes(d, D, K, nd, rows)));
    cudaStream_t st = S(stream);
    if (rows == 0) {
        if (g_pf_weights) NFB_CUDA(cudaMemsetAsync(g_pf_weights, 0, (size_t)pf_n_periodic * 2 * 4, st));
        if (g_pf_bias) NFB_CUDA(cudaMemsetAsync(g_pf_bias, 0, (size_t)pf_n_periodic * 4, st));
        return resnet_zero_grads(d, g_w, g_b, g_wc, g_bc, st);
    }
    ResnetPass r{d, rows, {nullptr, st}};
    NFB_TRY(glow_err_buf(&r.g.err));
    float *Pm = nullptr, *pbar = nullptr, *gin = nullptr, *gxin = nullptr, *xin = nullptr;
    ar_rqs_layout(d, D, K, nd, rows, static_cast<char*>(workspace), r.ws, &Pm, &pbar, &gin, &gxin, &xin);
    // one recompute at pre(x), x the layer's output; its ReLU masks and gate logits serve every pass below
    const float* in = x;
    if (pf) {
        NFB_TRY(launch_periodic_features(x, xin, rows, D, pf_slot, pf_weights, pf_scale, pf_bias, st));
        in = xin;
    }
    NFB_TRY(resnet_recompute(r, in, context));
    const int H = d->net.hidden_features, nb = d->net.num_blocks;
    NFB_TRY(r.g.w(fwd_args(r.ws.h[nb], H, 0, r.wf, d->net.b_final, Pm, rows, D * P, H)));
    auto spline = [&](const float* lam_in, float* gz) {   // pbar (and g_z) for lam = g_x + lam_in
        return launch_spline_inverse_adjoint(z, Pm, 0, g_x, lam_in, g_log_det, rows, D, K, nd, tails, circular,
                                             tail_bound, 1.f, pbar, gz, st);
    };
    // lam = g_x + pre'(x) MADE_dgrad(pbar(lam)), D - 1 times: exact, as MADE's Jacobian in x is strictly lower
    // triangular (in the degree order)
    for (int it = 0; it + 1 < D; ++it) {
        NFB_TRY(spline(it ? gin : nullptr, nullptr));
        NFB_TRY(resnet_adjoint(r, context, pbar, true, pf ? gxin : gin, nullptr, {}, {}, {}, {}));
        if (pf)
            NFB_TRY(launch_periodic_features_bwd(x, gxin, rows, D, pf_slot, pf_weights, pf_scale, pf_n_periodic, gin,
                                                 nullptr, nullptr, st));
    }
    NFB_TRY(spline(D > 1 ? gin : nullptr, g_z));
    const bool pf_grads = pf && (g_pf_weights || g_pf_bias);
    NFB_TRY(resnet_adjoint(r, context, pbar, false, pf_grads ? gxin : nullptr, g_context, g_w, g_b, g_wc, g_bc));
    if (pf_grads)
        NFB_TRY(launch_periodic_features_bwd(x, gxin, rows, D, pf_slot, pf_weights, pf_scale, pf_n_periodic, nullptr,
                                             g_pf_weights, g_pf_bias, st));
    return NFB_OK;
}

namespace {
// Scratch of nfb_mlp_backward: A[l] [rows, sizes[l + 1]], l < num_layers - 1 (hidden activations), two cotangent
// buffers [rows, max width].
int64_t mlp_layout(const nfb_mlp_desc_t* d, long long rows, char* base, float** A, float** Y) {
    if (!d || d->num_layers < 1 || d->num_layers > 6 || rows < 0 || d->leaky < 0.f) return -1;
    Carver c{base};
    int wmax = 0;
    for (int l = 0; l <= d->num_layers; ++l) {
        if (d->sizes[l] < 1) return -1;
        wmax = std::max(wmax, (int)d->sizes[l]);
    }
    for (int l = 0; l + 1 < d->num_layers; ++l) {
        float* p = c.take<float>((size_t)rows * d->sizes[l + 1]);
        if (A) A[l] = p;
    }
    for (int i = 0; i < 2; ++i) { float* p = c.take<float>((size_t)rows * wmax); if (Y) Y[i] = p; }
    return (int64_t)c.off;
}

// nets.MLP on the tensor core: L Linear layers, LeakyReLU(slope) after every one but the last
struct MlpNet { int L; const int* sizes; const float* const* w; const float* const* b; float slope; };

// A[l] = act(A[l - 1] W_l^T + b_l), l < L - 1 (A[-1] = x, row stride ldx; ReLU fused into the GEMM for slope 0); with
// `out`, the last Linear into out [rows, sizes[L]]
int mlp_forward(const GemmRun& g, const MlpNet& m, const float* x, long long ldx, long long rows, float* const* A,
                float* out) {
    const int* w = m.sizes;
    for (int l = 0; l < m.L; ++l) {
        const bool last = l + 1 == m.L;
        if (last && !out) break;
        GemmTcArgs a = fwd_args(l ? A[l - 1] : x, l ? w[l] : ldx, 0, m.w[l], m.b[l], last ? out : A[l], rows, w[l + 1], w[l]);
        a.relu_out = !last && m.slope == 0.f;
        NFB_TRY(g.w(a));
        if (!last && m.slope != 0.f) {
            NFB_TRY(launch_leaky_gate(A[l], A[l], m.slope, rows * w[l + 1], A[l], g.st));
            g.count(1);
        }
    }
    return NFB_OK;
}

// back-propagates gY [rows, sizes[L]] through the net whose hidden activations mlp_forward left in A (Y: two cotangent
// buffers [rows, widest hidden layer]): weight / bias gradients (each optional; accumulate: added to), and the input
// gradient g_x (optional, row stride ldgx), written or, with gx_add, added after a product with the row vector gx_mul
// (optional)
int mlp_adjoint(const GemmRun& g, const MlpNet& m, const float* x, long long ldx, const float* gY, long long rows,
                float* const* A, float* const* Y, float* g_x, long long ldgx, int gx_add, const float* gx_mul,
                float* const* g_w, float* const* g_b, int accumulate) {
    const int* w = m.sizes;
    for (int l = m.L - 1; l >= 0; --l) {
        const float* X = l ? A[l - 1] : x;
        NFB_TRY(wgrad(g, gY, w[l + 1], X, l ? w[l] : ldx, w[l], 0, nullptr, rows, g_w ? g_w[l] : nullptr,
                      g_b ? g_b[l] : nullptr, accumulate));
        if (l == 0) {
            if (g_x) {
                GemmTcArgs a = dgrad_args(gY, m.w[0], g_x, rows, w[0], w[1]);
                a.ldc = ldgx; a.accumulate = gx_add; a.mulm = gx_mul;
                NFB_TRY(g.w(a));
            }
            break;
        }
        float* gA = Y[l & 1];
        GemmTcArgs a = dgrad_args(gY, m.w[l], gA, rows, w[l], w[l + 1]);
        if (m.slope == 0.f) { a.mask = A[l - 1]; a.ldmask = w[l]; }
        NFB_TRY(g.w(a));
        if (m.slope != 0.f) {
            NFB_TRY(launch_leaky_gate(gA, A[l - 1], m.slope, rows * w[l], gA, g.st));
            g.count(1);
        }
        gY = gA;
    }
    return NFB_OK;
}
}  // namespace

int64_t nfb_mlp_backward_workspace_bytes(const nfb_mlp_desc_t* d, int64_t rows) {
    return mlp_layout(d, rows, nullptr, nullptr, nullptr);
}

int nfb_mlp_backward(const nfb_mlp_desc_t* d, const float* x, const float* g_out, int64_t rows, void* workspace,
                     int64_t workspace_bytes, float* g_x, float* const* g_w, float* const* g_b, void* stream) {
    const int64_t need = mlp_layout(d, rows, nullptr, nullptr, nullptr);
    NFB_CHECK(need >= 0, NFB_ERR_ARG, "nfb_mlp_backward: bad descriptor or shape");
    NFB_CHECK(workspace_bytes >= need && (need == 0 || workspace), NFB_ERR_ARG,
              "nfb_mlp_backward: workspace of %lld bytes, needs %lld", (long long)workspace_bytes, (long long)need);
    const int L = d->num_layers;
    const int* w = d->sizes;
    for (int l = 0; l < L; ++l) NFB_CHECK(d->w[l] && d->b[l], NFB_ERR_ARG, "nfb_mlp_backward: null weight or bias");
    NFB_CHECK(rows == 0 || (x && g_out), NFB_ERR_ARG, "nfb_mlp_backward: null input");
    cudaStream_t st = S(stream);
    if (rows == 0) {
        for (int l = 0; l < L; ++l) {
            if (g_w && g_w[l]) NFB_CUDA(cudaMemsetAsync(g_w[l], 0, (size_t)w[l + 1] * w[l] * 4, st));
            if (g_b && g_b[l]) NFB_CUDA(cudaMemsetAsync(g_b[l], 0, (size_t)w[l + 1] * 4, st));
        }
        return NFB_OK;
    }
    float* A[6] = {}; float* Y[2] = {};
    mlp_layout(d, rows, static_cast<char*>(workspace), A, Y);
    int* err_dev = nullptr;
    NFB_TRY(glow_err_buf(&err_dev));
    const GemmRun g{err_dev, st};
    const MlpNet m{L, w, d->w, d->b, d->leaky};
    NFB_TRY(mlp_forward(g, m, x, w[0], rows, A, nullptr));
    return mlp_adjoint(g, m, x, w[0], g_out, rows, A, Y, g_x, w[0], 0, nullptr, g_w, g_b, 0);
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
    // (one feature: no off-diagonal entries, so the two empty tensors may have no storage)
    NFB_CHECK(d->permutation && (f->D == 1 || (d->lower_entries && d->upper_entries)) && d->unconstrained_upper_diag &&
              d->bias, NFB_ERR_ARG, "LULinearPermute: null pointer");
    NFB_CHECK(f->D <= 64, NFB_ERR_UNSUPPORTED, "LULinearPermute: features %d > 64", f->D);
    L->lu = *d;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_masked_affine(nfb_flow_t* f, const nfb_masked_affine_desc_t* d) {
    NFB_NEW_LAYER(L_MASKED_AFFINE);
    NFB_CHECK(d->b, NFB_ERR_ARG, "MaskedAffineFlow: null mask");
    L->op.type = kOpMasked; L->op.p0 = d->b; L->op.slope = 0.f;
    NFB_TRY(copy_mlp(d->s, L->op.s, &L->op.slope));
    L->op.slope_t = 0.f;
    NFB_TRY(copy_mlp(d->t, L->op.t, &L->op.slope_t));
    if (d->s.num_layers) NFB_CHECK(d->s.sizes[0] == f->D && d->s.sizes[d->s.num_layers] == f->D, NFB_ERR_ARG, "s-net must map D -> D");
    if (d->t.num_layers) NFB_CHECK(d->t.sizes[0] == f->D && d->t.sizes[d->t.num_layers] == f->D, NFB_ERR_ARG, "t-net must map D -> D");
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_affine_coupling(nfb_flow_t* f, const nfb_affine_coupling_desc_t* d) {
    NFB_NEW_LAYER(L_AFFINE_COUPLING);
    NFB_CHECK(d->scale_map >= 0 && d->scale_map <= 2, NFB_ERR_UNSUPPORTED, "This scale map is not implemented.");
    NFB_CHECK(d->split_mode == 0 || d->split_mode == 1, NFB_ERR_UNSUPPORTED, "split mode is not implemented.");
    L->op.type = kOpCoupling;
    L->op.flags = (d->scale ? 1 : 0) | (d->scale_map << 1) | (d->split_mode << 3);
    NFB_TRY(copy_mlp(d->param_map, L->op.s, &L->op.slope));
    const CouplingSplit c(f->D, d->split_mode != 0);
    const int n1 = c.n1, n2 = c.n2;
    NFB_CHECK(d->param_map.num_layers >= 1 && d->param_map.sizes[0] == n1 &&
              d->param_map.sizes[d->param_map.num_layers] == (d->scale ? 2 : 1) * n2,
              NFB_ERR_ARG, "param_map must map %d -> %d", n1, (d->scale ? 2 : 1) * n2);
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_affine_const(nfb_flow_t* f, const nfb_affine_const_desc_t* d) {
    NFB_NEW_LAYER(L_AFFINE_CONST);
    NFB_CHECK(d->s && d->t, NFB_ERR_ARG, "AffineConstFlow: null s/t");
    L->op.type = kOpConst; L->op.p0 = d->s; L->op.p1 = d->t;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_permute(nfb_flow_t* f, const nfb_permute_desc_t* d) {
    NFB_NEW_LAYER(L_PERMUTE);
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

int nfb_flow_add_planar(nfb_flow_t* f, const nfb_planar_desc_t* d) {
    NFB_NEW_LAYER(L_PLANAR);
    NFB_CHECK(f->D <= kPlanarMaxD, NFB_ERR_UNSUPPORTED, "Planar: features %d > %d", f->D, kPlanarMaxD);
    NFB_CHECK(d->u && d->w && d->b, NFB_ERR_ARG, "Planar: null parameter");
    NFB_CHECK(d->act == NFB_PLANAR_TANH || d->act == NFB_PLANAR_LEAKY_RELU, NFB_ERR_UNSUPPORTED,
              "Nonlinearity is not implemented.");
    L->pop.type = d->act == NFB_PLANAR_TANH ? kPlanarTanh : kPlanarLeaky;
    L->pop.slope = d->slope;
    L->pop.a = d->u; L->pop.w = d->w; L->pop.b = d->b;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_add_radial(nfb_flow_t* f, const nfb_radial_desc_t* d) {
    NFB_NEW_LAYER(L_RADIAL);
    NFB_CHECK(f->D <= kPlanarMaxD, NFB_ERR_UNSUPPORTED, "Radial: features %d > %d", f->D, kPlanarMaxD);
    NFB_CHECK(d->beta && d->alpha && d->z0, NFB_ERR_ARG, "Radial: null parameter");
    L->pop.type = kRadial;
    L->pop.a = d->z0; L->pop.b = d->beta; L->pop.alpha = d->alpha;
    f->layers.push_back(std::move(L));
    return NFB_OK;
}

int nfb_flow_set_base_diag_gaussian(nfb_flow_t* f, const float* loc, const float* log_scale) {
    NFB_CHECK(f && loc && log_scale, NFB_ERR_ARG, "null argument");
    f->base_loc = loc; f->base_log_scale = log_scale;
    f->base_weight_scores = nullptr; f->base_modes = 0;
    return NFB_OK;
}

int nfb_flow_set_base_gaussian_mixture(nfb_flow_t* f, int32_t n_modes, const float* loc, const float* log_scale,
                                       const float* weight_scores) {
    NFB_CHECK(f && loc && log_scale && weight_scores, NFB_ERR_ARG, "null argument");
    NFB_CHECK(n_modes >= 1, NFB_ERR_ARG, "GaussianMixture: n_modes %d < 1", n_modes);
    f->base_loc = loc; f->base_log_scale = log_scale;
    f->base_weight_scores = weight_scores; f->base_modes = n_modes;
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
            // the narrow kernel holds a row, and every net's activations, in one thread: over its limits the group
            // takes the wide path
            g.wide = f->D > kAffMaxD;
            g.wo = f->D;
            for (const AffineOp& op : ops)
                for (int n = 0; n < 2; ++n) {
                    const AffMlp& m = n ? op.t : op.s;
                    int hidden = 0;
                    for (int l = 0; l <= m.n_layers && m.n_layers; ++l) {
                        g.wide = g.wide || m.sizes[l] > kAffMaxW;
                        g.wy = std::max(g.wy, m.sizes[l]);
                        if (l > 0 && l < m.n_layers) hidden += m.sizes[l];
                    }
                    if (m.n_layers) g.wo = std::max(g.wo, m.sizes[m.n_layers]);
                    (n ? g.ht : g.hs) = std::max(n ? g.ht : g.hs, hidden);
                }
            NFB_TRY(g.ops.upload(ops));
            f->groups.push_back(std::move(g));
            i = j + 1;
        } else if (is_planar_kind(L)) {
            // one launch for the run: every layer's constants are formed on the device, so a parameter update needs no
            // repack.  Workspace plan of the sampling backward: planar 2D + 3 units / sums per layer, radial D + 2
            int j = i;
            while (j + 1 < n && is_planar_kind(*f->layers[j + 1])) ++j;
            Group g; g.kind = G_PLANAR; g.first = i; g.last = j;
            const int D = f->D;
            int u = 0;
            long long e = 0;
            for (int k = i; k <= j; ++k) {
                PlanarOp op = f->layers[k]->pop;
                const int w = op.type == kRadial ? D + 2 : 2 * D + 3;
                op.u_off = u; op.s_off = (int)e;
                if (op.type == kRadial) {   // column sums of g_dz, the beta_hat and the alpha_hat terms
                    g.items.push_back(AffRedItem{-1, u, 0, D + 2, e, nullptr, nullptr});
                } else {                    // sum c z and sum c; sum h g (and sum h, unused); sum e
                    g.items.push_back(AffRedItem{u, u + 2 * D, D, 1, e, nullptr, nullptr});
                    g.items.push_back(AffRedItem{u + D, u + 2 * D + 1, D, 1, e + D + 1, nullptr, nullptr});
                    g.items.push_back(AffRedItem{-1, u + 2 * D + 2, 0, 1, e + 2 * D + 2, nullptr, nullptr});
                }
                g.invertible = g.invertible && op.type == kPlanarLeaky;
                g.pops.push_back(op);
                u += w; e += w;
            }
            g.units = u;
            g.n_elem = e;
            NFB_TRY(g.ops.upload(g.pops));
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
}  // extern "C"

namespace {
const Group* affine_group_of(const nfb_flow* f, int index) {
    for (auto& g : f->groups)
        if (g.kind == G_AFFINE && index >= g.first && index <= g.last) return &g;
    return nullptr;
}
}  // namespace

extern "C" {
int64_t nfb_flow_last_launch_count(const nfb_flow_t* f) { return f ? f->launches : 0; }
int nfb_flow_layer_is_fused(const nfb_flow_t* f, int32_t index) {
    if (!f || index < 0 || index >= (int)f->layers.size()) return 0;
    for (auto& g : f->groups)
        if ((g.kind == G_FUSED || g.kind == G_FUSED_PAIR) && index >= g.first && index <= g.last) return 1;
    return 0;
}
int nfb_flow_sampling_units(const nfb_flow_t* f) { return f ? f->fwd_n : 0; }

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
    if (is_planar_kind(L)) {
        // the group holding the layer has its descriptor in place: launch that one entry
        const Group* gp = nullptr;
        for (auto& g : f->groups)
            if (g.kind == G_PLANAR && index >= g.first && index <= g.last) gp = &g;
        NFB_CHECK(gp, NFB_ERR_STATE, "planar layer outside a planar group");
        NFB_CHECK(direction == NFB_FORWARD || L.pop.type == kPlanarLeaky, NFB_ERR_UNSUPPORTED,
                  "This flow has no algebraic inverse.");
        rc = launch_planar_stack(static_cast<const PlanarOp*>(gp->ops.p) + (index - gp->first), 1, z_in, out, log_det,
                                 rows, f->D, 1, direction, st);
    } else if (is_affine_kind(L) && affine_group_of(f, index)->wide) {
        rc = affine_wide_apply(f, *affine_group_of(f, index), index, index, direction, z_in, out, log_det, rows, st);
    } else if (is_affine_kind(L)) {
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
    if (f->groups.size() == 1 && f->groups[0].kind == G_PLANAR && z_in != z_out) {   // one launch, log-det written
        Group& g = f->groups[0];
        NFB_CHECK(direction == NFB_FORWARD || g.invertible, NFB_ERR_UNSUPPORTED, "This flow has no algebraic inverse.");
        NFB_TRY(launch_planar_stack(g.ops.p, g.last - g.first + 1, z_in, z_out, ld, rows, f->D, 0, direction, st));
        f->launches++;
        return NFB_OK;
    }
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

namespace {
// log_q += log q0(z): the flow's base, a DiagGaussian or a Gaussian mixture (one launch either way)
int launch_base_log_prob(nfb_flow* f, const float* z, float* log_q, int64_t rows, cudaStream_t st) {
    if (f->base_weight_scores)
        return launch_mixture_log_prob(z, f->base_loc, f->base_log_scale, f->base_weight_scores, log_q, rows,
                                       f->base_modes, f->D, 1, st);
    return launch_diag_gauss(z, f->base_loc, f->base_log_scale, log_q, rows, f->D, 1, st);
}
}  // namespace

int nfb_flow_log_prob(nfb_flow_t* f, const float* x, float* log_q, int64_t rows, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(f->base_loc && f->base_log_scale, NFB_ERR_STATE, "no base distribution set");
    NFB_CHECK(x && log_q, NFB_ERR_ARG, "null pointer");
    if (rows == 0) return NFB_OK;
    NFB_TRY(ensure_ws(f, rows));
    NFB_TRY(f->zfinal.reserve((size_t)rows * f->D * 4));
    float* z = f->zfinal.as<float>();
    NFB_TRY(nfb_flow_transform(f, NFB_INVERSE, x, z, log_q, rows, stream));
    NFB_TRY(launch_base_log_prob(f, z, log_q, rows, S(stream)));
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
    // the spline adjoint kernels take 8 bins only: other counts have no native backward (the caller falls back)
    case L_AR_RQS: return L.K == 8 ? 4 + 4 * L.net.nb : -1;
    case L_COUPLED_RQS: return L.K == 8 ? 4 + 4 * L.net.nb + 3 : -1;
    case L_LU: return 4;
    // affine family, in each layer's parameter registration order: MaskedAffineFlow s then t (weight, bias per Linear),
    // AffineConstFlow s, t, AffineCouplingBlock param_map, Permute none
    case L_MASKED_AFFINE: return 2 * (L.op.s.n_layers + L.op.t.n_layers);
    case L_AFFINE_CONST: return 2;
    case L_AFFINE_COUPLING: return 2 * L.op.s.n_layers;
    case L_PERMUTE: return 0;
    // planar: u, w, b; radial: beta, alpha, z_0 (registration order)
    case L_PLANAR: return 3;
    case L_RADIAL: return 3;
    default: return -1;
    }
}
long long grad_slot_numel(const Layer& L, int s) {
    const NetDesc& n = L.net;
    if (L.kind == L_AFFINE_CONST) return L.D;
    if (L.kind == L_PLANAR) return s == 2 ? 1 : L.D;
    if (L.kind == L_RADIAL) return s == 2 ? L.D : 1;
    if (L.kind == L_MASKED_AFFINE || L.kind == L_AFFINE_COUPLING) {
        const bool t_net = L.kind == L_MASKED_AFFINE && s >= 2 * L.op.s.n_layers;
        const AffMlp& m = t_net ? L.op.t : L.op.s;
        const int k = t_net ? s - 2 * L.op.s.n_layers : s, l = k / 2;
        return (k & 1) ? m.sizes[l + 1] : (long long)m.sizes[l + 1] * m.sizes[l];
    }
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

// The conditioner of a spline block (no context), recomputed on the forward's effective weights (L.pack), each weight
// operand split to bf16 records before its GEMM.  x: [rows x D]; the conditioner reads all its columns (autoregressive)
// or the identity columns x[:, id], gathered into f->tr_in (coupling).  Sets up d / r for the adjoint and leaves the
// conditioner's output in f->tr_P.
int conditioner_recompute(nfb_flow* f, Layer& L, const float* x, long long rows, nfb_resnet_ctx_desc_t& d,
                          ResnetPass& r, cudaStream_t st) {
    const NetDesc& n = L.net;
    d = nfb_resnet_ctx_desc_t{};
    d.net = {n.in, n.H, n.out, n.nb, n.w0, n.b0, n.m0, n.wb.data(), n.bb.data(), n.mb.data(), n.wf, n.bf, n.mf};
    r = ResnetPass{&d, rows, {f->err.as<int>(), st, &f->tr_wpack, &f->launches}};
    r.w0 = L.pack.w0; r.wf = L.pack.wf; r.wb = L.pack.wb;
    Carver c;
    resnet_layout(&d, rows, c, r.ws, false);
    NFB_TRY(f->tr_net.reserve(c.off));
    c = Carver{f->tr_net.as<char>()};
    resnet_layout(&d, rows, c, r.ws, false);
    NFB_TRY(f->tr_P.reserve((size_t)rows * n.out * 4));
    NFB_TRY(f->tr_gP.reserve((size_t)rows * n.out * 4));
    const float* in = x;
    if (L.kind == L_COUPLED_RQS) {
        NFB_TRY(f->tr_in.reserve((size_t)rows * L.n_id * 4));
        NFB_TRY(f->tr_gin.reserve((size_t)rows * L.n_id * 4));
        NFB_TRY(launch_gather_cols_ld(x, L.D, f->tr_in.as<float>(), L.n_id, L.id_idx.as<int>(), rows, st));
        in = f->tr_in.as<float>();
    }
    NFB_TRY(resnet_recompute(r, in, nullptr));
    return r.g.w(fwd_args(r.ws.h[n.nb], n.H, 0, r.wf, n.bf, f->tr_P.as<float>(), rows, n.out, n.H));
}

// The coupling block's conditioner adjoint from the gradient on its output (f->tr_gP): weight gradients into `slots`
// (each Linear's weight and bias interleaved: w0, b0, w_blocks..., wf, bf), and the data gradient of the identity
// columns (W0 read unpacked) scatter-added into g[:, id].
int coupled_conditioner_adjoint(nfb_flow* f, Layer& L, const ResnetPass& r, long long rows, float* const* slots,
                                float* g, cudaStream_t st) {
    const Slots g_w(slots, 2), g_b(slots + 1, 2);
    NFB_TRY(resnet_adjoint(r, nullptr, f->tr_gP.as<float>(), false, nullptr, nullptr, g_w, g_b, {}, {}));
    NFB_TRY(r.g(dgrad_args(r.ws.ga, r.w0, f->tr_gin.as<float>(), rows, L.n_id, L.net.H)));
    NFB_TRY(launch_scatter_cols(f->tr_gin.as<float>(), g, L.id_idx.as<int>(), rows, L.n_id, L.D, 1, st));
    f->launches++;
    return NFB_OK;
}

// backward of one spline layer: xp = the layer's input [rows x D], gy = gradient w.r.t. its output; writes the
// gradient w.r.t. its input into gxp ([rows x D]) and the parameter gradients into `slots`.
int rqs_layer_backward(nfb_flow* f, Layer& L, const float* xp, const float* gy, const float* glq, long long rows,
                       float* gxp, float* const* slots, cudaStream_t st) {
    const NetDesc& n = L.net;
    const int D = L.D, T = L.n_tr, P = 3 * L.K - 1;
    const bool coupled = L.kind == L_COUPLED_RQS;
    NFB_CHECK(L.K == 8, NFB_ERR_UNSUPPORTED, "native backward: num_bins %d != 8", L.K);
    nfb_resnet_ctx_desc_t d;
    ResnetPass r;
    NFB_TRY(conditioner_recompute(f, L, xp, rows, d, r, st));
    float* Pm = f->tr_P.as<float>();
    float* gP = f->tr_gP.as<float>();
    // spline element backward -> gP, gxp (transformed columns)
    NFB_TRY(launch_spline_bwd_rows(xp, D, Pm, gy, glq, coupled ? L.tr_idx.as<int>() : nullptr, rows, T, L.K, L.tail,
                                   L.wh_scale, gP, gxp, st));
    f->launches++;
    const int nlin = 2 + 2 * n.nb;
    if (coupled) {
        // the table gradient [n_id x P] at the front; at least the LU scratch behind it (lu_layer_backward's layout)
        NFB_TRY(f->tr_small.reserve((size_t)(64 * 64 + std::max(64, L.n_id) * P + 64) * 4));
        float* gtab = f->tr_small.as<float>();
        NFB_CUDA(cudaMemsetAsync(gtab, 0, (size_t)L.n_id * P * 4, st));
        NFB_TRY(launch_spline_bwd_shared(xp, D, L.uncond.as<float>(), gy, glq, L.id_idx.as<int>(), rows, L.n_id, L.K, L.tail,
                                         gtab, gxp, st));
        NFB_TRY(launch_split_table(gtab, L.n_id, slots[2 * nlin], slots[2 * nlin + 1], slots[2 * nlin + 2], st));
        f->launches += 3;
    }
    if (!coupled) {  // gxp += the conditioner's data gradient (in place)
        const Slots g_w(slots, 2), g_b(slots + 1, 2);
        return resnet_adjoint(r, nullptr, gP, false, gxp, nullptr, g_w, g_b, {}, {}, true);
    }
    return coupled_conditioner_adjoint(f, L, r, rows, slots, gxp, st);
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
    const GemmRun g{f->err.as<int>(), st, nullptr, &f->launches};
    NFB_TRY(launch_gather_cols(zin, zp, L.lu_perm.as<int>(), rows, D, 1, st));
    f->launches++;
    if (slots[0] || slots[1] || slots[2]) {
        GemmTcArgs a{};
        a.A = gxp; a.lda = D; a.a_mn = 1; a.B = zp; a.ldb = D; a.b_mn = 1; a.C = dW; a.ldc = D; a.M = D; a.N = D; a.K = rows;
        NFB_TRY(g(a));
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
    NFB_TRY(g(a));
    NFB_TRY(launch_scatter_cols(gzp, gz, L.lu_perm.as<int>(), rows, D, D, 0, st));
    f->launches++;
    return NFB_OK;
}

// the affine family's backward (defined with the sampling-direction entry points below)
int plan_affine_bwd(nfb_flow* f, Group& g);
long long affine_bwd_chunk_rows(const nfb_flow* f, const Group& g, long long rows);
size_t affine_bwd_ws_bytes(const nfb_flow* f, const Group& g, long long R);
int affine_group_backward(nfb_flow* f, Group& g, int direction, const float* in, const float* g_out, const float* g_ld,
                          int64_t rows, float* ws, long long R, float* g_in, float* const* grad_slots, cudaStream_t st);

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
    return n + (f->base_loc ? (f->base_weight_scores ? 3 : 2) : 0);
}

int64_t nfb_flow_grad_slot_numel(const nfb_flow_t* f, int32_t slot) {
    if (!f || slot < 0) return -1;
    for (auto& L : f->layers) {
        const int k = grad_slots_of(*L);
        if (k < 0) return -1;
        if (slot < k) return grad_slot_numel(*L, slot);
        slot -= k;
    }
    if (f->base_weight_scores) return slot < 2 ? (int64_t)f->base_modes * f->D : slot == 2 ? f->base_modes : -1;
    return (f->base_loc && slot < 2) ? f->D : -1;
}

int nfb_flow_log_prob_backward(nfb_flow_t* f, const float* x, const float* g_logq, int64_t rows, float* log_q_out,
                               float* gx_out, float* const* grad_slots, void* stream) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(f->base_loc && f->base_log_scale, NFB_ERR_STATE, "no base distribution set");
    NFB_CHECK((rows == 0 || (x && g_logq)) && grad_slots, NFB_ERR_ARG, "null pointer");
    const int n_slots = nfb_flow_num_grad_slots(f);
    NFB_CHECK(n_slots >= 0, NFB_ERR_UNSUPPORTED,
              "native backward covers spline blocks + LULinearPermute + the affine family + DiagGaussian / GaussianMixture");
    for (auto& grp : f->groups)   // (the planar family has slots for its sampling-direction backward only)
        NFB_CHECK(grp.kind != G_PLANAR, NFB_ERR_UNSUPPORTED, "native backward: planar-family group");
    cudaStream_t st = S(stream);
    if (rows == 0) {   // zero gradients
        for (int i = 0; i < n_slots; ++i)
            if (grad_slots[i]) NFB_CUDA(cudaMemsetAsync(grad_slots[i], 0, (size_t)nfb_flow_grad_slot_numel(f, i) * 4, st));
        return NFB_OK;
    }
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
    NFB_TRY(launch_base_log_prob(f, zfin, logq, rows, st));
    // ---- backward ----
    // slot offsets per layer
    std::vector<int> off(f->layers.size() + 1, 0);
    for (size_t i = 0; i < f->layers.size(); ++i) off[i + 1] = off[i] + grad_slots_of(*f->layers[i]);
    float* const* base_slots = grad_slots + off[f->layers.size()];
    NFB_CUDA(cudaMemsetAsync(glq_sum, 0, 4, st));
    NFB_TRY(launch_colsum(g_logq, 1, rows, 1, glq_sum, st));
    float* g = f->tr_g0.as<float>();
    float* g2 = f->tr_g1.as<float>();
    if (f->base_weight_scores) {
        const long long wsb = mixture_bwd_ws_bytes(rows, f->base_modes, D);
        NFB_TRY(f->tr_mix.reserve((size_t)wsb));
        NFB_TRY(launch_mixture_bwd(zfin, f->base_loc, f->base_log_scale, f->base_weight_scores, g_logq, rows,
                                   f->base_modes, D, f->tr_mix.p, wsb, g, base_slots[0], base_slots[1], base_slots[2],
                                   st));
    } else {
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
        if (grp.kind == G_AFFINE) {   // recompute + adjoint walk + fixed-order reduction, chunked (internal workspace)
            NFB_TRY(plan_affine_bwd(f, grp));
            const long long R = affine_bwd_chunk_rows(f, grp, rows);
            NFB_TRY(f->tr_aff.reserve(affine_bwd_ws_bytes(f, grp, R)));
            NFB_TRY(affine_group_backward(f, grp, NFB_INVERSE, zin, g, g_logq, rows, f->tr_aff.as<float>(), R, g2,
                                          grad_slots + off[grp.first], st));
            std::swap(g, g2);
            continue;
        }
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

// ==========================================================================================
// sampling-direction backward of an all-affine stack (affine_stack_kernel with direction = 1)
// ==========================================================================================
namespace {

constexpr long long kAffBwdWsCap = 256ll << 20;   // workspace bound: rows are processed in chunks below it

// ---- wide path: an affine group over affine_stack_kernel's limits, layer by layer ----------------------------------------
// Per layer: the nets on gemm_tc (mlp_forward / mlp_adjoint, weights split once per GEMM into f->tr_wpack), the coupling
// arithmetic in nfb_affine_wide.cu.  Rows go in chunks whose scratch stays under kAffBwdWsCap.
struct WideWs {
    std::vector<float*> zs;   // backward: the input of op k (application order), k >= 1; forward: two ping-pong rows
    float* g[2];              // backward: the running input cotangent and a spare (Permute)
    float *zm, *S, *T, *As, *At;
    float* Y[2];              // backward: mlp_adjoint's cotangent buffers
};

size_t wide_layout(const Group& g, int D, long long R, bool bwd, char* base, WideWs* ws) {
    Carver c{base};
    WideWs w{};
    const int nz = bwd ? g.last - g.first : 2;
    for (int k = 0; k < nz; ++k) w.zs.push_back(c.take<float>((size_t)R * D));
    if (bwd) for (auto& p : w.g) p = c.take<float>((size_t)R * D);
    w.zm = c.take<float>((size_t)R * D);
    w.S = c.take<float>((size_t)R * g.wo);
    w.T = c.take<float>((size_t)R * g.wo);
    w.As = c.take<float>((size_t)R * g.hs);
    w.At = c.take<float>((size_t)R * g.ht);
    if (bwd) for (auto& p : w.Y) p = c.take<float>((size_t)R * g.wy);
    if (ws) *ws = std::move(w);
    return c.off;
}

long long wide_chunk_rows(const Group& g, int D, long long rows, bool bwd) {
    const size_t fixed = wide_layout(g, D, 0, bwd, nullptr, nullptr) + 256 * 32;   // alignment slack of the pieces
    const size_t per_row = (wide_layout(g, D, 1024, bwd, nullptr, nullptr) + 1023) / 1024;
    long long R = std::max(1ll, (long long)((kAffBwdWsCap - (long long)fixed) / (long long)per_row));
    if (R > kAffSegRows) R -= R % kAffSegRows;
    return std::max(1ll, std::min(R, rows));
}

MlpNet mlp_net(const AffMlp& m, float slope) { return MlpNet{m.n_layers, m.sizes, m.w, m.b, slope}; }

// the hidden activation buffers of net m inside the region `base` of R rows
void hidden_ptrs(const AffMlp& m, float* base, long long R, float** A) {
    long long off = 0;
    for (int l = 0; l + 1 < m.n_layers; ++l) { A[l] = base + off * R; off += m.sizes[l + 1]; }
}

// one layer in direction dir: zi -> zo (m rows), log-det added into ld (optional); leaves the nets' activations and
// outputs in ws (R-row buffers) for the adjoint.  zo = null: the nets only (the backward's recompute of a layer)
int wide_layer_fwd(nfb_flow* f, const GemmRun& gr, const Layer& L, int dir, const float* zi, float* zo, float* ld,
                   long long m, long long R, const WideWs& ws, cudaStream_t st) {
    const int D = f->D;
    const AffineOp& op = L.op;
    float* A[kAffMaxLayers];
    if (!zo && (L.kind == L_PERMUTE || L.kind == L_AFFINE_CONST)) return NFB_OK;
    switch (L.kind) {
    case L_PERMUTE:
        NFB_TRY(launch_gather_cols(zi, zo, dir ? op.fwd_idx : op.inv_idx, m, D, 1, st));
        break;
    case L_AFFINE_CONST:
        NFB_TRY(launch_affine_wide_elem(op, D, dir, zi, nullptr, nullptr, zo, ld, m, st));
        break;
    case L_MASKED_AFFINE:
        NFB_TRY(launch_affine_wide_mask(zi, op.p0, ws.zm, m, D, st));
        f->launches++;
        if (op.s.n_layers) {
            hidden_ptrs(op.s, ws.As, R, A);
            NFB_TRY(mlp_forward(gr, mlp_net(op.s, op.slope), ws.zm, D, m, A, ws.S));
        }
        if (op.t.n_layers) {
            hidden_ptrs(op.t, ws.At, R, A);
            NFB_TRY(mlp_forward(gr, mlp_net(op.t, op.slope_t), ws.zm, D, m, A, ws.T));
        }
        if (!zo) return NFB_OK;
        NFB_TRY(launch_affine_wide_elem(op, D, dir, zi, op.s.n_layers ? ws.S : nullptr, op.t.n_layers ? ws.T : nullptr,
                                        zo, ld, m, st));
        break;
    case L_AFFINE_COUPLING: {
        const CouplingSplit c(D, (op.flags >> 3) & 1);
        hidden_ptrs(op.s, ws.As, R, A);
        NFB_TRY(mlp_forward(gr, mlp_net(op.s, op.slope), zi + c.o1, D, m, A, ws.S));
        if (!zo) return NFB_OK;
        NFB_TRY(launch_affine_wide_elem(op, D, dir, zi, ws.S, nullptr, zo, ld, m, st));
        break;
    }
    default:
        nfb_set_error("wide affine path: layer kind %d", (int)L.kind);
        return NFB_ERR_STATE;
    }
    f->launches++;
    return NFB_OK;
}

// layers first..last of wide group g in direction dir (density: last to first), zin -> zout (distinct), log-det added into
// logdet (optional)
int affine_wide_apply(nfb_flow* f, const Group& g, int first, int last, int dir, const float* zin, float* zout,
                      float* logdet, long long rows, cudaStream_t st) {
    if (rows == 0) return NFB_OK;
    const int D = f->D, n = last - first + 1;
    const long long R = wide_chunk_rows(g, D, rows, false);
    NFB_TRY(f->aw_fwd.reserve(wide_layout(g, D, R, false, nullptr, nullptr)));
    WideWs ws;
    wide_layout(g, D, R, false, f->aw_fwd.as<char>(), &ws);
    const GemmRun gr{f->err.as<int>(), st, &f->tr_wpack, &f->launches};
    for (long long r0 = 0; r0 < rows; r0 += R) {
        const long long m = std::min(R, rows - r0);
        const float* cur = zin + r0 * D;
        for (int k = 0; k < n; ++k) {
            float* out = k == n - 1 ? zout + r0 * D : ws.zs[k & 1];
            NFB_TRY(wide_layer_fwd(f, gr, *f->layers[dir ? first + k : last - k], dir, cur, out,
                                   logdet ? logdet + r0 : nullptr, m, R, ws, st));
            cur = out;
        }
    }
    return NFB_OK;
}

// backward of wide group g in direction dir (the arguments of affine_group_backward).  Per chunk: recompute every op's
// input, then take the ops in reverse: recompute the layer's nets, the adjoint element kernel, the nets' dgrad / wgrad
// (bias gradients by launch_colsum), their input gradient added into g (masked by b, or into the identity half).
int affine_wide_backward(nfb_flow* f, Group& g, int dir, const float* in, const float* g_out, const float* g_ld,
                         int64_t rows, float* wsp, long long R, float* g_in, float* const* grad_slots, cudaStream_t st) {
    const int D = f->D, n_ops = g.last - g.first + 1;
    std::vector<int> off(n_ops + 1, 0);
    for (int k = 0; k < n_ops; ++k) off[k + 1] = off[k] + grad_slots_of(*f->layers[g.first + k]);
    if (rows == 0) {   // zero parameter gradients
        for (int k = 0; k < n_ops; ++k)
            for (int s = off[k]; s < off[k + 1]; ++s)
                if (grad_slots && grad_slots[s]) {
                    NFB_CUDA(cudaMemsetAsync(grad_slots[s], 0, (size_t)grad_slot_numel(*f->layers[g.first + k], s - off[k]) * 4, st));
                    f->launches++;
                }
        return NFB_OK;
    }
    WideWs ws;
    wide_layout(g, D, R, true, reinterpret_cast<char*>(wsp), &ws);
    const GemmRun gr{f->err.as<int>(), st, &f->tr_wpack, &f->launches};
    // application order: sampling first..last, density last..first
    auto layer_at = [&](int k) -> int { return dir ? g.first + k : g.last - k; };
    for (long long r0 = 0; r0 < rows; r0 += R) {
        const long long m = std::min(R, (long long)rows - r0);
        const int acc = r0 > 0;
        std::vector<const float*> zs(n_ops);
        zs[0] = in + r0 * D;
        for (int k = 0; k + 1 < n_ops; ++k) {
            NFB_TRY(wide_layer_fwd(f, gr, *f->layers[layer_at(k)], dir, zs[k], ws.zs[k], nullptr, m, R, ws, st));
            zs[k + 1] = ws.zs[k];
        }
        float* G = ws.g[0];
        float* G2 = ws.g[1];
        if (g_out) NFB_CUDA(cudaMemcpyAsync(G, g_out + r0 * D, (size_t)m * D * 4, cudaMemcpyDeviceToDevice, st));
        else NFB_CUDA(cudaMemsetAsync(G, 0, (size_t)m * D * 4, st));
        f->launches++;
        const float* gl = g_ld ? g_ld + r0 : nullptr;
        for (int k = n_ops - 1; k >= 0; --k) {
            const int li = layer_at(k);
            const Layer& L = *f->layers[li];
            const AffineOp& op = L.op;
            float* const* slots = grad_slots ? grad_slots + off[li - g.first] : nullptr;
            auto slot = [&](int s) -> float* { return slots ? slots[s] : nullptr; };
            float* A[kAffMaxLayers];
            float *gw[kAffMaxLayers], *gb[kAffMaxLayers];
            auto net_slots = [&](int s0, int n_lin) {
                for (int l = 0; l < n_lin; ++l) { gw[l] = slot(s0 + 2 * l); gb[l] = slot(s0 + 2 * l + 1); }
            };
            if (L.kind == L_PERMUTE) {   // sampling x[j] = z[fwd[j]]: g_z[i] = g_x[inv[i]]; density the other way
                NFB_TRY(launch_gather_cols(G, G2, dir ? op.inv_idx : op.fwd_idx, m, D, 1, st));
                f->launches++;
                std::swap(G, G2);
                continue;
            }
            if (L.kind == L_AFFINE_CONST) {
                NFB_TRY(launch_affine_wide_adjoint(op, D, dir, zs[k], ws.S, ws.T, G, gl, m, st));
                f->launches++;
                for (int j = 0; j < 2; ++j)
                    if (slot(j)) {
                        if (!acc) { NFB_CUDA(cudaMemsetAsync(slot(j), 0, (size_t)D * 4, st)); f->launches++; }
                        NFB_TRY(launch_colsum(j ? ws.T : ws.S, D, m, D, slot(j), st));
                        f->launches++;
                    }
                continue;
            }
            // recompute the layer's nets (and the masked input) on its input
            NFB_TRY(wide_layer_fwd(f, gr, L, dir, zs[k], nullptr, nullptr, m, R, ws, st));
            if (L.kind == L_MASKED_AFFINE) {
                NFB_TRY(launch_affine_wide_adjoint(op, D, dir, zs[k], op.s.n_layers ? ws.S : nullptr,
                                                   op.t.n_layers ? ws.T : nullptr, G, gl, m, st));
                f->launches++;
                if (op.s.n_layers) {
                    hidden_ptrs(op.s, ws.As, R, A);
                    net_slots(0, op.s.n_layers);
                    NFB_TRY(mlp_adjoint(gr, mlp_net(op.s, op.slope), ws.zm, D, ws.S, m, A, ws.Y, G, D, 1, op.p0, gw, gb,
                                        acc));
                }
                if (op.t.n_layers) {
                    hidden_ptrs(op.t, ws.At, R, A);
                    net_slots(2 * op.s.n_layers, op.t.n_layers);
                    NFB_TRY(mlp_adjoint(gr, mlp_net(op.t, op.slope_t), ws.zm, D, ws.T, m, A, ws.Y, G, D, 1, op.p0, gw,
                                        gb, acc));
                }
            } else {
                const CouplingSplit c(D, (op.flags >> 3) & 1);
                NFB_TRY(launch_affine_wide_adjoint(op, D, dir, zs[k], ws.S, nullptr, G, gl, m, st));
                f->launches++;
                hidden_ptrs(op.s, ws.As, R, A);
                net_slots(0, op.s.n_layers);
                NFB_TRY(mlp_adjoint(gr, mlp_net(op.s, op.slope), zs[k] + c.o1, D, ws.S, m, A, ws.Y, G + c.o1, D, 1,
                                    nullptr, gw, gb, acc));
            }
        }
        if (g_in) {
            NFB_CUDA(cudaMemcpyAsync(g_in + r0 * D, G, (size_t)m * D * 4, cudaMemcpyDeviceToDevice, st));
            f->launches++;
        }
    }
    return NFB_OK;
}

// units per row of the workspace, each op's unit table and the weight reduction's items, in grad-slot order
int plan_affine_bwd(nfb_flow* f, Group& g) {
    if (g.bwd_planned || g.wide) return NFB_OK;
    std::vector<AffBwdOp> bops;
    g.items.clear();
    int u = 0;
    long long e = 0;
    auto add_net = [&](const AffMlp& m, AffBwdOp& bo, int n) {
        for (int l = 0; l < m.n_layers; ++l) {
            bo.u_act[n][l] = u; u += m.sizes[l];
            bo.u_del[n][l] = u; u += m.sizes[l + 1];
            g.items.push_back(AffRedItem{bo.u_act[n][l], bo.u_del[n][l], m.sizes[l], m.sizes[l + 1], e, nullptr, nullptr});
            e += (long long)m.sizes[l + 1] * (m.sizes[l] + 1);
        }
    };
    for (int k = g.first; k <= g.last; ++k) {
        const Layer& L = *f->layers[k];
        AffBwdOp bo{};
        bo.u_z = u; u += f->D;
        if (L.kind == L_MASKED_AFFINE) {
            add_net(L.op.s, bo, 0);
            add_net(L.op.t, bo, 1);
        } else if (L.kind == L_AFFINE_COUPLING) {
            add_net(L.op.s, bo, 0);
        } else if (L.kind == L_AFFINE_CONST) {
            for (int n = 0; n < 2; ++n) {
                bo.u_del[n][0] = u; u += f->D;
                g.items.push_back(AffRedItem{-1, bo.u_del[n][0], 0, f->D, e, nullptr, nullptr});
                e += f->D;
            }
        }
        bops.push_back(bo);
    }
    NFB_TRY(g.bops.upload(bops));
    g.units = u;
    g.n_elem = e;
    g.bwd_planned = true;
    return NFB_OK;
}

long long affine_bwd_chunk_rows(const nfb_flow* f, const Group& g, long long rows) {
    if (g.wide) return wide_chunk_rows(g, f->D, rows, true);
    const long long per_row = 4ll * g.units + (4 * g.n_elem + kAffSegRows - 1) / kAffSegRows + 1;
    long long R = std::max(1ll, kAffBwdWsCap / per_row);
    if (R > kAffSegRows) R -= R % kAffSegRows;
    return std::max(1ll, std::min(R, rows));
}

size_t affine_bwd_ws_bytes(const nfb_flow* f, const Group& g, long long R) {
    if (g.wide) return wide_layout(g, f->D, R, true, nullptr, nullptr);
    const size_t data = ((size_t)g.units * R * 4 + 255) & ~(size_t)255;
    return data + (size_t)((R + kAffSegRows - 1) / kAffSegRows) * g.n_elem * 4;
}

// planar group: the same chunking, plus the reduced sums (n_elem floats) after the segment partials
long long planar_bwd_chunk_rows(const Group& g, long long rows) {
    const long long per_row = 4ll * g.units + (4 * g.n_elem + kAffSegRows - 1) / kAffSegRows + 1;
    long long R = std::max(1ll, (kAffBwdWsCap - 4 * g.n_elem) / per_row);
    if (R > kAffSegRows) R -= R % kAffSegRows;
    return std::max(1ll, std::min(R, rows));
}

size_t planar_bwd_partial_off(const Group& g, long long R) { return ((size_t)g.units * R * 4 + 255) & ~(size_t)255; }

size_t planar_bwd_sums_off(const Group& g, long long R) {
    return (planar_bwd_partial_off(g, R) + (size_t)((R + kAffSegRows - 1) / kAffSegRows) * g.n_elem * 4 + 255) &
           ~(size_t)255;
}

size_t planar_bwd_ws_bytes(const Group& g, long long R) { return planar_bwd_sums_off(g, R) + (size_t)g.n_elem * 4; }

Group* planar_only_group(nfb_flow* f) {
    return (f && f->finalized && f->groups.size() == 1 && f->groups[0].kind == G_PLANAR) ? &f->groups[0] : nullptr;
}

// sampling backward of a stack that is one planar / radial group: per chunk of rows the row kernel and the fixed-order
// reduction (2 launches) into the sums, then one launch through the parameter maps into the slots
int planar_sampling_backward(nfb_flow* f, Group& g, const float* z, const float* g_x, const float* g_ld, int64_t rows,
                             void* ws, int64_t ws_bytes, float* g_z, float* const* grad_slots, cudaStream_t st) {
    NFB_CHECK(rows >= 0, NFB_ERR_ARG, "rows < 0");
    NFB_CHECK(rows == 0 || z, NFB_ERR_ARG, "null z");
    const long long R = planar_bwd_chunk_rows(g, rows);
    NFB_CHECK(ws && ws_bytes >= (int64_t)planar_bwd_ws_bytes(g, R), NFB_ERR_ARG,
              "sampling backward: workspace of %lld bytes, %lld needed", (long long)ws_bytes,
              (long long)planar_bwd_ws_bytes(g, R));
    f->launches = 0;
    const int n_items = (int)g.items.size(), n_ops = (int)g.pops.size();
    float* W = static_cast<float*>(ws);
    float* partial = reinterpret_cast<float*>(static_cast<char*>(ws) + planar_bwd_partial_off(g, R));
    float* sums = reinterpret_cast<float*>(static_cast<char*>(ws) + planar_bwd_sums_off(g, R));
    // this call's reduction outputs (into the sums) and gradient slots (three per layer), staged through pinned memory
    const size_t items_bytes = n_items * sizeof(AffRedItem), bytes = items_bytes + n_ops * sizeof(PlanarGradOut);
    if (!f->plb_ev) NFB_CUDA(cudaEventCreateWithFlags(&f->plb_ev, cudaEventDisableTiming));
    else NFB_CUDA(cudaEventSynchronize(f->plb_ev));   // the previous call's staging copy has been read
    if (f->plb_cap < bytes) {
        if (f->plb_host) cudaFreeHost(f->plb_host);
        f->plb_host = nullptr; f->plb_cap = 0;
        NFB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&f->plb_host), bytes));
        f->plb_cap = bytes;
    }
    AffRedItem* items = reinterpret_cast<AffRedItem*>(f->plb_host);
    for (int i = 0; i < n_items; ++i) {
        AffRedItem it = g.items[i];
        if (it.n_in > 0) it.dw = sums + it.e_off;
        it.db = sums + it.e_off + (long long)it.n_out * it.n_in;
        items[i] = it;
    }
    PlanarGradOut* outs = reinterpret_cast<PlanarGradOut*>(f->plb_host + items_bytes);
    for (int k = 0; k < n_ops; ++k)
        for (int s = 0; s < 3; ++s) outs[k].g[s] = grad_slots ? grad_slots[3 * k + s] : nullptr;
    NFB_TRY(f->plb_dev.reserve(bytes));
    NFB_CUDA(cudaMemcpyAsync(f->plb_dev.p, f->plb_host, bytes, cudaMemcpyHostToDevice, st));
    NFB_CUDA(cudaEventRecord(f->plb_ev, st));
    const void* items_dev = f->plb_dev.p;
    const void* outs_dev = static_cast<char*>(f->plb_dev.p) + items_bytes;
    const int D = f->D;
    if (rows == 0) {   // zero sums
        NFB_TRY(launch_affine_bwd_reduce(items_dev, n_items, g.n_elem, W, 0, partial, 0, st));
        f->launches++;
    }
    for (long long r0 = 0; r0 < rows; r0 += R) {
        const long long n = std::min(R, (long long)rows - r0);
        NFB_TRY(launch_planar_bwd_rows(g.ops.p, n_ops, z + r0 * D, g_x ? g_x + r0 * D : nullptr, g_ld ? g_ld + r0 : nullptr,
                                       g_z ? g_z + r0 * D : nullptr, W, n, D, st));
        NFB_TRY(launch_affine_bwd_reduce(items_dev, n_items, g.n_elem, W, n, partial, r0 > 0, st));
        f->launches += 3;
    }
    NFB_TRY(launch_planar_bwd_chain(g.ops.p, outs_dev, n_ops, sums, D, st));
    f->launches++;
    return NFB_OK;
}

int affine_only_group(nfb_flow* f, Group** out, const char* who) {
    NFB_CHECK(f && f->finalized, NFB_ERR_STATE, "flow not finalized");
    NFB_CHECK(f->groups.size() == 1 && f->groups[0].kind == G_AFFINE, NFB_ERR_UNSUPPORTED,
              "%s backward: the stack must be affine-family layers only%s", who,
              who[0] == 's' ? ", planar / radial layers only, or coupled splines / LULinearPermute only" : "");
    *out = &f->groups[0];
    return plan_affine_bwd(f, **out);
}

// backward of one affine group in either direction (affine_bwd_rows_kernel / affine_density_bwd_rows_kernel): `in` is
// the group's input in that direction, g_out / g_ld the cotangents of its output and log-det; writes g_in and the
// group's slots (in grad-slot order, NULL entries skipped).  Per chunk of R rows: the row kernel, then the fixed-order
// reduction.  ws holds affine_bwd_ws_bytes(g, R) bytes.
int affine_group_backward(nfb_flow* f, Group& g, int direction, const float* in, const float* g_out, const float* g_ld,
                          int64_t rows, float* ws, long long R, float* g_in, float* const* grad_slots, cudaStream_t st) {
    if (g.wide) return affine_wide_backward(f, g, direction, in, g_out, g_ld, rows, ws, R, g_in, grad_slots, st);
    const int n_items = (int)g.items.size();
    if (n_items) {
        // this call's output pointers, in slot order (a Linear takes two slots, a column sum one)
        if (!f->afb_ev) NFB_CUDA(cudaEventCreateWithFlags(&f->afb_ev, cudaEventDisableTiming));
        else NFB_CUDA(cudaEventSynchronize(f->afb_ev));   // the previous call's staging copy has been read
        if (f->afb_cap < (size_t)n_items) {
            if (f->afb_host) cudaFreeHost(f->afb_host);
            f->afb_host = nullptr; f->afb_cap = 0;
            NFB_CUDA(cudaMallocHost(reinterpret_cast<void**>(&f->afb_host), n_items * sizeof(AffRedItem)));
            f->afb_cap = n_items;
        }
        int s = 0;
        for (int i = 0; i < n_items; ++i) {
            AffRedItem it = g.items[i];
            if (it.n_in > 0) { it.dw = grad_slots ? grad_slots[s] : nullptr; it.db = grad_slots ? grad_slots[s + 1] : nullptr; s += 2; }
            else { it.db = grad_slots ? grad_slots[s] : nullptr; s += 1; }
            f->afb_host[i] = it;
        }
        NFB_TRY(f->afb_items.reserve(n_items * sizeof(AffRedItem)));
        NFB_CUDA(cudaMemcpyAsync(f->afb_items.p, f->afb_host, n_items * sizeof(AffRedItem), cudaMemcpyHostToDevice, st));
        NFB_CUDA(cudaEventRecord(f->afb_ev, st));
    }
    const int D = f->D, n_ops = g.last - g.first + 1;
    float* partial = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + (((size_t)g.units * R * 4 + 255) & ~(size_t)255));
    if (rows == 0) {   // zero parameter gradients
        NFB_TRY(launch_affine_bwd_reduce(f->afb_items.p, n_items, g.n_elem, ws, 0, partial, 0, st));
        f->launches += g.n_elem ? 1 : 0;
        return NFB_OK;
    }
    for (long long r0 = 0; r0 < rows; r0 += R) {
        const long long n = std::min(R, (long long)rows - r0);
        NFB_TRY(launch_affine_bwd_rows(g.ops.p, g.bops.p, n_ops, direction, in + r0 * D, g_out ? g_out + r0 * D : nullptr,
                                       g_ld ? g_ld + r0 : nullptr, g_in ? g_in + r0 * D : nullptr, ws, n, D, st));
        NFB_TRY(launch_affine_bwd_reduce(f->afb_items.p, n_items, g.n_elem, ws, n, partial, r0 > 0, st));
        f->launches += 1 + (g.n_elem ? 2 : 0);
    }
    return NFB_OK;
}

// the entry points' common checks; R = the chunk size the workspace is planned for
int affine_entry_checks(const char* who, nfb_flow* f, Group& g, const float* in, int64_t rows, void* ws,
                        int64_t ws_bytes, long long* R) {
    NFB_CHECK(rows >= 0, NFB_ERR_ARG, "rows < 0");
    NFB_CHECK(rows == 0 || in, NFB_ERR_ARG, "null input");
    *R = affine_bwd_chunk_rows(f, g, rows);
    NFB_CHECK(ws && ws_bytes >= (int64_t)affine_bwd_ws_bytes(f, g, *R), NFB_ERR_ARG,
              "%s backward: workspace of %lld bytes, %lld needed", who, (long long)ws_bytes,
              (long long)affine_bwd_ws_bytes(f, g, *R));
    return NFB_OK;
}

// ---- sampling-direction backward of a coupled-spline / LULinearPermute stack ----------------------------------------
// Every layer a CoupledRationalQuadraticSpline (no context; num_bins 8, the limit of the spline adjoint kernels) or an
// LULinearPermute (D <= 64): the coupled blocks fused or not, the LU maps paired with the block before them or alone.
bool coupled_lu_stack(const nfb_flow* f) {
    if (!f || !f->finalized || f->layers.empty()) return false;
    for (auto& Lp : f->layers)
        if (!(Lp->kind == L_LU || (Lp->kind == L_COUPLED_RQS && Lp->K == 8))) return false;
    return true;
}

// LULinearPermute, sampling direction: t = W^-1 (y - b) = y Ws^T + bs, x = t[:, inv_perm], log_det = -sum log diag.
// Given g (the cotangent of x) and xin (= y): g_t = g[:, perm], g_y = g_t Ws -> gin; W's gradient is
// -W^-T g_t t^T = -sum_rows g_y t^T, b's is -colsum(g_y), and -sum(g_ld) is the cotangent of log|det W|: the sums enter
// lu_param_bwd_kernel negated.  gld_sum: device scalar sum of g_ld; scratch: 64 + 64 x 64 floats (b's sums, dW).
int lu_sampling_backward(nfb_flow* f, Layer& L, const float* xin, const float* g, const float* gld_sum, long long rows,
                         float* gin, float* const* slots, float* scratch, cudaStream_t st) {
    const int D = L.D;
    NFB_TRY(f->tr_zp.reserve((size_t)rows * D * 4));
    NFB_TRY(f->tr_gzp.reserve((size_t)rows * D * 4));
    float* t = f->tr_zp.as<float>();
    float* gt = f->tr_gzp.as<float>();
    const GemmRun gr{f->err.as<int>(), st, nullptr, &f->launches};
    NFB_TRY(launch_gather_cols(g, gt, L.lu_perm.as<int>(), rows, D, 1, st));
    f->launches++;
    GemmTcArgs a{};
    a.A = gt; a.lda = D; a.B = L.lu_Ws.as<float>(); a.ldb = D; a.b_mn = 1; a.C = gin; a.ldc = D; a.M = rows; a.N = D; a.K = D;
    NFB_TRY(gr(a));
    if (slots[0] || slots[1] || slots[2]) {
        NFB_TRY(launch_linear(xin, D, nullptr, L.lu_Ws.as<float>(), L.lu_bs.as<float>(), nullptr, 0, t, D, rows, D, D, 0, 0,
                              0.f, st));
        f->launches++;
        float* dW = scratch + 64;
        GemmTcArgs w{};
        w.A = gin; w.lda = D; w.a_mn = 1; w.B = t; w.ldb = D; w.b_mn = 1; w.C = dW; w.ldc = D; w.M = D; w.N = D; w.K = rows;
        NFB_TRY(gr(w));
        NFB_TRY(launch_lu_param_bwd(dW, L.lu.lower_entries, L.lu.upper_entries, L.lu.unconstrained_upper_diag, L.lu.eps, D,
                                    gld_sum, slots[0], slots[1], slots[2], st, 1));
        f->launches++;
    }
    if (slots[3]) {
        NFB_CUDA(cudaMemsetAsync(scratch, 0, (size_t)D * 4, st));
        NFB_TRY(launch_colsum(gin, D, rows, D, scratch, st));
        NFB_TRY(launch_axpy(scratch, -1.f, slots[3], D, 0, st));
        f->launches += 3;
    }
    return NFB_OK;
}

// Coupling block, sampling direction (Coupling.inverse): x_id = the unconditional CDF's inverse at z_id, the conditioner
// reads x_id, x_tr = the inverse spline at z_tr with its per-row parameters.  zin: the block's input z, xout: its output x,
// g: the cotangent of x (its identity columns are updated in place), gld: of the log-det; writes g_z into gin.
int coupled_sampling_backward(nfb_flow* f, Layer& L, const float* zin, const float* xout, float* g, const float* gld,
                              long long rows, float* gin, float* const* slots, float* gtab, cudaStream_t st) {
    const int D = L.D, P = 3 * L.K - 1, nlin = 2 + 2 * L.net.nb;
    nfb_resnet_ctx_desc_t d;
    ResnetPass r;
    NFB_TRY(conditioner_recompute(f, L, xout, rows, d, r, st));
    // transform columns: inverse-spline adjoint -> gP, gin[:, tr]
    NFB_TRY(launch_spline_bwd_rows(zin, D, f->tr_P.as<float>(), g, gld, L.tr_idx.as<int>(), rows, L.n_tr, L.K, L.tail,
                                   L.wh_scale, f->tr_gP.as<float>(), gin, st, 1));
    f->launches++;
    // the conditioner's weights, and g[:, id] += its data gradient
    NFB_TRY(coupled_conditioner_adjoint(f, L, r, rows, slots, g, st));
    // identity columns: the unconditional CDF's inverse adjoint on the whole cotangent of x_id -> gin[:, id], table
    NFB_CUDA(cudaMemsetAsync(gtab, 0, (size_t)L.n_id * P * 4, st));
    NFB_TRY(launch_spline_bwd_shared(zin, D, L.uncond.as<float>(), g, gld, L.id_idx.as<int>(), rows, L.n_id, L.K, L.tail,
                                     gtab, gin, st, 1));
    NFB_TRY(launch_split_table(gtab, L.n_id, slots[2 * nlin], slots[2 * nlin + 1], slots[2 * nlin + 2], st));
    f->launches += 3;
    return NFB_OK;
}

// Recompute, then walk the layers last-to-first.  The recompute keeps each layer's input and, for a coupled block, its
// output (the conditioner reads x_id).  Whole-stack plan (f->fwd_n > 0): one launch of the persistent kernel, unit u
// ([LU map of layer fwd_units[u].first, if any] + block fwd_units[u].second) reading store[u] and writing store[u + 1];
// a block behind an LU map gets its input by that map again (launch_linear on lu_Ws / lu_bs), a trailing LU reads
// store[fwd_n].  Otherwise layer i runs on its own from store[i] into store[i + 1], as nfb_flow_transform runs it.
// Workspace: the flow's training buffers (tr_*).
int coupled_lu_sampling_backward(nfb_flow* f, const float* z, const float* g_x, const float* g_ld, int64_t rows,
                                 float* g_z, float* const* grad_slots, cudaStream_t st) {
    NFB_CHECK(rows >= 0, NFB_ERR_ARG, "rows < 0");
    NFB_CHECK(rows == 0 || z, NFB_ERR_ARG, "null z");
    const int n = (int)f->layers.size(), D = f->D;
    std::vector<int> off(n + 1, 0);
    for (int i = 0; i < n; ++i) off[i + 1] = off[i] + grad_slots_of(*f->layers[i]);
    std::vector<float*> slots(off[n], nullptr);
    if (grad_slots) std::copy(grad_slots, grad_slots + off[n], slots.begin());
    f->launches = 0;
    if (rows == 0) {   // zero gradients
        for (int i = 0; i < off[n]; ++i)
            if (slots[i]) NFB_CUDA(cudaMemsetAsync(slots[i], 0, (size_t)nfb_flow_grad_slot_numel(f, i) * 4, st));
        return NFB_OK;
    }
    const size_t ZS = (size_t)rows * D;
    const bool whole = f->fwd_n > 0;
    const int n_store = whole ? f->fwd_n + 1 : n + 1;
    int max_id = 0;
    for (auto& Lp : f->layers) max_id = std::max(max_id, Lp->n_id);
    NFB_TRY(ensure_ws(f, rows));
    NFB_TRY(f->tr_store.reserve((size_t)n_store * ZS * 4));
    NFB_TRY(f->tr_glq.reserve((size_t)rows * 4 + 64));
    NFB_TRY(f->tr_g0.reserve(ZS * 4));
    NFB_TRY(f->tr_g1.reserve(ZS * 4));
    NFB_TRY(f->tr_xp.reserve(ZS * 4));
    NFB_TRY(f->tr_small.reserve((size_t)(64 + 64 * 64 + 64 + (size_t)max_id * 23) * 4));
    float* store = f->tr_store.as<float>();
    float* lu_scratch = f->tr_small.as<float>();              // [64] LU bias sums, then [64 x 64] dW
    float* gld_sum = lu_scratch + 64 + 64 * 64;
    float* gtab = gld_sum + 64;
    // ---- recompute ----
    NFB_CUDA(cudaMemcpyAsync(store, z, ZS * 4, cudaMemcpyDeviceToDevice, st));
    float* ld = f->logq.as<float>();   // (the recompute's log-det is not used)
    NFB_TRY(launch_fill(ld, rows, 0.f, st));
    f->launches++;
    std::vector<const float*> src(n), out(n, nullptr);
    std::vector<int> lu_before(n, -1);
    if (whole) {
        NFB_TRY(launch_fused_stack(f, store, store + ZS, ld, rows, st, 1, (long long)ZS));
        for (int u = 0; u < f->fwd_n; ++u) {
            const int lu = f->fwd_units[u].first, b = f->fwd_units[u].second;
            if (lu >= 0) src[lu] = store + u * ZS;
            src[b] = store + u * ZS;
            lu_before[b] = lu;
            out[b] = store + (u + 1) * ZS;
        }
        if (f->fwd_trailing_lu >= 0) src[f->fwd_trailing_lu] = store + (size_t)f->fwd_n * ZS;
    } else {
        for (int i = 0; i < n; ++i) {
            Layer& L = *f->layers[i];
            src[i] = store + i * ZS;
            out[i] = store + (i + 1) * ZS;
            float* o = store + (i + 1) * ZS;
            if (L.kind == L_COUPLED_RQS && L.fused.ok)
                NFB_TRY(launch_fused_layer(f, L, nullptr, src[i], o, ld, rows, 1, st, 1));
            else
                NFB_TRY(apply_layer_generic(f, L, NFB_FORWARD, src[i], o, ld, rows, 1, st));
        }
    }
    // ---- backward ----
    float* g = f->tr_g0.as<float>();
    float* g2 = f->tr_g1.as<float>();
    if (g_x) NFB_CUDA(cudaMemcpyAsync(g, g_x, ZS * 4, cudaMemcpyDeviceToDevice, st));
    else NFB_CUDA(cudaMemsetAsync(g, 0, ZS * 4, st));
    const float* gld = g_ld;
    if (!gld) {
        NFB_TRY(launch_fill(f->tr_glq.as<float>(), rows, 0.f, st));
        gld = f->tr_glq.as<float>();
    }
    NFB_CUDA(cudaMemsetAsync(gld_sum, 0, 4, st));
    NFB_TRY(launch_colsum(gld, 1, rows, 1, gld_sum, st));
    f->launches += 3;
    for (int i = n - 1; i >= 0; --i) {
        Layer& L = *f->layers[i];
        const float* xin = src[i];
        if (lu_before[i] >= 0) {   // the block's input: the LU map in front of it, again
            NFB_TRY(apply_layer_generic(f, *f->layers[lu_before[i]], NFB_FORWARD, src[i], f->tr_xp.as<float>(), nullptr,
                                        rows, 1, st));
            xin = f->tr_xp.as<float>();
        }
        if (L.kind == L_LU)
            NFB_TRY(lu_sampling_backward(f, L, xin, g, gld_sum, rows, g2, slots.data() + off[i], lu_scratch, st));
        else
            NFB_TRY(coupled_sampling_backward(f, L, xin, out[i], g, gld, rows, g2, slots.data() + off[i], gtab, st));
        std::swap(g, g2);
    }
    if (g_z) NFB_CUDA(cudaMemcpyAsync(g_z, g, ZS * 4, cudaMemcpyDeviceToDevice, st));
    return NFB_OK;
}

}  // namespace

extern "C" {

int64_t nfb_flow_sampling_backward_workspace_bytes(const nfb_flow_t* fc, int64_t rows) {
    nfb_flow* f = const_cast<nfb_flow*>(fc);
    Group* g = planar_only_group(f);
    if (g) return rows < 0 ? -1 : (int64_t)planar_bwd_ws_bytes(*g, planar_bwd_chunk_rows(*g, rows));
    if (coupled_lu_stack(f)) return rows < 0 ? -1 : 0;   // (the flow's own training buffers serve)
    if (rows < 0 || affine_only_group(f, &g, "sampling") != NFB_OK) return -1;
    return (int64_t)affine_bwd_ws_bytes(f, *g, affine_bwd_chunk_rows(f, *g, rows));
}

int nfb_flow_sampling_backward(nfb_flow_t* f, const float* z, const float* g_x, const float* g_ld, int64_t rows,
                               void* ws, int64_t ws_bytes, float* g_z, float* const* grad_slots, void* stream) {
    if (Group* pg = planar_only_group(f))
        return planar_sampling_backward(f, *pg, z, g_x, g_ld, rows, ws, ws_bytes, g_z, grad_slots, S(stream));
    if (coupled_lu_stack(f)) return coupled_lu_sampling_backward(f, z, g_x, g_ld, rows, g_z, grad_slots, S(stream));
    Group* gp = nullptr;
    NFB_TRY(affine_only_group(f, &gp, "sampling"));
    long long R = 0;
    NFB_TRY(affine_entry_checks("sampling", f, *gp, z, rows, ws, ws_bytes, &R));
    f->launches = 0;
    return affine_group_backward(f, *gp, NFB_FORWARD, z, g_x, g_ld, rows, static_cast<float*>(ws), R, g_z, grad_slots,
                                 S(stream));
}

int64_t nfb_flow_density_backward_workspace_bytes(const nfb_flow_t* fc, int64_t rows) {
    Group* g = nullptr;
    nfb_flow* f = const_cast<nfb_flow*>(fc);
    if (rows < 0 || affine_only_group(f, &g, "density") != NFB_OK) return -1;
    return (int64_t)affine_bwd_ws_bytes(f, *g, affine_bwd_chunk_rows(f, *g, rows));
}

int nfb_flow_density_backward(nfb_flow_t* f, const float* x, const float* g_z, const float* g_ld, int64_t rows,
                              void* ws, int64_t ws_bytes, float* g_x, float* const* grad_slots, void* stream) {
    Group* gp = nullptr;
    NFB_TRY(affine_only_group(f, &gp, "density"));
    long long R = 0;
    NFB_TRY(affine_entry_checks("density", f, *gp, x, rows, ws, ws_bytes, &R));
    f->launches = 0;
    return affine_group_backward(f, *gp, NFB_INVERSE, x, g_z, g_ld, rows, static_cast<float*>(ws), R, g_x, grad_slots,
                                 S(stream));
}

}  // extern "C"
