// nfb_vae.cu -- the flow-VAE's encoder draw, its densities and the Bernoulli decoder likelihood (reference
// distributions/encoder.py, distributions/decoder.py, core.py NormalizingFlowVAE), forward and backward.  Element math
// in nfb_vae.cuh.
//
// Row layout: row r = b S + s of the flattened [B, S] sample grid belongs to data row b (sample-major, as the
// reference's view(-1, ...)).  A parameter row (mean, scale column) is read at row * param_stride; param_stride = 0 is
// one row shared by every row (ConstDiagGaussian's broadcast loc / scale).
//
// Forward kernels (draw, Gaussian density, Bernoulli): one warp per row, lanes over the columns, the row sum by a
// fixed xor-shuffle tree.
// Backward kernels: one thread per (group, column) -- a group is the run of rows that share one parameter row (the
// draw, the encoder's density) or one value row (the decoder's repeated x) -- walking the group's rows in order; for
// large groups (the const encoder's B S rows) a CTA column splits them over kGroupLanes lanes and sums the lanes'
// partials in lane order.  No atomics: two calls give identical bits.
#include "../../include/nfb200.h"
#include "nfb_common.cuh"
#include "nfb_vae.cuh"

#include <algorithm>

namespace nfb {
namespace {

constexpr int kRowsPerCta = 8;        // forward: warps (rows) per CTA
constexpr int kGroupCols = 32;        // backward: columns per CTA
constexpr int kGroupLanes = 8;        // backward: row lanes per column for groups of >= kWideGroup rows
constexpr long long kWideGroup = 256;
constexpr long long kMaxGridY = 65535;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__global__ void __launch_bounds__(32 * kRowsPerCta) vae_draw_kernel(
    const float* __restrict__ mean, const float* __restrict__ scale, long long pstride, int kind,
    const float* __restrict__ eps, long long rows, int samples, int D, float* __restrict__ z, float* __restrict__ log_q) {
    const long long r = (long long)blockIdx.x * kRowsPerCta + threadIdx.y;
    if (r >= rows) return;
    const long long prow = (r / samples) * pstride;
    float acc = 0.f;
    for (int j = threadIdx.x; j < D; j += 32) {
        float sd, lsd, nlq;
        vae_std(scale[prow + j], kind, sd, lsd);
        z[r * D + j] = vae_draw(mean[prow + j], sd, lsd, eps[r * D + j], nlq);
        acc += nlq;
    }
    acc = warp_sum(acc);
    if (threadIdx.x == 0) log_q[r] = -(float)D * (float)kVaeHalfLog2Pi - acc;
}

__global__ void __launch_bounds__(32 * kRowsPerCta) vae_density_kernel(
    const float* __restrict__ v, const float* __restrict__ mean, const float* __restrict__ scale, long long pstride,
    int kind, long long rows, int D, long long v_div, long long p_div, float norm_dim, float* __restrict__ out) {
    const long long r = (long long)blockIdx.x * kRowsPerCta + threadIdx.y;
    if (r >= rows) return;
    const long long vrow = (r / v_div) * D, prow = (r / p_div) * pstride;
    float acc = 0.f;
    for (int j = threadIdx.x; j < D; j += 32) {
        float sd, lsd;
        vae_std(scale[prow + j], kind, sd, lsd);
        acc += vae_density_term(v[vrow + j], mean[prow + j], sd, lsd);
    }
    acc = warp_sum(acc);
    if (threadIdx.x == 0) out[r] = -norm_dim * (float)kVaeHalfLog2Pi - acc;
}

// Adjoint of the draw (eps != nullptr; cotangents g_z [rows, D] and g [rows], either may be null) or of the density
// (eps == nullptr; cotangent g [rows], value rows v).  Group `gi` = rows [gi G, gi G + G):
//   group_params: the group shares parameter row gi (G = p_div, v_div = 1): g_mean / g_scale of row gi are the
//                 group's sums, g_v is written per row;
//   otherwise:    the group shares value row gi (G = v_div, p_div = 1): g_v of row gi is the group's sum, g_mean /
//                 g_scale are written per row.
__global__ void vae_group_bwd_kernel(const float* __restrict__ v, const float* __restrict__ eps,
                                     const float* __restrict__ mean, const float* __restrict__ scale, long long pstride,
                                     int kind, const float* __restrict__ g_z, const float* __restrict__ g,
                                     long long rows, int D, long long G, int group_params, float* __restrict__ g_v,
                                     float* __restrict__ g_mean, float* __restrict__ g_scale) {
    __shared__ float red[3][kGroupLanes][kGroupCols];
    const int j = blockIdx.x * kGroupCols + threadIdx.x;
    const bool col = j < D;
    const long long groups = (rows + G - 1) / G;
    for (long long gi = blockIdx.y; gi < groups; gi += gridDim.y) {
        const long long r0 = gi * G, r1 = min(rows, r0 + G);
        float a_m = 0.f, a_sd = 0.f, a_v = 0.f;
        float sd = 1.f, lsd = 0.f, m = 0.f;
        if (col && group_params) {
            m = mean[gi * pstride + j];
            vae_std(scale[gi * pstride + j], kind, sd, lsd);
        }
        for (long long r = r0 + threadIdx.y; col && r < r1; r += blockDim.y) {
            const float gr = g ? g[r] : 0.f;
            float gm, gsd, gv = 0.f;
            if (eps) {
                vae_draw_adjoint(sd, eps[r * D + j], g_z ? g_z[r * D + j] : 0.f, gr, gm, gsd);
            } else if (group_params) {
                vae_density_adjoint(v[r * D + j], m, sd, gr, gv, gm, gsd);
                if (g_v) g_v[r * D + j] = gv;
            } else {
                float sdr, lsdr;
                vae_std(scale[r * pstride + j], kind, sdr, lsdr);
                vae_density_adjoint(v[gi * D + j], mean[r * pstride + j], sdr, gr, gv, gm, gsd);
                if (g_mean) g_mean[r * pstride + j] = gm;
                if (g_scale) g_scale[r * pstride + j] = gsd * vae_dstd(sdr, kind);
                a_v += gv;
                continue;
            }
            a_m += gm;
            a_sd += gsd;
        }
        if (blockDim.y > 1) {   // the lanes' partials, summed in lane order
            __syncthreads();   // (the previous group's sums are read)
            red[0][threadIdx.y][threadIdx.x] = a_m;
            red[1][threadIdx.y][threadIdx.x] = a_sd;
            red[2][threadIdx.y][threadIdx.x] = a_v;
            __syncthreads();
            a_m = a_sd = a_v = 0.f;
            for (int l = 0; l < (int)blockDim.y; ++l) {
                a_m += red[0][l][threadIdx.x];
                a_sd += red[1][l][threadIdx.x];
                a_v += red[2][l][threadIdx.x];
            }
        }
        if (!col || threadIdx.y != 0) continue;
        if (group_params) {
            if (g_mean) g_mean[gi * pstride + j] = a_m;
            if (g_scale) g_scale[gi * pstride + j] = a_sd * vae_dstd(sd, kind);
        } else if (g_v) {
            g_v[gi * D + j] = a_v;
        }
    }
}

__global__ void __launch_bounds__(32 * kRowsPerCta) vae_bernoulli_kernel(
    const float* __restrict__ score, const float* __restrict__ x, long long rows, int D, long long x_div,
    float* __restrict__ out) {
    const long long r = (long long)blockIdx.x * kRowsPerCta + threadIdx.y;
    if (r >= rows) return;
    const float* s = score + r * D;
    const float* xr = x + (r / x_div) * D;
    float acc = 0.f;
    for (int j = threadIdx.x; j < D; j += 32) acc += vae_bernoulli_term(s[j], xr[j]);
    acc = warp_sum(acc);
    if (threadIdx.x == 0) out[r] = acc;
}

// one thread per (data row b, column j): g_score of the rows b x_div ... and, if wanted, their sum into g_x
__global__ void vae_bernoulli_bwd_kernel(const float* __restrict__ score, const float* __restrict__ x,
                                         const float* __restrict__ g, long long rows, int D, long long x_div,
                                         float* __restrict__ g_score, float* __restrict__ g_x) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= D) return;
    const long long n_b = (rows + x_div - 1) / x_div;
    for (long long b = blockIdx.y; b < n_b; b += gridDim.y) {
        const long long r0 = b * x_div, r1 = min(rows, r0 + x_div);
        const float xv = x[b * D + j];
        float acc = 0.f;
        for (long long r = r0; r < r1; ++r) {
            const float s = score[r * D + j], gr = g[r];
            if (g_score) g_score[r * D + j] = gr * vae_bernoulli_dscore(s, xv);
            acc += gr * s;
        }
        if (g_x) g_x[b * D + j] = acc;
    }
}

__global__ void vae_sigmoid_kernel(const float* __restrict__ in, float* __restrict__ out, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        out[i] = vae_sigmoid(in[i]);
}

__global__ void vae_sigmoid_bwd_kernel(const float* __restrict__ y, const float* __restrict__ gy,
                                       float* __restrict__ gin, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        gin[i] = gy[i] * y[i] * (1.f - y[i]);
}

unsigned row_blocks(long long rows) { return (unsigned)((rows + kRowsPerCta - 1) / kRowsPerCta); }

unsigned elem_blocks(long long n) { return (unsigned)std::min<long long>((n + 255) / 256, 8192); }

int launch_group_bwd(const float* v, const float* eps, const float* mean, const float* scale, long long pstride,
                     int kind, const float* g_z, const float* g, long long rows, int D, long long G, int group_params,
                     float* g_v, float* g_mean, float* g_scale, cudaStream_t st) {
    const long long groups = (rows + G - 1) / G;
    const dim3 grid((D + kGroupCols - 1) / kGroupCols, (unsigned)std::min<long long>(groups, kMaxGridY));
    const dim3 block(kGroupCols, G >= kWideGroup ? kGroupLanes : 1);
    vae_group_bwd_kernel<<<grid, block, 0, st>>>(v, eps, mean, scale, pstride, kind, g_z, g, rows, D, G, group_params,
                                                 g_v, g_mean, g_scale);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

// rows = 0: the gradients of a shared (stride-0) parameter row are zero; per-row parameters have no rows
int zero_shared_row(float* g_mean, float* g_scale, long long pstride, int D, cudaStream_t st) {
    if (pstride) return NFB_OK;
    if (g_mean) NFB_CUDA(cudaMemsetAsync(g_mean, 0, (size_t)D * 4, st));
    if (g_scale) NFB_CUDA(cudaMemsetAsync(g_scale, 0, (size_t)D * 4, st));
    return NFB_OK;
}

}  // namespace
}  // namespace nfb

using namespace nfb;

static cudaStream_t vae_stream(void* s) { return static_cast<cudaStream_t>(s); }

int nfb_vae_reparam_sample(const float* mean, const float* scale, int64_t param_stride, int32_t scale_kind,
                           const float* eps, int64_t batch, int32_t samples, int32_t dim, float* z, float* log_q,
                           void* stream) {
    NFB_CHECK(batch >= 0 && samples >= 1 && dim >= 1 && param_stride >= 0, NFB_ERR_ARG,
              "nfb_vae_reparam_sample: bad shape");
    NFB_CHECK(scale_kind == NFB_VAE_LOGVAR || scale_kind == NFB_VAE_SCALE, NFB_ERR_ARG,
              "nfb_vae_reparam_sample: unknown scale kind %d", scale_kind);
    const long long rows = (long long)batch * samples;
    if (rows == 0) return NFB_OK;
    NFB_CHECK(mean && scale && eps && z && log_q, NFB_ERR_ARG, "nfb_vae_reparam_sample: null pointer");
    NFB_CHECK(row_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_vae_reparam_sample: %lld rows", rows);
    vae_draw_kernel<<<row_blocks(rows), dim3(32, kRowsPerCta), 0, vae_stream(stream)>>>(
        mean, scale, param_stride, scale_kind, eps, rows, samples, dim, z, log_q);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int nfb_vae_reparam_sample_backward(const float* mean, const float* scale, int64_t param_stride, int32_t scale_kind,
                                    const float* eps, const float* g_z, const float* g_log_q, int64_t batch,
                                    int32_t samples, int32_t dim, float* g_mean, float* g_scale, void* stream) {
    NFB_CHECK(batch >= 0 && samples >= 1 && dim >= 1 && param_stride >= 0, NFB_ERR_ARG,
              "nfb_vae_reparam_sample_backward: bad shape");
    NFB_CHECK(scale_kind == NFB_VAE_LOGVAR || scale_kind == NFB_VAE_SCALE, NFB_ERR_ARG,
              "nfb_vae_reparam_sample_backward: unknown scale kind %d", scale_kind);
    const long long rows = (long long)batch * samples;
    cudaStream_t st = vae_stream(stream);
    if (rows == 0)   // only the shared row of a stride-0 encoder has gradients to zero
        return zero_shared_row(g_mean, g_scale, param_stride, dim, st);
    NFB_CHECK(mean && scale && eps, NFB_ERR_ARG, "nfb_vae_reparam_sample_backward: null pointer");
    return launch_group_bwd(nullptr, eps, mean, scale, param_stride, scale_kind, g_z, g_log_q, rows, dim,
                            param_stride ? samples : rows, 1, nullptr, g_mean, g_scale, st);
}

int nfb_vae_gaussian_log_prob(const float* v, const float* mean, const float* scale, int64_t param_stride,
                              int32_t scale_kind, int64_t rows, int32_t dim, int64_t v_div, int64_t p_div,
                              float norm_dim, float* out, void* stream) {
    NFB_CHECK(rows >= 0 && dim >= 1 && v_div >= 1 && p_div >= 1 && param_stride >= 0, NFB_ERR_ARG,
              "nfb_vae_gaussian_log_prob: bad shape");
    NFB_CHECK(scale_kind == NFB_VAE_LOGVAR || scale_kind == NFB_VAE_SCALE, NFB_ERR_ARG,
              "nfb_vae_gaussian_log_prob: unknown scale kind %d", scale_kind);
    if (rows == 0) return NFB_OK;
    NFB_CHECK(v && mean && scale && out, NFB_ERR_ARG, "nfb_vae_gaussian_log_prob: null pointer");
    NFB_CHECK(row_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_vae_gaussian_log_prob: %lld rows", (long long)rows);
    vae_density_kernel<<<row_blocks(rows), dim3(32, kRowsPerCta), 0, vae_stream(stream)>>>(
        v, mean, scale, param_stride, scale_kind, rows, dim, v_div, p_div, norm_dim, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int nfb_vae_gaussian_log_prob_backward(const float* v, const float* mean, const float* scale, int64_t param_stride,
                                       int32_t scale_kind, const float* g_out, int64_t rows, int32_t dim,
                                       int64_t v_div, int64_t p_div, float* g_v, float* g_mean, float* g_scale,
                                       void* stream) {
    NFB_CHECK(rows >= 0 && dim >= 1 && v_div >= 1 && p_div >= 1 && param_stride >= 0, NFB_ERR_ARG,
              "nfb_vae_gaussian_log_prob_backward: bad shape");
    NFB_CHECK(scale_kind == NFB_VAE_LOGVAR || scale_kind == NFB_VAE_SCALE, NFB_ERR_ARG,
              "nfb_vae_gaussian_log_prob_backward: unknown scale kind %d", scale_kind);
    // a stride-0 parameter row is shared by every row: one group
    const long long pd = param_stride ? p_div : (rows ? rows : 1);
    NFB_CHECK(v_div == 1 || pd == 1, NFB_ERR_UNSUPPORTED,
              "nfb_vae_gaussian_log_prob_backward: value rows and parameter rows cannot both repeat");
    cudaStream_t st = vae_stream(stream);
    if (rows == 0) return zero_shared_row(g_mean, g_scale, param_stride, dim, st);
    NFB_CHECK(v && mean && scale && g_out, NFB_ERR_ARG, "nfb_vae_gaussian_log_prob_backward: null pointer");
    const int group_params = v_div == 1;
    return launch_group_bwd(v, nullptr, mean, scale, param_stride, scale_kind, nullptr, g_out, rows, dim,
                            group_params ? pd : v_div, group_params, g_v, g_mean, g_scale, st);
}

int nfb_bernoulli_log_prob(const float* score, const float* x, int64_t rows, int32_t dim, int64_t x_div, float* out,
                           void* stream) {
    NFB_CHECK(rows >= 0 && dim >= 1 && x_div >= 1, NFB_ERR_ARG, "nfb_bernoulli_log_prob: bad shape");
    if (rows == 0) return NFB_OK;
    NFB_CHECK(score && x && out, NFB_ERR_ARG, "nfb_bernoulli_log_prob: null pointer");
    NFB_CHECK(row_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_bernoulli_log_prob: %lld rows", (long long)rows);
    vae_bernoulli_kernel<<<row_blocks(rows), dim3(32, kRowsPerCta), 0, vae_stream(stream)>>>(score, x, rows, dim,
                                                                                             x_div, out);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int nfb_bernoulli_log_prob_backward(const float* score, const float* x, const float* g_out, int64_t rows, int32_t dim,
                                    int64_t x_div, float* g_score, float* g_x, void* stream) {
    NFB_CHECK(rows >= 0 && dim >= 1 && x_div >= 1, NFB_ERR_ARG, "nfb_bernoulli_log_prob_backward: bad shape");
    if (rows == 0) return NFB_OK;
    NFB_CHECK(score && x && g_out, NFB_ERR_ARG, "nfb_bernoulli_log_prob_backward: null pointer");
    const long long groups = (rows + x_div - 1) / x_div;
    const int bx = dim >= 128 ? 128 : 32;
    vae_bernoulli_bwd_kernel<<<dim3((dim + bx - 1) / bx, (unsigned)std::min<long long>(groups, kMaxGridY)), bx, 0, vae_stream(stream)>>>(
        score, x, g_out, rows, dim, x_div, g_score, g_x);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int nfb_sigmoid(const float* in, float* out, int64_t n, void* stream) {
    NFB_CHECK(n >= 0, NFB_ERR_ARG, "nfb_sigmoid: negative size");
    if (n == 0) return NFB_OK;
    NFB_CHECK(in && out, NFB_ERR_ARG, "nfb_sigmoid: null pointer");
    vae_sigmoid_kernel<<<elem_blocks(n), 256, 0, vae_stream(stream)>>>(in, out, n);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int nfb_sigmoid_backward(const float* out, const float* g_out, float* g_in, int64_t n, void* stream) {
    NFB_CHECK(n >= 0, NFB_ERR_ARG, "nfb_sigmoid_backward: negative size");
    if (n == 0) return NFB_OK;
    NFB_CHECK(out && g_out && g_in, NFB_ERR_ARG, "nfb_sigmoid_backward: null pointer");
    vae_sigmoid_bwd_kernel<<<elem_blocks(n), 256, 0, vae_stream(stream)>>>(out, g_out, g_in, n);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}
