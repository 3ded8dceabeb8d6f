// nfb_stochastic.cu -- the stochastic layers of a stochastic normalizing flow and Hamiltonian AIS (reference
// flows/stochastic.py HamiltonianMonteCarlo / MetropolisHastings, sampling/hais.py) on native densities: log p(z) =
// sum_i coef_i log p_i(z) over Gaussian mixtures (nfb_mixture.cuh mixture_row_log_prob_grad; a DiagGaussian is the
// one-mode mixture).
//
//   hmc_chain_kernel   one thread per row runs `transitions` HMC transitions back to back: momentum from the noise,
//                      the leapfrog steps with log p and grad log p in registers, the accept test, the log weight.  A
//                      HAIS run is one launch whatever the number of betas (per noise chunk, see normflows/sampling).
//   hmc_bwd_kernel     per accepted row, the leapfrog again (grad log p is a constant of the reference's graph, so
//                      z_L - z = L eps n exp(-lm/2) + eps^2 exp(-lm) S with S = L/2 g_0 + sum_{i=1}^{L-1} (L - i) g_i),
//                      and the row's contribution g_z_out * dz_L/dlog_step = g_z_out (A + 2B) into a feature-major
//                      [D, rows] workspace (dz_L/dlog_mass = -A/2 - B is exactly -1/2 of it)
//   feature_sum_kernel one CTA per feature sums the rows in a fixed order (fp64, coalesced reads): no atomics,
//                      identical bits per call; g_log_mass = -g_log_step / 2
//   mh_chain_kernel    MetropolisHastings with a diagonal Gaussian proposal, one thread per row, every step in registers
//
// The feature arrays of a row (z, the proposal, the momentum, the gradient) are register arrays of a compile-time
// bound DMAX in {4, 16, 64}; the row's D selects the smallest bound that holds it.
#include "../../include/nfb200.h"
#include "nfb_kernels.h"
#include "nfb_mixture.cuh"

namespace nfb {

namespace {

constexpr int kStoRows = 128;   // rows per CTA (one per thread)
constexpr int kSumThreads = 256;

// log p of the row at coefficients coef [n_terms]; with grad, grad log p is written to grad [D]
template <int DMAX>
__device__ __forceinline__ float density_lp(const nfb_density_t& P, const float* __restrict__ coef, const float* z,
                                           float* grad) {
    const int D = P.dim;
    if (grad) {
#pragma unroll
        for (int d = 0; d < DMAX; ++d) grad[d] = 0.f;
    }
    float lp = 0.f;
    for (int i = 0; i < P.n_terms; ++i) {
        const nfb_density_term_t& T = P.term[i];
        const float c = __ldg(coef + i);
        lp += c * mixture_row_log_prob_grad<DMAX, float>(z, D, T.loc, T.log_scale, T.weight_scores, T.n_modes, c, grad);
    }
    return lp;
}

// torch.clamp(g, -c, c) (NaN stays NaN); max_abs_grad = 0 is the reference's falsy "no clamp"
template <int DMAX>
__device__ __forceinline__ void clamp_grad(float* g, float c) {
    if (c == 0.f) return;
#pragma unroll
    for (int d = 0; d < DMAX; ++d) {
        float v = g[d] < -c ? -c : g[d];
        g[d] = v > c ? c : v;
    }
}

struct HmcArgs {
    nfb_density_t P;
    long long rows;
    int L;            // transitions
    int leapfrog;
    float max_abs_grad;
    const float* coef;       // [L, n_terms]
    const float* log_step;   // [L, D]
    const float* log_mass;   // [L, D]
    const float* noise;      // [L, rows, D]
    const float* unif;       // [L, rows]
};

template <int DMAX>
__global__ void __launch_bounds__(kStoRows) hmc_chain_kernel(HmcArgs a, const float* z_in,
                                                             float* z_out, float* log_w, uint8_t* accept) {
    const long long r = (long long)blockIdx.x * kStoRows + threadIdx.x;
    if (r >= a.rows) return;
    const int D = a.P.dim;
    float z[DMAX], zn[DMAX], p[DMAX], g[DMAX];
#pragma unroll
    for (int d = 0; d < DMAX; ++d) z[d] = d < D ? z_in[r * D + d] : 0.f;
    float lw = log_w ? log_w[r] : 0.f;
    for (int t = 0; t < a.L; ++t) {
        const float* coef = a.coef + (long long)t * a.P.n_terms;
        const float* lse = a.log_step + (long long)t * D;
        const float* lm = a.log_mass + (long long)t * D;
        const float* n = a.noise + ((long long)t * a.rows + r) * D;
        float k0 = 0.f;
#pragma unroll
        for (int d = 0; d < DMAX; ++d) {
            zn[d] = z[d];
            p[d] = 0.f;
            if (d < D) {
                p[d] = n[d] * expf(0.5f * __ldg(lm + d));
                k0 += p[d] * p[d] / expf(__ldg(lm + d));
            }
        }
        const float lp0 = density_lp<DMAX>(a.P, coef, zn, g);
        clamp_grad<DMAX>(g, a.max_abs_grad);
        float lp1 = lp0;
        for (int j = 0; j < a.leapfrog; ++j) {
#pragma unroll
            for (int d = 0; d < DMAX; ++d) {
                if (d < D) {
                    const float eps = expf(__ldg(lse + d));
                    p[d] = p[d] - (eps * 0.5f) * -g[d];
                    zn[d] = zn[d] + eps * (p[d] / expf(__ldg(lm + d)));
                }
            }
            lp1 = density_lp<DMAX>(a.P, coef, zn, g);
            clamp_grad<DMAX>(g, a.max_abs_grad);
#pragma unroll
            for (int d = 0; d < DMAX; ++d)
                if (d < D) p[d] = p[d] - (expf(__ldg(lse + d)) * 0.5f) * -g[d];
        }
        float k1 = 0.f;
#pragma unroll
        for (int d = 0; d < DMAX; ++d)
            if (d < D) k1 += p[d] * p[d] / expf(__ldg(lm + d));
        const float prob = expf(lp1 - lp0 - 0.5f * k1 + 0.5f * k0);
        const bool acc = a.unif[(long long)t * a.rows + r] < prob;   // NaN: reject; overflow to inf: accept
        if (acc) {
#pragma unroll
            for (int d = 0; d < DMAX; ++d) z[d] = zn[d];
        }
        lw += lp0 - (acc ? lp1 : lp0);
        if (accept) accept[(long long)t * a.rows + r] = acc;
    }
#pragma unroll
    for (int d = 0; d < DMAX; ++d)
        if (d < D) z_out[r * D + d] = z[d];
    if (log_w) log_w[r] = lw;
}

template <int DMAX>
__global__ void __launch_bounds__(kStoRows) hmc_bwd_kernel(HmcArgs a, const float* __restrict__ z_in,
                                                           const uint8_t* __restrict__ accept,
                                                           const float* __restrict__ g_out, float* __restrict__ contrib) {
    const long long r = (long long)blockIdx.x * kStoRows + threadIdx.x;
    if (r >= a.rows) return;
    const int D = a.P.dim;
    float* c = contrib + r;   // feature d of this row at c[d * rows]: a warp writes 32 consecutive floats
    if (!accept[r]) {
        for (int d = 0; d < D; ++d) c[d * a.rows] = 0.f;
        return;
    }
    const float* lse = a.log_step;
    const float* lm = a.log_mass;
    const float* n = a.noise + r * D;
    float zn[DMAX], p[DMAX], g[DMAX], S[DMAX];
#pragma unroll
    for (int d = 0; d < DMAX; ++d) {
        zn[d] = d < D ? z_in[r * D + d] : 0.f;
        p[d] = d < D ? n[d] * expf(0.5f * __ldg(lm + d)) : 0.f;
        S[d] = 0.f;
    }
    const int Lf = a.leapfrog;
    for (int j = 0; j < Lf; ++j) {
        density_lp<DMAX>(a.P, a.coef, zn, g);     // g_j at z_j (the forward's g_0 ... g_{L-1})
        clamp_grad<DMAX>(g, a.max_abs_grad);
        const float w = j == 0 ? 0.5f * (float)Lf : (float)(Lf - j);
#pragma unroll
        for (int d = 0; d < DMAX; ++d) {
            if (d < D) {
                const float eps = expf(__ldg(lse + d));
                S[d] += w * g[d];
                // the forward's p_half and z update (the closing half step of step j is the opening one of j + 1)
                p[d] = p[d] - (eps * 0.5f) * -g[d];
                if (j > 0) p[d] = p[d] - (eps * 0.5f) * -g[d];
                zn[d] = zn[d] + eps * (p[d] / expf(__ldg(lm + d)));
            }
        }
    }
#pragma unroll
    for (int d = 0; d < DMAX; ++d) {
        if (d < D) {
            const float eps = expf(__ldg(lse + d)), l = __ldg(lm + d);
            const float A = (float)Lf * eps * n[d] * expf(-0.5f * l);
            const float B = eps * eps * expf(-l) * S[d];
            c[d * a.rows] = g_out[r * D + d] * (A + 2.f * B);
        }
    }
}

// g_log_step[j] = sum_r v[j, r] over v [D, rows], in a fixed order; g_log_mass[j] = -g_log_step[j] / 2
__global__ void __launch_bounds__(kSumThreads) feature_sum_kernel(const float* __restrict__ v, long long rows,
                                                                  float* __restrict__ g_log_step,
                                                                  float* __restrict__ g_log_mass) {
    __shared__ double s[kSumThreads];
    const int j = blockIdx.x;
    const float* col = v + (long long)j * rows;
    double acc = 0.0;
    for (long long r = threadIdx.x; r < rows; r += kSumThreads) acc += col[r];
    s[threadIdx.x] = acc;
    __syncthreads();
    for (int h = kSumThreads / 2; h > 0; h >>= 1) {
        if (threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float g = (float)s[0];
        g_log_step[j] = g;
        g_log_mass[j] = -0.5f * g;
    }
}

template <int DMAX>
__global__ void __launch_bounds__(kStoRows) mh_chain_kernel(nfb_density_t P, long long rows, int steps,
                                                            const float* __restrict__ coef,
                                                            const float* __restrict__ scale,
                                                            const float* __restrict__ noise,
                                                            const float* __restrict__ unif,
                                                            const float* z_in, float* z_out,
                                                            float* __restrict__ log_det, uint8_t* __restrict__ moved) {
    const long long r = (long long)blockIdx.x * kStoRows + threadIdx.x;
    if (r >= rows) return;
    const int D = P.dim;
    float z[DMAX], zn[DMAX];
#pragma unroll
    for (int d = 0; d < DMAX; ++d) z[d] = d < D ? z_in[r * D + d] : 0.f;
    float lp0 = density_lp<DMAX>(P, coef, z, nullptr), ld = 0.f;
    bool any = false;
    for (int s = 0; s < steps; ++s) {
        const float* n = noise + ((long long)s * rows + r) * D;
#pragma unroll
        for (int d = 0; d < DMAX; ++d) zn[d] = d < D ? n[d] * __ldg(scale + d) + z[d] : 0.f;
        const float lp1 = density_lp<DMAX>(P, coef, zn, nullptr);
        float w_accept = expf(lp1 - lp0 + 0.f);         // log_p_diff of DiagGaussianProposal is 0
        w_accept = w_accept > 1.f ? 1.f : w_accept;      // torch.clamp(max=1): NaN stays NaN and rejects
        if (unif[(long long)s * rows + r] <= w_accept) {
#pragma unroll
            for (int d = 0; d < DMAX; ++d) z[d] = zn[d];
            ld = ld + (lp0 - lp1);
            lp0 = lp1;
            any = true;
        }
    }
#pragma unroll
    for (int d = 0; d < DMAX; ++d)
        if (d < D) z_out[r * D + d] = z[d];
    log_det[r] = ld;
    if (moved) moved[r] = any;
}

int check_density(const nfb_density_t& P, const char* who) {
    NFB_CHECK(P.n_terms >= 1 && P.n_terms <= NFB_DENSITY_MAX_TERMS, NFB_ERR_ARG, "%s: %d density terms (1 to %d)", who,
              P.n_terms, NFB_DENSITY_MAX_TERMS);
    NFB_CHECK(P.dim >= 1, NFB_ERR_ARG, "%s: dim %d", who, P.dim);
    NFB_CHECK(P.dim <= NFB_STOCHASTIC_MAX_DIM, NFB_ERR_UNSUPPORTED,
              "%s: dim %d; the stochastic kernels hold a row in registers and take at most %d features", who, P.dim,
              NFB_STOCHASTIC_MAX_DIM);
    for (int i = 0; i < P.n_terms; ++i)
        NFB_CHECK(P.term[i].n_modes >= 1 && P.term[i].loc && P.term[i].log_scale && P.term[i].weight_scores,
                  NFB_ERR_ARG, "%s: density term %d: %d modes or a null pointer", who, i, P.term[i].n_modes);
    return NFB_OK;
}

unsigned sto_blocks(long long rows) { return (unsigned)((rows + kStoRows - 1) / kStoRows); }

}  // namespace

int launch_hmc_chain(const nfb_density_t& P, long long rows, int L, int leapfrog, float max_abs_grad,
                     const float* coef, const float* log_step, const float* log_mass, const float* noise,
                     const float* unif, const float* z, float* z_out, float* log_w, uint8_t* accept, cudaStream_t st) {
    if (const int rc = check_density(P, "nfb_hmc_chain")) return rc;
    NFB_CHECK(rows >= 0 && L >= 0 && leapfrog >= 0, NFB_ERR_ARG, "nfb_hmc_chain: negative size");
    if (rows == 0 || L == 0) {
        if (rows > 0 && z_out != z) NFB_CUDA(cudaMemcpyAsync(z_out, z, rows * P.dim * 4, cudaMemcpyDeviceToDevice, st));
        return NFB_OK;
    }
    NFB_CHECK(coef && log_step && log_mass && noise && unif && z && z_out, NFB_ERR_ARG, "nfb_hmc_chain: null pointer");
    NFB_CHECK(sto_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_hmc_chain: %lld rows", rows);
    const HmcArgs a{P, rows, L, leapfrog, max_abs_grad, coef, log_step, log_mass, noise, unif};
    if (P.dim <= 4) hmc_chain_kernel<4><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, z_out, log_w, accept);
    else if (P.dim <= 16) hmc_chain_kernel<16><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, z_out, log_w, accept);
    else hmc_chain_kernel<64><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, z_out, log_w, accept);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

long long hmc_bwd_ws_bytes(long long rows, int D) { return rows * (long long)D * 4; }

int launch_hmc_bwd(const nfb_density_t& P, long long rows, int leapfrog, float max_abs_grad, const float* coef,
                   const float* log_step, const float* log_mass, const float* noise, const float* z,
                   const uint8_t* accept, const float* g_out, void* wsp, long long ws_bytes, float* g_log_step,
                   float* g_log_mass, cudaStream_t st) {
    if (const int rc = check_density(P, "nfb_hmc_backward")) return rc;
    NFB_CHECK(rows >= 0 && leapfrog >= 0, NFB_ERR_ARG, "nfb_hmc_backward: negative size");
    NFB_CHECK(g_log_step && g_log_mass, NFB_ERR_ARG, "nfb_hmc_backward: null pointer");
    const int D = P.dim;
    if (rows == 0) {
        NFB_CUDA(cudaMemsetAsync(g_log_step, 0, D * 4, st));
        NFB_CUDA(cudaMemsetAsync(g_log_mass, 0, D * 4, st));
        return NFB_OK;
    }
    NFB_CHECK(coef && log_step && log_mass && noise && z && accept && g_out && wsp, NFB_ERR_ARG,
              "nfb_hmc_backward: null pointer");
    NFB_CHECK(ws_bytes >= hmc_bwd_ws_bytes(rows, D), NFB_ERR_ARG, "nfb_hmc_backward: workspace of %lld bytes, needs %lld",
              ws_bytes, hmc_bwd_ws_bytes(rows, D));
    NFB_CHECK(sto_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_hmc_backward: %lld rows", rows);
    const HmcArgs a{P, rows, 1, leapfrog, max_abs_grad, coef, log_step, log_mass, noise, nullptr};
    float* contrib = static_cast<float*>(wsp);
    if (D <= 4) hmc_bwd_kernel<4><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, accept, g_out, contrib);
    else if (D <= 16) hmc_bwd_kernel<16><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, accept, g_out, contrib);
    else hmc_bwd_kernel<64><<<sto_blocks(rows), kStoRows, 0, st>>>(a, z, accept, g_out, contrib);
    feature_sum_kernel<<<D, kSumThreads, 0, st>>>(contrib, rows, g_log_step, g_log_mass);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

int launch_mh_chain(const nfb_density_t& P, long long rows, int steps, const float* coef, const float* scale,
                    const float* noise, const float* unif, const float* z, float* z_out, float* log_det,
                    uint8_t* moved, cudaStream_t st) {
    if (const int rc = check_density(P, "nfb_mh_chain")) return rc;
    NFB_CHECK(rows >= 0 && steps >= 0, NFB_ERR_ARG, "nfb_mh_chain: negative size");
    if (rows == 0) return NFB_OK;
    NFB_CHECK(coef && scale && z && z_out && log_det && (steps == 0 || (noise && unif)), NFB_ERR_ARG,
              "nfb_mh_chain: null pointer");
    NFB_CHECK(sto_blocks(rows) < (1u << 31), NFB_ERR_ARG, "nfb_mh_chain: %lld rows", rows);
    if (P.dim <= 4)
        mh_chain_kernel<4><<<sto_blocks(rows), kStoRows, 0, st>>>(P, rows, steps, coef, scale, noise, unif, z, z_out,
                                                                   log_det, moved);
    else if (P.dim <= 16)
        mh_chain_kernel<16><<<sto_blocks(rows), kStoRows, 0, st>>>(P, rows, steps, coef, scale, noise, unif, z, z_out,
                                                                    log_det, moved);
    else
        mh_chain_kernel<64><<<sto_blocks(rows), kStoRows, 0, st>>>(P, rows, steps, coef, scale, noise, unif, z, z_out,
                                                                    log_det, moved);
    NFB_LAUNCH_CHECK();
    return NFB_OK;
}

}  // namespace nfb
