/* nfb200.h -- C ABI of libnfb200.so: the coupling-stack hot path of normflows as native H100 (sm_90a) kernels.
 *
 * The reference (normflows 1.7.3, pure Python/PyTorch) has no FFI; its seam for this path is the
 * `Flow` protocol `forward(z)/inverse(z) -> (z', log_det[B])` (normflows/flows/base.py:13-24) driven
 * by `NormalizingFlow.forward_kld / log_prob / inverse_and_log_det / forward_and_log_det`
 * (normflows/core.py:40-102,182-197).  This header is what a binding for that seam calls: plain
 * pointers and sizes, no torch types.  All tensors are fp32, row-major, contiguous.
 *
 *   - "dev" pointers are CUDA device pointers on the current device; `stream` is a cudaStream_t
 *     passed as void* (NULL = default stream).  Nothing here synchronises unless its name ends in
 *     `_host`; those take HOST pointers and include the host<->device copies (pinned or pageable).
 *   - Parameter descriptors carry the layer's parameters EXACTLY as the reference stores them in
 *     `state_dict()` (same shapes, nn.Linear [out,in] layout).  Packing for the kernels (mask
 *     pre-multiply, bf16 hi/lo split, swizzle, LU assembly) happens inside `nfb_flow_finalize` /
 *     `nfb_flow_repack`; the descriptor pointers must stay valid and are re-read on repack.
 *   - Every function returns 0 on success; on failure a non-zero code and `nfb_last_error()`
 *     holds a message (thread-local).  Argument errors mirror the reference's ValueErrors.
 *   - direction: NFB_INVERSE is the reference's `.inverse()` (density pass, x -> z);
 *     NFB_FORWARD is `.forward()` (sampling pass, z -> x).
 *
 * There is no CPU implementation behind this ABI: without a CUDA device every compute entry point
 * fails with NFB_ERR_CUDA.
 */
#ifndef NFB200_H
#define NFB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built -fvisibility=hidden; these are its exports */
#endif

#define NFB_ABI_VERSION 1
#define NFB_INVERSE 0
#define NFB_FORWARD 1

typedef struct nfb_flow nfb_flow_t;

/* ---- library ---- */
int nfb_abi_version(void);
const char* nfb_last_error(void);
/* sm count / compute capability of the current device */
int nfb_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---- stand-alone operators (device pointers) ---- */

/* utils/splines.py:16-97 `unconstrained_rational_quadratic_spline(tails="linear")`.
 * x,y: [rows, feats]; params: [rows, feats*(3*num_bins-1)] laid out per feature as
 * [widths(K) | heights(K) | derivatives(K-1)] (neural_spline/coupling.py:157-160,:330-332).
 * wh_scale multiplies the width/height logits (1/sqrt(hidden) in the coupling layer).
 * log_det: [rows]; += sum over features when `accumulate`, else overwritten.  May be NULL. */
int nfb_rqs_spline(const float* x_dev, const float* params_dev, float* y_dev, float* log_det_dev,
                   int64_t rows, int32_t feats, int32_t num_bins, float tail_bound, float wh_scale,
                   int32_t inverse, int32_t accumulate, void* stream);

/* The same spline with PER-FEATURE tails (utils/splines.py:42-57; the circular NSF layers of
 * flows/neural_spline/wrapper.py:88-183,247-311): params [rows, feats * (2K + num_derivatives)] with num_derivatives =
 * K + 1 (tails given as a list: every knot has a parameter; linear features overwrite both ends with the constant of
 * :35-38, circular features copy knot 0 into knot K; inputs outside a feature's interval come out as 0 with log-det 0 --
 * the reference's list branch never copies them, :31,48-57) or K (tails="circular": identity outside, :46-47).  tail_bound_dev[feats], circular_dev[feats]
 * (int32, != 0 = circular) live on the device. */
int nfb_rqs_spline_tails(const float* x_dev, const float* params_dev, float* y_dev, float* log_det_dev, int64_t rows,
                         int32_t feats, int32_t num_bins, int32_t num_derivatives, const float* tail_bound_dev,
                         const int32_t* circular_dev, float wh_scale, int32_t inverse, int32_t accumulate, void* stream);

/* utils/nn.py:64-130 PeriodicFeaturesElementwise.forward: y[r, j] = w[k,0] sin(scale[k] x) + w[k,1] cos(scale[k] x)
 * (+ bias[k]) for the features with slot_dev[j] = k >= 0, y = x for slot -1.  weights_dev [n_periodic, 2],
 * scale_dev / bias_dev [n_periodic] (bias may be NULL). */
int nfb_periodic_features(const float* x_dev, float* y_dev, int64_t rows, int32_t dim, const int32_t* slot_dev,
                          const float* weights_dev, const float* scale_dev, const float* bias_dev, void* stream);

/* ---- training pass of the stand-alone splines (density direction, inverse = 0): gradients of
 *   sum_r,j g_y[r, j] y[r, j] + sum_r g_log_det[r] log_det[r]
 * w.r.t. x and the parameters, with the forward's semantics in every tails mode (analytic adjoint, nfb_spline_bwd.cuh).
 * params_row_stride = feats * P (P = 2 num_bins + num_derivatives): one parameter record per element, g_params has the
 * same layout; params_row_stride = 0: ONE table [feats, P] shared by every row (the unconditional CDF of the coupling
 * layers), g_params [feats, P] receives the sum over rows.  g_y / g_log_det may be NULL (zero); g_x / g_params are
 * optional and overwritten.  Circular features: derivative K repeats derivative 0, so both gradients land on parameter
 * 2K (parameter 3K, in the tails-list layout, gets 0); tails-list inputs outside the interval come out as 0, so their
 * g_x and parameter gradients are 0; NaN inputs pass through. */
int nfb_rqs_spline_backward(const float* x_dev, const float* params_dev, int64_t params_row_stride, const float* g_y_dev,
                            const float* g_log_det_dev, float* g_x_dev, float* g_params_dev, int64_t rows, int32_t feats,
                            int32_t num_bins, float tail_bound, float wh_scale, void* stream);
int nfb_rqs_spline_tails_backward(const float* x_dev, const float* params_dev, int64_t params_row_stride,
                                  const float* g_y_dev, const float* g_log_det_dev, float* g_x_dev, float* g_params_dev,
                                  int64_t rows, int32_t feats, int32_t num_bins, int32_t num_derivatives,
                                  const float* tail_bound_dev, const int32_t* circular_dev, float wh_scale, void* stream);
/* ---- training pass of the stand-alone splines in the sampling direction (inverse = 1): gradients of
 * sum g_x . x + g_log_det . log_det through x = g(z), log_det = -sum log f'(x) (utils/splines.py:172-198), f the forward
 * spline.  Same arguments, layouts and conventions as the _backward pair above, but z_dev is the input of the inverse
 * spline and g_x_dev the cotangent of its output; g_z_dev receives the gradient of z.  The bin is the one the inverse
 * spline selects (search on the height knots at z), also for a z on an interior knot. */
int nfb_rqs_spline_inverse_backward(const float* z_dev, const float* params_dev, int64_t params_row_stride,
                                    const float* g_x_dev, const float* g_log_det_dev, float* g_z_dev,
                                    float* g_params_dev, int64_t rows, int32_t feats, int32_t num_bins, float tail_bound,
                                    float wh_scale, void* stream);
int nfb_rqs_spline_tails_inverse_backward(const float* z_dev, const float* params_dev, int64_t params_row_stride,
                                          const float* g_x_dev, const float* g_log_det_dev, float* g_z_dev,
                                          float* g_params_dev, int64_t rows, int32_t feats, int32_t num_bins,
                                          int32_t num_derivatives, const float* tail_bound_dev,
                                          const int32_t* circular_dev, float wh_scale, void* stream);
/* Adjoint of nfb_periodic_features: g_x (optional, overwritten; passes g_y through on non-periodic features),
 * g_weights [n_periodic, 2] and g_bias [n_periodic] (optional, overwritten with the sums over rows). */
int nfb_periodic_features_backward(const float* x_dev, const float* g_y_dev, int64_t rows, int32_t dim,
                                   const int32_t* slot_dev, const float* weights_dev, const float* scale_dev,
                                   int32_t n_periodic, float* g_x_dev, float* g_weights_dev, float* g_bias_dev,
                                   void* stream);

/* distributions/base.py:94-103 DiagGaussian.log_prob: log_q[r] (+)= log N(z_r; loc, exp(log_scale)) */
int nfb_diag_gaussian_log_prob(const float* z_dev, const float* loc_dev, const float* log_scale_dev,
                               float* log_q_dev, int64_t rows, int32_t dim, int32_t accumulate,
                               void* stream);

/* ---- invertible residual block (flows/residual.py:12-251, nets/lipschitz.py:14-67,642-648), element-wise pieces;
 * the Linear layers of g, of its Jacobian-vector and vector-Jacobian products run through nfb_gemm_f32 ---- */
/* Swish of the Lipschitz MLP: a = x sigmoid(b x) / 1.1 with b = softplus(beta); da (optional) = d a / d x */
int nfb_swish(const float* x_dev, float beta_softplus, int64_t n, float* a_dev, float* da_dev, void* stream);
/* dst[t*n + i] = src[t*n + i] * m[i], t < nt (tangents / cotangents through an activation; in place allowed) */
int nfb_mul_rows(const float* src_dev, const float* m_dev, int64_t n, int32_t nt, float* dst_dev, void* stream);
/* residual.py:148-161 (2-D, eval / brute_force): jt [2, batch, 2] = Jacobian columns -> out[r] = log|det(I + J_r)| */
int nfb_logabsdet_i_plus_j_2x2(const float* jt_dev, int64_t batch, float* out_dev, void* stream);
/* nets/resnet.py:48-50, nets/made.py:212-214: out = h + t * sigmoid(c), the GLU gate of a context-conditioned residual
 * block (t = block output, c = context_layer(context), h = block input); element-wise over n values */
int nfb_glu_residual(const float* h_dev, const float* t_dev, const float* c_dev, int64_t n, float* out_dev, void* stream);
/* Adjoint of nfb_glu_residual: g_h = g_out, g_t = g_out sigmoid(c), g_c = g_out t sigmoid'(c); each optional, g_t / g_c
 * may alias g_out. */
int nfb_glu_residual_backward(const float* g_out_dev, const float* t_dev, const float* c_dev, int64_t n, float* g_h_dev,
                              float* g_t_dev, float* g_c_dev, void* stream);
/* out[r] (+)= c * sum_j a[r, j] b[r, j]  (one Hutchinson trace term v^T J^k eps per sample, residual.py:355-366) */
int nfb_rowdot(const float* a_dev, const float* b_dev, int64_t rows, int32_t d, float c, int32_t accumulate,
               float* out_dev, void* stream);

/* ---- training pass of the residual block (`forward_kld(x).backward()` of examples/residual.ipynb) ----
 * g = Linear_L o Swish_L o ... o Linear_1 o Swish_1 (nets/lipschitz.py LipschitzMLP) pushed forward together with nt
 * tangents t_0 (the "dual" network: t_l = W_l (sigma_l'(h_{l-1}) * t_{l-1})), then reverse mode over it.  Stacked
 * tensors hold the primal rows first, then tangent 0, 1, ...: [(1 + nt) rows, width].
 * Swish: sigma(h) = h sigmoid(b h) / 1.1 with b = softplus(beta). */
#define NFB_LIPSCHITZ_MLP_MAX_LAYERS 8
typedef struct {
    int32_t num_layers;                                 /* Linear layers, 1 .. NFB_LIPSCHITZ_MLP_MAX_LAYERS */
    int32_t widths[NFB_LIPSCHITZ_MLP_MAX_LAYERS + 1];   /* widths[0] = input features, widths[num_layers] = output */
    const float* w[NFB_LIPSCHITZ_MLP_MAX_LAYERS];       /* effective weight W~_l [widths[l+1], widths[l]] (compute_weight) */
    const float* bias[NFB_LIPSCHITZ_MLP_MAX_LAYERS];    /* [widths[l+1]] */
    float b[NFB_LIPSCHITZ_MLP_MAX_LAYERS];              /* softplus(beta) of the Swish in front of Linear l */
} nfb_lipschitz_mlp_desc_t;
/* Bytes of device scratch nfb_lipschitz_mlp_dual_backward needs for `rows` rows and nt tangents (-1: bad descriptor). */
int64_t nfb_lipschitz_mlp_dual_backward_workspace_bytes(const nfb_lipschitz_mlp_desc_t* desc, int32_t nt, int64_t rows);
/* Gradients of  sum_r g_seed[r] . g(x_r) + sum_t sum_r t_seeds[t, r] . (J(x_r) tangents0[t, r])  w.r.t. x, every W~_l,
 * bias_l and b_l, in one call: the dual forward is recomputed from x and tangents0 [nt, rows, widths[0]], then the
 * adjoint runs layer by layer (dgrad and wgrad GEMMs on the tensor core over the stacked rows, the element-wise adjoint
 * of the Swish with its second derivative).  g_seed [rows, out] and t_seeds [nt, rows, out] may be NULL (zero).
 * Outputs, each OVERWRITTEN and each optional: gx [rows, widths[0]]; gW[l] [widths[l+1], widths[l]]; gbias[l];
 * gb [num_layers] (the b_l gradients, reduced in a fixed order: deterministic).  gW / gbias themselves may be NULL. */
int nfb_lipschitz_mlp_dual_backward(const nfb_lipschitz_mlp_desc_t* desc, const float* x_dev, const float* tangents0_dev,
                                    int32_t nt, const float* g_seed_dev, const float* t_seeds_dev, int64_t rows,
                                    void* workspace_dev, int64_t workspace_bytes, float* gx_dev, float* const* gW_dev,
                                    float* const* gbias_dev, float* gb_dev, void* stream);
/* The element-wise pieces of that pass, stand-alone (H, A: stacked [(1 + nt) rows, width]; H without the bias, which
 * is added to the primal rows; bias may be NULL).  swish_dual: A = [sigma(h); sigma'(h) t_1; ...].
 * swish_dual_adjoint: from Abar (the cotangent of A) writes hbar = sigma' abar + sigma'' sum_t t_t tabar_t to
 * out_primal [rows, width] and tbar_t = sigma' tabar_t to out_tangent [nt rows, width] (either may be NULL or alias
 * Abar), and *g_b_dev = d/db (fixed-order sum; partials_dev: NFB_SWISH_DUAL_PARTIALS doubles of scratch). */
#define NFB_SWISH_DUAL_PARTIALS 1024
int nfb_swish_dual(const float* H_dev, const float* bias_dev, float b, int64_t rows, int32_t width, int32_t nt,
                   float* A_dev, void* stream);
int nfb_swish_dual_adjoint(const float* H_dev, const float* bias_dev, float b, int64_t rows, int32_t width, int32_t nt,
                           const float* Abar_dev, float* out_primal_dev, float* out_tangent_dev, double* partials_dev,
                           float* g_b_dev, void* stream);
/* Adjoint of nfb_logabsdet_i_plus_j_2x2: seeds [2, batch, 2] = g_ld[r] * (column t of (I + J_r)^-T). */
int nfb_logabsdet_i_plus_j_2x2_backward(const float* jt_dev, const float* g_ld_dev, int64_t batch, float* seeds_dev,
                                        void* stream);

/* flows/affine/autoregressive.py:96-128 MaskedAffineAutoregressive, element-wise part: params [rows, features, 2] =
 * (unconstrained_scale, shift) from the MADE conditioner; scale = sigmoid(u + 2) + 1e-3.  inverse = 0: y = scale x + shift,
 * log_det (+)= sum log scale; inverse = 1: y = (x - shift) / scale, log_det (+)= -sum log scale. */
int nfb_maf_affine(const float* x_dev, const float* params_dev, float* y_dev, float* log_det_dev, int64_t rows,
                   int32_t features, int32_t inverse, int32_t accumulate, void* stream);

/* transforms.py:8-47 Logit pre-transform of image data (RealNVP): direction NFB_INVERSE = Logit.inverse (density pass:
 * y = logit(alpha + (1 - 2 alpha) x)), NFB_FORWARD = Logit.forward (sampling); log_det[b] (+)= the per-sample log-det
 * over the `inner` elements of sample b.  in/out: [batch, inner] contiguous; may alias. */
int nfb_logit_transform(const float* in_dev, float* out_dev, float* log_det_dev, int64_t batch, int64_t inner,
                        float alpha, int32_t direction, int32_t accumulate, void* stream);

/* Dense product of the training pass (what `F.linear` and its autograd formulas compute for every Linear of the
 * conditioners: nets/resnet.py:37-50,92-104, nets/made.py:80-81,199-214): C[M x N] (+)= opA(A) opB(B)^T on the tensor
 * core (split-bf16, fp32 accumulate).  A, B, C are row-major fp32 device matrices; `a_mn` / `b_mn` = 1 say that the
 * operand is stored with its M / N dimension contiguous (element (i, k) at base[k*ld + i]) -- forward Y = X W^T is
 * (0, 0), dgrad gX = gY W is (0, 1) with B = W, wgrad dW = gY^T X is (1, 1) with A = gY, B = X.  Optional fused
 * epilogue: + bias[N]; * (mask[M x N] > 0); * mulm[M x N]; + resid[M x N]; ReLU; `a_relu` / `b_relu` apply ReLU to an
 * operand while it is loaded; `accumulate` adds into C (red.global.add).  Products whose output has few tiles are
 * split along K automatically (C is zeroed first unless `accumulate`). */
typedef struct nfb_gemm_desc {
    const float* A; const float* B; float* C;
    int64_t lda, ldb, ldc, M, N, K;
    int32_t a_mn, b_mn, a_relu, b_relu, relu_out, accumulate;
    const float* bias; const float* mask; const float* mulm; int64_t ldmask; const float* resid; int64_t ldres;
} nfb_gemm_desc_t;
int nfb_gemm_f32(const nfb_gemm_desc_t* desc, void* stream);

/* ---- image-shaped (NCHW) operators of the Glow block, density direction (device pointers) ---- */

/* nets/cnn.py:33-61 one layer of ConvNet2d: y = act(conv2d(x[:, c0:c0+cin], w[cout,cin,k,k], stride 1, pad k/2) + b);
 * x is a channel slice of an NCHW tensor with `x_channels` channels; leaky < 0 means no activation,
 * otherwise LeakyReLU(leaky) (0 = ReLU).  y: [B, cout, H, W]. */
int nfb_conv2d(const float* x_dev, int32_t x_channels, int32_t c0, const float* w_dev, const float* b_dev,
               float* y_dev, int64_t batch, int32_t cin, int32_t height, int32_t width, int32_t cout,
               int32_t ksize, float leaky, void* stream);
/* nets/cnn.py:33-61 ConvNet2d with kernel sizes (3, 1, 3) -- the parameter map of a GlowBlock's coupling
 * (flows/affine/glow.py:48-62) -- as ONE kernel: conv3x3 + LeakyReLU, conv1x1 + LeakyReLU and the nine stacked 1x1
 * products of the last 3x3 convolution, the two hidden tensors never leaving the SM.  x: channel slice [c0, c0+cin) of
 * an NCHW tensor with `x_channels` channels; w1 [hidden, cin, 3, 3], w2 [hidden, hidden(,1,1)], w3_taps [9*cout, hidden]
 * (row (kh*3+kw)*cout + n = W3[n, :, kh, kw]); y_taps: [B, 9*cout, H, W], to be summed by nfb_tap_shift_add (+ bias). */
int nfb_glow_conditioner(const float* x_dev, int32_t x_channels, int32_t c0, int32_t cin, const float* w1_dev,
                         const float* b1_dev, const float* w2_dev, const float* b2_dev, const float* w3_taps_dev,
                         float* y_taps_dev, int64_t batch, int32_t height, int32_t width, int32_t hidden, int32_t cout,
                         float leaky, void* stream);
/* The same conditioner with its weights PRE-PACKED (bf16 hi | lo records in the kernel's swizzled layout): pack once per
 * parameter version with nfb_glow_conditioner_pack into a device buffer of nfb_glow_conditioner_packed_bytes(...) bytes
 * (-1: shape not supported), then call nfb_glow_conditioner_packed on every pass. */
int64_t nfb_glow_conditioner_packed_bytes(int32_t cin, int32_t hidden, int32_t cout);
int nfb_glow_conditioner_pack(const float* w1_dev, const float* w2_dev, const float* w3_taps_dev, int32_t cin,
                              int32_t hidden, int32_t cout, void* packed_dev, void* stream);
int nfb_glow_conditioner_packed(const float* x_dev, int32_t x_channels, int32_t c0, int32_t cin, const void* packed_dev,
                                const float* b1_dev, const float* b2_dev, float* y_taps_dev, int64_t batch,
                                int32_t height, int32_t width, int32_t hidden, int32_t cout, float leaky, void* stream);
/* flows/affine/glow.py:72-84 GlowBlock.forward / .inverse as ONE call: [AffineCouplingBlock(ConvNet2d (3,1,3)),
 * Invertible1x1Conv, ActNorm] with the parameter preparation done once per parameter version by the caller --
 * w1x1 [C, C], b1x1 [C], logdet_const (device scalar): the folded 1x1 convolution of nfb_glow_fold_actnorm_conv1x1
 * (density) / nfb_glow_fold_conv1x1_actnorm_forward (sampling); cond_packed: nfb_glow_conditioner_pack; cond_b1/b2/b3:
 * the three convolution biases.  z_in, z_out: [B, C, H, W] (distinct); y_taps: work space [B, 9 * cout, H, W] with
 * cout = (scale ? 2 : 1) * #transformed channels; scratch: [B, C, H, W], sampling direction only; log_det [B] is
 * overwritten.  NFB_ERR_UNSUPPORTED when the conditioner shape is outside the fused kernels. */
int nfb_glow_block(const float* z_in_dev, float* z_out_dev, float* scratch_dev, float* y_taps_dev, float* log_det_dev,
                   const float* w1x1_dev, const float* b1x1_dev, const float* logdet_const_dev, const void* cond_packed_dev,
                   const float* cond_b1_dev, const float* cond_b2_dev, const float* cond_b3_dev, int64_t batch,
                   int32_t channels, int32_t height, int32_t width, int32_t hidden, int32_t scale, int32_t scale_map,
                   int32_t split_mode, float leaky, int32_t direction, void* stream);
/* Second half of a k x k convolution computed as k*k stacked 1x1 products (the last, 256 -> few-channel layer of
 * ConvNet2d, nets/cnn.py:50-57): y_taps [B, k*k*cout, H, W] holds, for tap t = kh*k + kw, channel t*cout + n =
 * sum_c W[n, c, kh, kw] x[b, c]; out[b, n, y, x] = bias[n] + sum_t y_taps[b, t*cout + n, y + kh - k/2, x + kw - k/2]. */
int nfb_tap_shift_add(const float* y_taps_dev, const float* bias_dev, float* out_dev, int64_t batch, int32_t cout,
                      int32_t height, int32_t width, int32_t ksize, void* stream);
/* flows/normalization.py:31-39 ActNorm.inverse followed by flows/mixing.py:123-133 Invertible1x1Conv.inverse
 * (LU parameterisation :88-104) folded into one 1x1 convolution: w_out[C,C], b_out[C] for nfb_conv2d, and
 * *logdet_out = H*W*(sum log_S - sum s), the per-sample log|det| of both layers. */
int nfb_glow_fold_actnorm_conv1x1(const float* P, const float* L, const float* U, const float* sign_S,
                                  const float* log_S, const float* s, const float* t, int32_t channels,
                                  int32_t hw, float* w_out, float* b_out, float* logdet_out, void* stream);
/* Sampling direction of the same two layers: Invertible1x1Conv.forward (flows/mixing.py:106-121; W^-1 formed in
 * double precision like :94-101) followed by ActNorm.forward (flows/affine/coupling.py:38-45), folded into one
 * 1x1 convolution: w_out = diag(exp(s)) W^-1, b_out = t, *logdet_out = H*W*(sum s - sum log_S).  channels <= 64. */
int nfb_glow_fold_conv1x1_actnorm_forward(const float* P, const float* L, const float* U, const float* sign_S,
                                          const float* log_S, const float* s, const float* t, int32_t channels,
                                          int32_t hw, float* w_out, float* b_out, float* logdet_out, void* stream);
/* flows/affine/coupling.py:113-171 AffineCoupling on images, in place on the z2 channels of z [B,C,H,W];
 * param = conditioner output [B, (scale?2:1)*n2, H, W] with shift/scale interleaved (:152-153).
 * scale_map 0 exp / 1 sigmoid / 2 sigmoid_inv; split_mode 0 channel / 1 channel_inv (reshape.py:27-31).
 * log_det[b] (+)= sum of log-scale terms + *logdet_const (may be NULL). */
int nfb_affine_coupling_image(float* z_dev, const float* param_dev, float* log_det_dev,
                              const float* logdet_const_dev, int64_t batch, int32_t channels, int32_t hw,
                              int32_t scale, int32_t scale_map, int32_t split_mode, int32_t direction,
                              int32_t accumulate, void* stream);
/* The same coupling fed with the conditioner's output still in tap form (nfb_glow_conditioner*: y_taps [B, 9 * cout, H, W]
 * with cout = (scale ? 2 : 1) * #transformed channels, bias [cout] or NULL): param[b, n, y, x] = bias[n] + sum over the
 * nine taps of y_taps[b, t * cout + n, y + kh - 1, x + kw - 1] is formed on the fly from a shared-memory copy of the
 * sample -- nfb_tap_shift_add and the summed parameter tensor are skipped.  ..._supported: 1 if one sample's taps
 * (9 * cout * H * W floats) fit the kernel's shared memory (200 KB). */
int nfb_affine_coupling_image_taps(float* z_dev, const float* y_taps_dev, const float* bias_dev, float* log_det_dev,
                                   const float* logdet_const_dev, int64_t batch, int32_t channels, int32_t height,
                                   int32_t width, int32_t scale, int32_t scale_map, int32_t split_mode, int32_t direction,
                                   int32_t accumulate, void* stream);
int32_t nfb_affine_coupling_image_taps_supported(int32_t channels, int32_t height, int32_t width, int32_t scale);
/* flows/reshape.py:114-128 Squeeze; (channels,height,width) describe the high-resolution side;
 * NFB_INVERSE: [B,C,H,W] -> [B,4C,H/2,W/2], NFB_FORWARD the reverse. */
int nfb_squeeze(const float* in_dev, float* out_dev, int64_t batch, int32_t channels, int32_t height,
                int32_t width, int32_t direction, void* stream);
/* flows/reshape.py:27-31 channel chunk made contiguous: out[b,j,:] = in[b,c0+j,:] */
int nfb_copy_channels(const float* in_dev, float* out_dev, int64_t batch, int32_t channels, int32_t c0,
                      int32_t n, int32_t hw, void* stream);
/* flows/reshape.py:68-74 Merge.forward on images: out[b,c0+j,:] = in[b,j,:] (out has `channels` channels) */
int nfb_paste_channels(const float* in_dev, float* out_dev, int64_t batch, int32_t channels, int32_t c0,
                       int32_t n, int32_t hw, void* stream);
/* distributions/base.py:327-344 ClassCondDiagGaussian.log_prob with integer labels y[B] (int64);
 * loc/log_scale: [dim, num_classes] (the reference's (*shape, num_classes) flattened). */
int nfb_class_cond_diag_gaussian_log_prob(const float* z_dev, const int64_t* y_dev, const float* loc_dev,
                                          const float* log_scale_dev, float* log_q_dev, int64_t batch,
                                          int32_t dim, int32_t num_classes, int32_t accumulate, void* stream);

/* ---- training pass of the image path (`MultiscaleFlow.forward_kld(x, y).backward()`, examples/glow.ipynb cell 4) ----
 * Adjoints of the density-direction operators above; g_* are gradients of a scalar loss. */

/* Weight / bias gradient of nfb_conv2d: gw[n, c, kh, kw] (+)= sum_{b,h,w} gy[b, n, h, w] x[b, c0+c, h+kh-k/2, w+kw-k/2]
 * and gb[n] (+)= sum_{b,h,w} gy[b, n, h, w] (gw or gb may be NULL); k = 1, 3 or 5.  Tensor core (split bf16, fp32
 * accumulation over pixel splits of <= 2048 pixels, splits summed in fp64): deterministic. */
int nfb_conv2d_wgrad(const float* x_dev, int32_t x_channels, int32_t c0, const float* gy_dev, float* gw_dev, float* gb_dev,
                     int64_t batch, int32_t cin, int32_t height, int32_t width, int32_t cout, int32_t ksize,
                     int32_t accumulate, void* stream);
/* Data gradient of nfb_conv2d (w [cout, cin, k, k]): gx [B, cin, H, W] (+)= conv2d(gy, w rotated by 180 degrees with
 * in/out swapped); mask_act (optional, [B, cin, H, W]) multiplies the result by LeakyReLU'(mask_act) =
 * (mask_act > 0 ? 1 : mask_slope) -- the post-activation tensor of the layer input suffices for slope >= 0. */
int nfb_conv2d_dgrad(const float* gy_dev, const float* w_dev, float* gx_dev, int64_t batch, int32_t cin, int32_t height,
                     int32_t width, int32_t cout, int32_t ksize, const float* mask_act_dev, float mask_slope,
                     int32_t accumulate, void* stream);
/* Adjoint of nfb_affine_coupling_image in the density direction: z = the coupling's input [B, C, H, W], param its
 * conditioner output, g_out [B, C, H, W], g_log_det [B] (may be NULL).  Writes the z2 channels of g_z [B, C, H, W]
 * (its z1 channels are left to the caller) and g_param [B, (scale?2:1)*n2, H, W] in param's interleaved layout. */
int nfb_affine_coupling_image_backward(const float* z_dev, const float* param_dev, const float* g_out_dev,
                                       const float* g_log_det_dev, float* g_z_dev, float* g_param_dev, int64_t batch,
                                       int32_t channels, int32_t hw, int32_t scale, int32_t scale_map, int32_t split_mode,
                                       void* stream);
/* Adjoint of a diagonal-Gaussian density with parameter tables (DiagGaussian, ClassCondDiagGaussian, GlowBase;
 * distributions/base.py): element i of a sample uses entry i / group of loc / log_scale [dim / group, num_classes] in
 * column y[b] (y NULL: num_classes = 1).  g_z [B, dim] (may be NULL) is overwritten; g_loc / g_log_scale (may be NULL)
 * receive the batch sums, formed deterministically (per-sample partials, fixed-order reduction). */
int nfb_gaussian_table_log_prob_backward(const float* z_dev, const int64_t* y_dev, const float* loc_dev,
                                         const float* log_scale_dev, const float* g_log_q_dev, float* g_z_dev,
                                         float* g_loc_dev, float* g_log_scale_dev, int64_t batch, int32_t dim,
                                         int32_t group, int32_t num_classes, void* stream);
/* distributions/base.py:573-659 GaussianMixture.log_prob: log_q[r] (+)= logsumexp_k [log_softmax(weight_scores)_k
 * - dim/2 log 2pi - sum_d log_scale[k,d] - 1/2 sum_d ((z[r,d] - loc[k,d]) / exp(log_scale[k,d]))^2], loc / log_scale
 * [n_modes, dim], weight_scores [n_modes].  Any n_modes >= 1 and dim >= 1; one launch.  log_softmax, not log(softmax):
 * a weight that underflows in the reference gives a finite, negligible term (and finite gradients) instead of -inf. */
int nfb_gaussian_mixture_log_prob(const float* z_dev, const float* loc_dev, const float* log_scale_dev,
                                  const float* weight_scores_dev, float* log_q_dev, int64_t rows, int32_t n_modes,
                                  int32_t dim, int32_t accumulate, void* stream);
/* Adjoint of nfb_gaussian_mixture_log_prob (accumulate = 0) with row cotangents g_log_q [rows]: g_z [rows, dim] and the
 * parameter gradients g_loc / g_log_scale [n_modes, dim], g_weight_scores [n_modes] are overwritten (each may be NULL).
 * Deterministic (fixed-order sums, no atomics) in two launches whatever rows and n_modes; the workspace
 * (nfb_gaussian_mixture_log_prob_backward_workspace_bytes, -1 for a bad shape) does not grow with rows beyond 256 row
 * blocks and stays under 64 MiB unless one copy of the parameters' gradients is larger.  rows = 0 writes zeros. */
int64_t nfb_gaussian_mixture_log_prob_backward_workspace_bytes(int64_t rows, int32_t n_modes, int32_t dim);
int nfb_gaussian_mixture_log_prob_backward(const float* z_dev, const float* loc_dev, const float* log_scale_dev,
                                           const float* weight_scores_dev, const float* g_log_q_dev, int64_t rows,
                                           int32_t n_modes, int32_t dim, void* ws, int64_t ws_bytes, float* g_z_dev,
                                           float* g_loc_dev, float* g_log_scale_dev, float* g_weight_scores_dev,
                                           void* stream);
/* ---- flow-VAE encoders and decoders (distributions/encoder.py, distributions/decoder.py) ----
 * Row r = b samples + s of a flattened [batch, samples] grid belongs to data row b.  A parameter row (mean and scale
 * column, each dim floats) sits at row * param_stride floats; param_stride = 0 is one row shared by every row.  The
 * scale column holds the log variance (NFB_VAE_LOGVAR: sd = exp(p / 2)) or the standard deviation (NFB_VAE_SCALE).
 * Every backward is deterministic (fixed-order sums, no atomics), one launch, and overwrites its outputs; rows = 0
 * writes zeros into the gradients of a shared (param_stride = 0) row. */
#define NFB_VAE_LOGVAR 0
#define NFB_VAE_SCALE 1
/* z [rows, dim] = mean[b] + sd[b] eps[r] and log_q [rows] = -dim/2 log 2pi - sum (log sd + eps^2 / 2), one launch. */
int nfb_vae_reparam_sample(const float* mean_dev, const float* scale_dev, int64_t param_stride, int32_t scale_kind,
                           const float* eps_dev, int64_t batch, int32_t samples, int32_t dim, float* z_dev,
                           float* log_q_dev, void* stream);
/* Adjoint of nfb_vae_reparam_sample with cotangents g_z [rows, dim] and g_log_q [rows] (either may be NULL): g_mean and
 * g_scale (the scale column's gradient) in the parameter layout, summed over each row's samples (over all rows for
 * param_stride = 0). */
int nfb_vae_reparam_sample_backward(const float* mean_dev, const float* scale_dev, int64_t param_stride,
                                    int32_t scale_kind, const float* eps_dev, const float* g_z_dev,
                                    const float* g_log_q_dev, int64_t batch, int32_t samples, int32_t dim,
                                    float* g_mean_dev, float* g_scale_dev, void* stream);
/* out[r] = -norm_dim/2 log 2pi - sum_j (log sd + (v - mean)^2 / (2 sd^2)) with value row r / v_div of v [., dim]
 * and parameter row r / p_div. */
int nfb_vae_gaussian_log_prob(const float* v_dev, const float* mean_dev, const float* scale_dev, int64_t param_stride,
                              int32_t scale_kind, int64_t rows, int32_t dim, int64_t v_div, int64_t p_div,
                              float norm_dim, float* out_dev, void* stream);
/* Adjoint of nfb_vae_gaussian_log_prob with cotangent g_out [rows]: g_v (summed over the rows that share a value row),
 * g_mean / g_scale (summed over the rows that share a parameter row); each may be NULL.  Value rows and parameter rows
 * may not both repeat (NFB_ERR_UNSUPPORTED). */
int nfb_vae_gaussian_log_prob_backward(const float* v_dev, const float* mean_dev, const float* scale_dev,
                                       int64_t param_stride, int32_t scale_kind, const float* g_out_dev, int64_t rows,
                                       int32_t dim, int64_t v_div, int64_t p_div, float* g_v_dev, float* g_mean_dev,
                                       float* g_scale_dev, void* stream);
/* Bernoulli log-likelihood of x row r / x_div under logits score [rows, dim]: out[r] = sum_j x log_sig(s) +
 * (1 - x) log_sig(-s) (NNBernoulliDecoder.log_prob). */
int nfb_bernoulli_log_prob(const float* score_dev, const float* x_dev, int64_t rows, int32_t dim, int64_t x_div,
                           float* out_dev, void* stream);
/* Adjoint with cotangent g_out [rows]: g_score = g (x - sigmoid(s)), 0 where s == 0 exactly (as the reference's
 * relu / abs derivatives give); g_x [rows / x_div, dim] = sum over the rows sharing x of g s.  Either may be NULL. */
int nfb_bernoulli_log_prob_backward(const float* score_dev, const float* x_dev, const float* g_out_dev, int64_t rows,
                                    int32_t dim, int64_t x_div, float* g_score_dev, float* g_x_dev, void* stream);
/* out = sigmoid(in) elementwise (NNBernoulliDecoder.forward), and its adjoint g_in = g_out out (1 - out). */
int nfb_sigmoid(const float* in_dev, float* out_dev, int64_t n, void* stream);
int nfb_sigmoid_backward(const float* out_dev, const float* g_out_dev, float* g_in_dev, int64_t n, void* stream);
/* Adjoint of nfb_logit_transform in the density direction (NFB_INVERSE): g_in = dy/dx g_out + d log_det/dx g_log_det
 * (g_out or g_log_det may be NULL). */
int nfb_logit_transform_backward(const float* in_dev, const float* g_out_dev, const float* g_log_det_dev, float* g_in_dev,
                                 int64_t batch, int64_t inner, float alpha, void* stream);

/* ---- layer parameter descriptors (device pointers into the caller's parameters) ---- */

/* A residual conditioner: nets/resnet.py:53-104 ResidualNet (mask pointers NULL) or
 * nets/made.py:217-304 MADE with residual blocks (mask pointers = the `mask` buffers).
 * blocks: 2*num_blocks entries, ordered blocks.0.linear_layers.0, blocks.0.linear_layers.1, ... */
typedef struct {
    int32_t in_features, hidden_features, out_features, num_blocks;
    const float* w_initial; const float* b_initial; const float* m_initial;
    const float* const* w_blocks; const float* const* b_blocks; const float* const* m_blocks;
    const float* w_final; const float* b_final; const float* m_final;
} nfb_resnet_desc_t;

/* A residual conditioner called on its own with an optional context (nets/resnet.py:92-104, nets/made.py:296-304):
 * ResidualNet concatenates the context to its input ahead of initial_layer (net.in_features = input + context
 * features), MADE adds context_layer(context) to the initial layer's output (w_context / b_context).  With a context,
 * every residual block ends in the GLU gate h + t * sigmoid(block_context_layer(context)). */
typedef struct {
    nfb_resnet_desc_t net;
    int32_t context_features;                 /* 0: no context (the pointers below are ignored) */
    const float* w_context;                   /* MADE context_layer.weight [hidden, context]; NULL: ResidualNet */
    const float* b_context;
    const float* const* w_block_context;      /* [num_blocks] blocks.<b>.context_layer.weight [hidden, context] */
    const float* const* b_block_context;
} nfb_resnet_ctx_desc_t;
/* Bytes of device scratch nfb_resnet_backward needs for `rows` rows (-1: bad descriptor). */
int64_t nfb_resnet_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* desc, int64_t rows);
/* Gradients of sum g_out . net(x, context) in one call: the activations are recomputed from x / context, then dgrad
 * and wgrad of every Linear run on the tensor core (the MADE masks multiply the weight gradients in the GEMM epilogue,
 * the ReLU masks gate the data gradients), with the GLU adjoint of every context-gated block.
 * x [rows, input features], context [rows, context_features], g_out [rows, out_features].  Outputs, each optional
 * and OVERWRITTEN: g_x, g_context; g_w / g_b: 2 + 2 num_blocks entries in the order of nfb_resnet_desc_t: initial,
 * blocks.0.linear_layers.0, ..., final; g_w_context / g_b_context: 1 + num_blocks entries (MADE context_layer, then
 * each block's context_layer).  The arrays themselves may be NULL. */
int nfb_resnet_backward(const nfb_resnet_ctx_desc_t* desc, const float* x_dev, const float* context_dev,
                        const float* g_out_dev, int64_t rows, void* workspace_dev, int64_t workspace_bytes,
                        float* g_x_dev, float* g_context_dev, float* const* g_w, float* const* g_b,
                        float* const* g_w_context, float* const* g_b_context, void* stream);

/* Bytes of device scratch nfb_maf_inverse_backward needs for `rows` rows (-1: bad descriptor). */
int64_t nfb_maf_inverse_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* desc, int32_t features, int64_t rows);
/* Gradients of sum g_y . y + g_log_det . log_det through the density pass of MaskedAffineAutoregressive
 * (flows/affine/autoregressive.py:26-33,114-128): y solves y = (x - shift) / scale with (u, shift) the interleaved
 * pairs of p = MADE(y, context) [rows, features, 2], scale = sigmoid(u + 2) + 1e-3, log_det = -sum log scale.
 * desc is the MADE (masks set, in_features = features, out_features = 2 features, context through w_context).
 * The MADE's activations are recomputed once at the forward's output y; the cotangent lam of y then follows
 * lam = g_y + MADE_dgrad_y(pbar(lam)) for features - 1 passes (exact: MADE's Jacobian in y is strictly lower
 * triangular), each pass one element kernel and one data-gradient-only MADE adjoint, and a last pass forms
 * g_x = lam / scale and the weight / context gradients of the final pbar.  Equals the gradient of the reference's
 * unrolled D-pass loop.  x, y [rows, features], context [rows, context_features], g_y [rows, features] and g_log_det
 * [rows] (either may be NULL: zero).  Outputs as in nfb_resnet_backward, each optional and OVERWRITTEN: g_x, g_context,
 * g_w / g_b (2 + 2 num_blocks entries: initial, blocks.0.linear_layers.0, ..., final), g_w_context / g_b_context
 * (1 + num_blocks entries: context_layer, then each block's context_layer).  rows = 0: every gradient is zero. */
int nfb_maf_inverse_backward(const nfb_resnet_ctx_desc_t* desc, int32_t features, const float* x_dev, const float* y_dev,
                             const float* context_dev, const float* g_y_dev, const float* g_log_det_dev, int64_t rows,
                             void* workspace_dev, int64_t workspace_bytes, float* g_x_dev, float* g_context_dev,
                             float* const* g_w, float* const* g_b, float* const* g_w_context,
                             float* const* g_b_context, void* stream);

/* Bytes of device scratch nfb_ar_rqs_sampling_backward needs for `rows` rows (-1: bad descriptor or shape). */
int64_t nfb_ar_rqs_sampling_backward_workspace_bytes(const nfb_resnet_ctx_desc_t* desc, int32_t features,
                                                     int32_t num_bins, int32_t num_derivatives, int64_t rows);
/* Gradients of sum g_x . x + g_log_det . log_det through the sampling direction of an autoregressive spline layer
 * (AutoregressiveRationalQuadraticSpline / CircularAutoregressiveRationalQuadraticSpline.forward,
 * flows/affine/autoregressive.py:29-38): x solves x = G(z; MADE(pre(x), context)) with G the inverse spline on the
 * records [rows, features, 2K + nd] of the MADE output and log_det = -sum log f'(x), computed by the reference with D
 * sequential passes.  desc is the MADE (masks set, in_features = features, out_features = features (2K + nd), context
 * through w_context).  The spline: num_bins K, num_derivatives nd = K - 1 with the scalar tail_bound (linear tails;
 * tail_bound_dev and circular_dev NULL), or nd = K / K + 1 with tail_bound_dev [features] and circular_dev [features]
 * as in nfb_rqs_spline_tails (tail_bound unused).  pre is PeriodicFeaturesElementwise given by its tables in the layout
 * of nfb_periodic_features (pf_slot_dev NULL: pre is the identity).
 * The MADE's activations are recomputed once at pre(x); the cotangent lam of x then follows
 * lam = g_x + pre'(x) MADE_dgrad(pbar(lam)) for features - 1 data-gradient-only passes (exact: MADE's Jacobian is
 * strictly lower triangular in its degree order), pbar(lam) the parameter gradient of the inverse-spline adjoint
 * (nfb_rqs_spline(_tails)_inverse_backward), and one last pass forms g_z and the weight / context / periodic-feature
 * gradients.  Equals the gradient of the reference's unrolled D-pass loop.  z, x [rows, features] (the layer's input and
 * output), context [rows, context_features], g_x [rows, features] and g_log_det [rows] (either may be NULL: zero).
 * Outputs, each optional and OVERWRITTEN: g_z, g_context, g_w / g_b / g_w_context / g_b_context in
 * nfb_resnet_backward's slot order, g_pf_weights [n_periodic, 2] and g_pf_bias [n_periodic].  rows = 0: every
 * gradient is zero. */
int nfb_ar_rqs_sampling_backward(const nfb_resnet_ctx_desc_t* desc, int32_t features, int32_t num_bins,
                                 int32_t num_derivatives, float tail_bound, const float* tail_bound_dev,
                                 const int32_t* circular_dev, const int32_t* pf_slot_dev, const float* pf_weights_dev,
                                 const float* pf_scale_dev, const float* pf_bias_dev, int32_t pf_n_periodic,
                                 const float* z_dev, const float* x_dev, const float* context_dev, const float* g_x_dev,
                                 const float* g_log_det_dev, int64_t rows, void* workspace_dev, int64_t workspace_bytes,
                                 float* g_z_dev, float* g_context_dev, float* const* g_w, float* const* g_b,
                                 float* const* g_w_context, float* const* g_b_context, float* g_pf_weights_dev,
                                 float* g_pf_bias_dev, void* stream);

/* flows/neural_spline/wrapper.py:186-244 AutoregressiveRationalQuadraticSpline */
typedef struct {
    int32_t features, num_bins;
    float tail_bound;
    nfb_resnet_desc_t net; /* mprqat.autoregressive_net.* */
} nfb_ar_rqs_desc_t;

/* flows/neural_spline/wrapper.py:14-85 CoupledRationalQuadraticSpline */
typedef struct {
    int32_t features, num_bins, num_identity, num_transform;
    float tail_bound;
    const int64_t* identity_features;  /* prqct.identity_features  (device, int64 as in state_dict) */
    const int64_t* transform_features; /* prqct.transform_features */
    nfb_resnet_desc_t net;             /* prqct.transform_net.* */
    const float* uncond_widths;        /* prqct.unconditional_transform.unnormalized_widths  [n_id,K]   */
    const float* uncond_heights;       /*                               unnormalized_heights [n_id,K]   */
    const float* uncond_derivatives;   /*                               unnormalized_derivatives [n_id,K-1] */
} nfb_coupled_rqs_desc_t;

/* flows/mixing.py:535-563 LULinearPermute */
typedef struct {
    int32_t features;
    const int64_t* permutation;   /* permutation._permutation [features] (device, int64) */
    const float* lower_entries;   /* linear.lower_entries  [n(n-1)/2] */
    const float* upper_entries;   /* linear.upper_entries  [n(n-1)/2] */
    const float* unconstrained_upper_diag; /* [n] */
    const float* bias;            /* linear.bias [n] */
    float eps;                    /* _LULinear eps (1e-3) */
} nfb_lu_desc_t;

/* nets/mlp.py:5-58 MLP (Linear / LeakyReLU stack, last layer linear) */
typedef struct {
    int32_t num_layers;           /* number of Linear layers, <= 6; 0 = net absent */
    int32_t sizes[7];             /* sizes[0]=in ... sizes[num_layers]=out */
    const float* w[6];
    const float* b[6];
    float leaky;
} nfb_mlp_desc_t;

/* nets/mlp.py MLP called on its own: gradients of sum g_out . mlp(x) (activations recomputed, LeakyReLU slope
 * desc->leaky >= 0).  g_x, g_w[l], g_b[l] optional and overwritten. */
int64_t nfb_mlp_backward_workspace_bytes(const nfb_mlp_desc_t* desc, int64_t rows);
int nfb_mlp_backward(const nfb_mlp_desc_t* desc, const float* x_dev, const float* g_out_dev, int64_t rows,
                     void* workspace_dev, int64_t workspace_bytes, float* g_x_dev, float* const* g_w,
                     float* const* g_b, void* stream);

/* flows/affine/coupling.py:174-229 MaskedAffineFlow */
typedef struct { int32_t features; const float* b; nfb_mlp_desc_t s; nfb_mlp_desc_t t; } nfb_masked_affine_desc_t;

/* flows/affine/coupling.py:232-267 AffineCouplingBlock with an MLP param_map */
typedef struct {
    int32_t features;
    int32_t scale;       /* bool */
    int32_t scale_map;   /* 0 exp, 1 sigmoid, 2 sigmoid_inv */
    int32_t split_mode;  /* 0 channel, 1 channel_inv */
    nfb_mlp_desc_t param_map;
} nfb_affine_coupling_desc_t;

/* flows/affine/coupling.py:9-54 AffineConstFlow; flows/normalization.py:7-39 ActNorm after init */
typedef struct { int32_t features; const float* s; const float* t; } nfb_affine_const_desc_t;

/* flows/mixing.py:9-54 Permute: forward z[:, perm], inverse z[:, inv_perm] (host int32 arrays) */
typedef struct { int32_t features; const int32_t* perm; const int32_t* inv_perm; } nfb_permute_desc_t;

/* flows/planar.py Planar: x = z + u_hat h(w.z + b), u_hat = u + (log(1 + exp(w.u)) - 1 - w.u) w / |w|^2.  u, w [features],
 * b [1]; act NFB_PLANAR_TANH or NFB_PLANAR_LEAKY_RELU (negative slope `slope`); features <= 64.  Only the leaky-ReLU
 * layer has a density direction (NFB_INVERSE on a group holding any other planar / radial layer: NFB_ERR_UNSUPPORTED). */
#define NFB_PLANAR_TANH 0
#define NFB_PLANAR_LEAKY_RELU 1
typedef struct { int32_t features; const float* u; const float* w; const float* b; int32_t act; float slope; } nfb_planar_desc_t;

/* flows/radial.py Radial: x = z + h (z - z0), h = beta_hat / (|alpha| + |z - z0|), beta_hat = log(1 + exp(beta)) - |alpha|.
 * beta, alpha [1], z0 [features]; features <= 64; sampling direction only.  Consecutive planar / radial layers run as one
 * launch that forms every layer's constants on the device (a parameter update needs no repack). */
typedef struct { int32_t features; const float* beta; const float* alpha; const float* z0; } nfb_radial_desc_t;

/* ---- flow object: an ordered list of layers + base density, packed for the device ---- */
int nfb_flow_create(nfb_flow_t** out, int32_t features);
int nfb_flow_destroy(nfb_flow_t* f);
int nfb_flow_add_ar_rqs(nfb_flow_t* f, const nfb_ar_rqs_desc_t* d);
int nfb_flow_add_coupled_rqs(nfb_flow_t* f, const nfb_coupled_rqs_desc_t* d);
int nfb_flow_add_lu_linear_permute(nfb_flow_t* f, const nfb_lu_desc_t* d);
/* Affine family (MaskedAffineFlow, AffineCouplingBlock, AffineConstFlow / ActNorm, Permute): any number of features and
 * any net width, nets of at most 6 Linear layers.  A run of consecutive affine layers with at most 16 features and nets at
 * most 128 wide executes as one launch of the one-thread-per-row stack kernel; a run with any layer over either limit
 * executes layer by layer on the wide path (nets on the tensor-core GEMM, element kernels for the coupling).  The choice
 * is made from the shapes at finalize. */
int nfb_flow_add_masked_affine(nfb_flow_t* f, const nfb_masked_affine_desc_t* d);
int nfb_flow_add_affine_coupling(nfb_flow_t* f, const nfb_affine_coupling_desc_t* d);
int nfb_flow_add_affine_const(nfb_flow_t* f, const nfb_affine_const_desc_t* d);
int nfb_flow_add_permute(nfb_flow_t* f, const nfb_permute_desc_t* d);
int nfb_flow_add_planar(nfb_flow_t* f, const nfb_planar_desc_t* d);
int nfb_flow_add_radial(nfb_flow_t* f, const nfb_radial_desc_t* d);
/* q0 = DiagGaussian(features): loc/log_scale [features] (distributions/base.py:71-76) */
int nfb_flow_set_base_diag_gaussian(nfb_flow_t* f, const float* loc_dev, const float* log_scale_dev);
/* q0 = GaussianMixture(n_modes, features): loc / log_scale [n_modes, features], weight_scores [n_modes]
 * (distributions/base.py:573-614).  Either setter replaces any earlier base.  log_prob, forward_kld, their _host forms
 * and nfb_flow_log_prob_backward then use the mixture (nfb_gaussian_mixture_log_prob, one launch after the stack). */
int nfb_flow_set_base_gaussian_mixture(nfb_flow_t* f, int32_t n_modes, const float* loc_dev, const float* log_scale_dev,
                                       const float* weight_scores_dev);
/* pack parameters; `use_tensor_cores`=0 forces the plain-fp32 kernels for every layer (A/B parity) */
int nfb_flow_finalize(nfb_flow_t* f, int32_t use_tensor_cores, void* stream);
/* re-read the descriptor pointers after a parameter update (optimizer step / load_state_dict) */
int nfb_flow_repack(nfb_flow_t* f, void* stream);
int nfb_flow_num_layers(const nfb_flow_t* f);
/* how many CUDA kernels the last pass launched (bench.py reports it as gpu_launches) */
int64_t nfb_flow_last_launch_count(const nfb_flow_t* f);
/* 1 if layer `index` runs on the fused tensor-core kernel in the density direction */
int nfb_flow_layer_is_fused(const nfb_flow_t* f, int32_t index);
/* units of the whole-stack sampling plan (one persistent launch for the sampling direction and for its backward's
   recompute); 0: the sampling direction runs layer by layer */
int nfb_flow_sampling_units(const nfb_flow_t* f);

/* flows/base.py:13-24: apply ONE layer.  log_det_dev [rows]: overwritten (accumulate=0) or += . */
int nfb_flow_layer_apply(nfb_flow_t* f, int32_t index, int32_t direction, const float* z_in_dev,
                         float* z_out_dev, float* log_det_dev, int64_t rows, int32_t accumulate,
                         void* stream);
/* core.py:70-85 inverse_and_log_det (direction=NFB_INVERSE, layers last-to-first) and
 * core.py:40-55 forward_and_log_det (NFB_FORWARD).  z_out may alias z_in. */
int nfb_flow_transform(nfb_flow_t* f, int32_t direction, const float* z_in_dev, float* z_out_dev,
                       float* log_det_dev, int64_t rows, void* stream);
/* core.py:182-197 log_prob: log_q[r] = sum log_det + q0.log_prob(z) */
int nfb_flow_log_prob(nfb_flow_t* f, const float* x_dev, float* log_q_dev, int64_t rows, void* stream);
/* core.py:87-102 forward_kld: *loss_dev = -mean(log_q).  sum_dev (optional, double[2]) receives
 * {sum(log_q), rows}: the per-rank partial a data-parallel caller all-reduces (one collective, 16 bytes),
 * written by the same reduction kernel so the caller adds no device work of its own. */
int nfb_flow_forward_kld(nfb_flow_t* f, const float* x_dev, int64_t rows, float* loss_dev,
                         double* sum_dev, void* stream);

/* ---- training pass (`loss.backward()` of examples/neural_spline_flow.ipynb cell 4; core.py:87-102 under autograd) ----
 * Gradients of sum_r g_logq[r] * log_prob(x_r) w.r.t. every parameter and (optionally) x, for stacks made of
 * autoregressive / coupled RQ-spline blocks (flows/neural_spline/wrapper.py), LULinearPermute (flows/mixing.py:535-563)
 * and a DiagGaussian or GaussianMixture base.  The pass re-runs the density direction keeping each layer group's input, recomputes the
 * conditioner activations per layer (nets/made.py:199-214, nets/resnet.py:37-50), applies the analytic adjoint of the
 * spline (utils/splines.py:100-219) and runs dgrad / wgrad of every Linear on the tensor core.
 * Gradient slots, in list order of the layers:
 *   spline block : weight, bias of initial_layer; of blocks[i].linear_layers[0], [1] ...; of final_layer; then (coupled
 *                  only) unconditional_transform.unnormalized_widths, _heights, _derivatives
 *   LULinearPermute : lower_entries, upper_entries, unconstrained_upper_diag, bias
 *   MaskedAffineFlow : net.<i>.weight, .bias of every Linear of s, then of t (an absent net has none)
 *   AffineConstFlow / ActNorm : s, t       AffineCouplingBlock : param_map's Linears       Permute : none
 *   Planar : u, w, b       Radial : beta, alpha, z_0
 *   base (last slots)     : DiagGaussian loc, log_scale [features] (two slots); GaussianMixture loc, log_scale
 *                           [n_modes * features], weight_scores [n_modes] (three slots)
 * `grad_slots[i]` is a device buffer of nfb_flow_grad_slot_numel(f, i) floats that is OVERWRITTEN, or NULL to skip.
 * nfb_flow_num_grad_slots returns -1 when the flow holds a layer kind without a native backward.  Groups of affine-family
 * layers may sit anywhere in the stack: each runs the same recompute + adjoint walk + fixed-order reduction as
 * nfb_flow_density_backward, with g_logq as its log-det cotangent, in an internal workspace chunked under the same bound.
 * The planar family's slots serve nfb_flow_sampling_backward only: nfb_flow_log_prob_backward rejects its groups
 * (NFB_ERR_UNSUPPORTED).  rows = 0 writes zeros into the slots. */
int nfb_flow_num_grad_slots(const nfb_flow_t* f);
int64_t nfb_flow_grad_slot_numel(const nfb_flow_t* f, int32_t slot);
int nfb_flow_log_prob_backward(nfb_flow_t* f, const float* x_dev, const float* g_logq_dev, int64_t rows,
                               float* log_q_dev /* optional out */, float* gx_dev /* optional out */,
                               float* const* grad_slots, void* stream);

/* ---- sampling-direction backward of an all-affine, all-planar/radial or coupled-spline / LU stack (reverse_kld /
 * reverse_alpha_div of examples/real_nvp.ipynb, planar.ipynb, a coupling NSF) -- gradients of
 * sum_r <g_x[r], x_r> + g_ld[r] log_det_r, with (x, log_det) = nfb_flow_transform(f, NFB_FORWARD, z), w.r.t. z and every
 * parameter, for stacks of MaskedAffineFlow, AffineConstFlow / ActNorm, AffineCouplingBlock and Permute only, of Planar
 * and Radial only, or of CoupledRationalQuadraticSpline (num_bins 8) and LULinearPermute only (any other stack, mixes of
 * these families and autoregressive blocks included: NFB_ERR_UNSUPPORTED).  z is the input that nfb_flow_transform was
 * given.  A planar / radial stack reduces each layer's row terms the same way, then takes the sums through u_hat(u, w),
 * softplus(beta) and |alpha| in one more launch (3 launches per chunk of rows + 1).  The affine call recomputes the
 * stack from z (the forward kernel's own arithmetic), walks the ops in reverse in one kernel, then reduces
 * every Linear's weight and bias gradient in a fixed order (no atomics: two calls give identical bits).  Rows run in
 * chunks, so the workspace (nfb_flow_sampling_backward_workspace_bytes, -1 for an unsupported stack) stays below a fixed
 * bound; the number of launches does not depend on the number of layers.  A stack on the wide path (over 16 features or a
 * net wider than 128, see nfb_flow_add_masked_affine) recomputes each chunk layer by layer and back-propagates each layer
 * with GEMMs: its launches grow linearly with depth, and weight gradients summed by split-K GEMMs are not bitwise
 * reproducible from call to call.
 * A coupled-spline / LU stack recomputes the sampling pass from z keeping every layer's input (the whole-stack
 * persistent launch when the stack takes it, each unit writing its own slice, else layer by layer), then walks the
 * layers last-to-first: an LU layer by two GEMMs (g_y = W^-T g_t; W's gradient -sum_rows g_y t^T) and the LU factor
 * gradient, a coupled block by the inverse-spline adjoint of its transform columns, its conditioner's recompute and
 * adjoint at the identity columns' output, and the inverse adjoint of the unconditional CDF.  It runs in the flow's
 * own training buffers (those of nfb_flow_log_prob_backward): its workspace size is 0; its launches grow linearly with
 * depth, and weight gradients summed by split-K GEMMs or atomics are not bitwise reproducible from call to call.
 * g_x / g_ld may be NULL (zero cotangent); g_z and individual slots may be NULL (not wanted).  grad_slots holds the
 * layers' slots in nfb_flow_grad_slot_numel order (a base's slots, if any, are not read); rows = 0 writes zeros. */
int64_t nfb_flow_sampling_backward_workspace_bytes(const nfb_flow_t* f, int64_t rows);
int nfb_flow_sampling_backward(nfb_flow_t* f, const float* z, const float* g_x, const float* g_ld, int64_t rows,
                               void* ws, int64_t ws_bytes, float* g_z, float* const* grad_slots, void* stream);

/* ---- density-direction backward of an all-affine stack (forward_kld / log_prob of examples/real_nvp_colab.ipynb, a
 * stand-alone ActNorm between Residual blocks) -- gradients of sum_r <g_z[r], z_r> + g_ld[r] log_det_r, with
 * (z, log_det) = nfb_flow_transform(f, NFB_INVERSE, x), w.r.t. x and every parameter, for stacks of MaskedAffineFlow,
 * AffineConstFlow / ActNorm, AffineCouplingBlock and Permute only (any other stack, Planar / Radial included:
 * NFB_ERR_UNSUPPORTED).  x is the input that nfb_flow_transform was given.  One kernel recomputes the stack from x
 * taking the ops last-to-first, then walks them first-to-last; the weight reduction, the row chunking, the workspace
 * bound and the launch count (and the wide path) are those of nfb_flow_sampling_backward.  g_z / g_ld may be NULL (zero cotangent); g_x and
 * individual slots may be NULL (not wanted); grad_slots is in nfb_flow_grad_slot_numel order (a base's slots, if any,
 * are not read); rows = 0 writes zeros. */
int64_t nfb_flow_density_backward_workspace_bytes(const nfb_flow_t* f, int64_t rows);
int nfb_flow_density_backward(nfb_flow_t* f, const float* x, const float* g_z, const float* g_ld, int64_t rows,
                              void* ws, int64_t ws_bytes, float* g_x, float* const* grad_slots, void* stream);

/* ---- stochastic layers and HAIS (flows/stochastic.py HamiltonianMonteCarlo / MetropolisHastings, sampling/hais.py) ----
 * A native density is log p(z) = sum_i coef_i log p_i(z) over n_terms Gaussian mixtures p_i (loc / log_scale
 * [n_modes, dim], weight_scores [n_modes]); a DiagGaussian is the one-mode mixture with weight score 0, a
 * LinearInterpolation(d1, d2, alpha) the two terms (alpha, 1 - alpha).  The coefficients are per transition (coef
 * [transitions, n_terms]) so that one call runs a whole annealing chain.  One thread per row; dim <= NFB_STOCHASTIC_MAX_DIM
 * (a larger dim: NFB_ERR_UNSUPPORTED).  Every random number is an input, drawn by the caller:
 * noise [transitions, rows, dim] standard normals, uniforms [transitions, rows] on [0, 1). */
#define NFB_DENSITY_MAX_TERMS 4
#define NFB_STOCHASTIC_MAX_DIM 64
typedef struct {
    int32_t n_modes;
    const float* loc;
    const float* log_scale;
    const float* weight_scores;
} nfb_density_term_t;
typedef struct {
    int32_t n_terms;
    int32_t dim;
    nfb_density_term_t term[NFB_DENSITY_MAX_TERMS];
} nfb_density_t;

/* `transitions` HMC transitions of HamiltonianMonteCarlo.forward (flows/stochastic.py:54-96), transition t with its own
 * log_step_size / log_mass [transitions, dim] and coefficients: momentum p = noise exp(log_mass / 2), `leapfrog` leapfrog
 * steps with grad log p clamped to +-max_abs_grad unless max_abs_grad is 0, accept when uniform < exp(log p(z') -
 * log p(z) - K(p') + K(p)) (a NaN exponent rejects, an overflowing one accepts).  z_out [rows, dim] is the last state;
 * log_w [rows] (may be NULL) is incremented by log p_t(z_t) - log p_t(z_{t+1}) for every t (0 on a rejected row);
 * accept [transitions, rows] (may be NULL) receives each decision.  z_out may alias z.  One launch. */
int nfb_hmc_chain(const nfb_density_t* density, int64_t rows, int32_t transitions, int32_t leapfrog, float max_abs_grad,
                  const float* coef, const float* log_step_size, const float* log_mass, const float* noise,
                  const float* uniforms, const float* z, float* z_out, float* log_w, uint8_t* accept, void* stream);
/* Gradients of one HMC transition (transitions = 1) with respect to log_step_size and log_mass [dim] (overwritten), given
 * the cotangent g_z_out [rows, dim] of z_out and the accept decisions of nfb_hmc_chain: grad log p is a constant and the
 * accept mask has none, so only accepted rows contribute, through the leapfrog arithmetic and the momentum draw.  One
 * kernel recomputes the leapfrog per row into the workspace ([dim, rows] floats,
 * nfb_hmc_backward_workspace_bytes), a second sums each feature in a fixed order: no atomics, identical bits on every
 * call.  g_log_mass is exactly -g_log_step_size / 2 (dz_out/dlog_mass = -dz_out/dlog_step_size / 2).  rows = 0 writes
 * zeros. */
int64_t nfb_hmc_backward_workspace_bytes(int64_t rows, int32_t dim);
int nfb_hmc_backward(const nfb_density_t* density, int64_t rows, int32_t leapfrog, float max_abs_grad, const float* coef,
                     const float* log_step_size, const float* log_mass, const float* noise, const float* z,
                     const uint8_t* accept, const float* g_z_out, void* ws, int64_t ws_bytes, float* g_log_step_size,
                     float* g_log_mass, void* stream);
/* `steps` steps of MetropolisHastings.forward (flows/stochastic.py:23-45) with DiagGaussianProposal(scale [dim]) on the
 * density with coefficients coef [n_terms]:
 * z' = noise scale + z, accept when uniform <= min(exp(log p(z') - log p(z)), 1).  z_out [rows, dim]; log_det [rows]
 * (overwritten) accumulates log p(z) - log p(z') over the accepted steps; moved [rows] (may be NULL) is 1 where any step
 * was accepted.  z_out may alias z.  One launch. */
int nfb_mh_chain(const nfb_density_t* density, int64_t rows, int32_t steps, const float* coef, const float* scale,
                 const float* noise,
                 const float* uniforms, const float* z, float* z_out, float* log_det, uint8_t* moved, void* stream);

/* ---- host-buffer entry points (what a non-CUDA caller binds; copies are inside) ---- */
int nfb_flow_log_prob_host(nfb_flow_t* f, const float* x_host, float* log_q_host, int64_t rows);
int nfb_flow_forward_kld_host(nfb_flow_t* f, const float* x_host, int64_t rows, float* loss_host);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* NFB200_H */
