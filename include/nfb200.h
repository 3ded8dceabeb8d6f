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
/* out[r] (+)= c * sum_j a[r, j] b[r, j]  (one Hutchinson trace term v^T J^k eps per sample, residual.py:355-366) */
int nfb_rowdot(const float* a_dev, const float* b_dev, int64_t rows, int32_t d, float c, int32_t accumulate,
               float* out_dev, void* stream);

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

/* ---- flow object: an ordered list of layers + base density, packed for the device ---- */
int nfb_flow_create(nfb_flow_t** out, int32_t features);
int nfb_flow_destroy(nfb_flow_t* f);
int nfb_flow_add_ar_rqs(nfb_flow_t* f, const nfb_ar_rqs_desc_t* d);
int nfb_flow_add_coupled_rqs(nfb_flow_t* f, const nfb_coupled_rqs_desc_t* d);
int nfb_flow_add_lu_linear_permute(nfb_flow_t* f, const nfb_lu_desc_t* d);
int nfb_flow_add_masked_affine(nfb_flow_t* f, const nfb_masked_affine_desc_t* d);
int nfb_flow_add_affine_coupling(nfb_flow_t* f, const nfb_affine_coupling_desc_t* d);
int nfb_flow_add_affine_const(nfb_flow_t* f, const nfb_affine_const_desc_t* d);
int nfb_flow_add_permute(nfb_flow_t* f, const nfb_permute_desc_t* d);
/* q0 = DiagGaussian(features): loc/log_scale [features] (distributions/base.py:71-76) */
int nfb_flow_set_base_diag_gaussian(nfb_flow_t* f, const float* loc_dev, const float* log_scale_dev);
/* pack parameters; `use_tensor_cores`=0 forces the plain-fp32 kernels for every layer (A/B parity) */
int nfb_flow_finalize(nfb_flow_t* f, int32_t use_tensor_cores, void* stream);
/* re-read the descriptor pointers after a parameter update (optimizer step / load_state_dict) */
int nfb_flow_repack(nfb_flow_t* f, void* stream);
int nfb_flow_num_layers(const nfb_flow_t* f);
/* how many CUDA kernels the last pass launched (bench.py reports it as gpu_launches) */
int64_t nfb_flow_last_launch_count(const nfb_flow_t* f);
/* 1 if layer `index` runs on the fused tensor-core kernel in the density direction */
int nfb_flow_layer_is_fused(const nfb_flow_t* f, int32_t index);

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
 * and a DiagGaussian base.  The pass re-runs the density direction keeping each layer group's input, recomputes the
 * conditioner activations per layer (nets/made.py:199-214, nets/resnet.py:37-50), applies the analytic adjoint of the
 * spline (utils/splines.py:100-219) and runs dgrad / wgrad of every Linear on the tensor core.
 * Gradient slots, in list order of the layers:
 *   spline block : weight, bias of initial_layer; of blocks[i].linear_layers[0], [1] ...; of final_layer; then (coupled
 *                  only) unconditional_transform.unnormalized_widths, _heights, _derivatives
 *   LULinearPermute : lower_entries, upper_entries, unconstrained_upper_diag, bias
 *   base (last two slots) : loc, log_scale
 * `grad_slots[i]` is a device buffer of nfb_flow_grad_slot_numel(f, i) floats that is OVERWRITTEN, or NULL to skip.
 * nfb_flow_num_grad_slots returns -1 when the flow holds a layer kind without a native backward. */
int nfb_flow_num_grad_slots(const nfb_flow_t* f);
int64_t nfb_flow_grad_slot_numel(const nfb_flow_t* f, int32_t slot);
int nfb_flow_log_prob_backward(nfb_flow_t* f, const float* x_dev, const float* g_logq_dev, int64_t rows,
                               float* log_q_dev /* optional out */, float* gx_dev /* optional out */,
                               float* const* grad_slots, void* stream);

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
