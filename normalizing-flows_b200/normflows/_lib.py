"""ctypes binding of libnfb200.so (C ABI: include/nfb200.h).

This is the ONLY compute path of the package: if the library cannot be loaded, or there is no CUDA
device, calls fail loudly -- there is no eager/CPU fallback (see DESIGN.md)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# NFB200_LIB: another build of the SAME library (A/B measurements of kernel variants on one GPU box); default: in-tree
LIB_PATH = os.environ.get("NFB200_LIB") or os.path.join(os.path.dirname(_HERE), "libnfb200.so")

NFB_INVERSE, NFB_FORWARD = 0, 1
NFB_PLANAR_TANH, NFB_PLANAR_LEAKY_RELU = 0, 1   # nfb_planar_desc_t.act
NFB_VAE_LOGVAR, NFB_VAE_SCALE = 0, 1   # scale_kind of the nfb_vae_* calls
_FP = C.POINTER(C.c_float)
_I64P = C.POINTER(C.c_int64)
_I32P = C.POINTER(C.c_int32)


class ResnetDesc(C.Structure):
    _fields_ = [("in_features", C.c_int32), ("hidden_features", C.c_int32),
                ("out_features", C.c_int32), ("num_blocks", C.c_int32),
                ("w_initial", C.c_void_p), ("b_initial", C.c_void_p), ("m_initial", C.c_void_p),
                ("w_blocks", C.POINTER(C.c_void_p)), ("b_blocks", C.POINTER(C.c_void_p)),
                ("m_blocks", C.POINTER(C.c_void_p)),
                ("w_final", C.c_void_p), ("b_final", C.c_void_p), ("m_final", C.c_void_p)]


class ResnetCtxDesc(C.Structure):
    _fields_ = [("net", ResnetDesc), ("context_features", C.c_int32),
                ("w_context", C.c_void_p), ("b_context", C.c_void_p),
                ("w_block_context", C.POINTER(C.c_void_p)), ("b_block_context", C.POINTER(C.c_void_p))]


class ArRqsDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("num_bins", C.c_int32), ("tail_bound", C.c_float),
                ("net", ResnetDesc)]


class CoupledRqsDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("num_bins", C.c_int32), ("num_identity", C.c_int32),
                ("num_transform", C.c_int32), ("tail_bound", C.c_float),
                ("identity_features", C.c_void_p), ("transform_features", C.c_void_p),
                ("net", ResnetDesc),
                ("uncond_widths", C.c_void_p), ("uncond_heights", C.c_void_p),
                ("uncond_derivatives", C.c_void_p)]


class LuDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("permutation", C.c_void_p), ("lower_entries", C.c_void_p),
                ("upper_entries", C.c_void_p), ("unconstrained_upper_diag", C.c_void_p),
                ("bias", C.c_void_p), ("eps", C.c_float)]


class MlpDesc(C.Structure):
    _fields_ = [("num_layers", C.c_int32), ("sizes", C.c_int32 * 7), ("w", C.c_void_p * 6),
                ("b", C.c_void_p * 6), ("leaky", C.c_float)]


class MaskedAffineDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("b", C.c_void_p), ("s", MlpDesc), ("t", MlpDesc)]


class AffineCouplingDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("scale", C.c_int32), ("scale_map", C.c_int32),
                ("split_mode", C.c_int32), ("param_map", MlpDesc)]


class AffineConstDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("s", C.c_void_p), ("t", C.c_void_p)]


class PermuteDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("perm", _I32P), ("inv_perm", _I32P)]


class PlanarDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("u", C.c_void_p), ("w", C.c_void_p), ("b", C.c_void_p), ("act", C.c_int32),
                ("slope", C.c_float)]


class RadialDesc(C.Structure):
    _fields_ = [("features", C.c_int32), ("beta", C.c_void_p), ("alpha", C.c_void_p), ("z0", C.c_void_p)]


class GemmDesc(C.Structure):
    _fields_ = [("A", C.c_void_p), ("B", C.c_void_p), ("C", C.c_void_p),
                ("lda", C.c_int64), ("ldb", C.c_int64), ("ldc", C.c_int64),
                ("M", C.c_int64), ("N", C.c_int64), ("K", C.c_int64),
                ("a_mn", C.c_int32), ("b_mn", C.c_int32), ("a_relu", C.c_int32), ("b_relu", C.c_int32),
                ("relu_out", C.c_int32), ("accumulate", C.c_int32),
                ("bias", C.c_void_p), ("mask", C.c_void_p), ("mulm", C.c_void_p), ("ldmask", C.c_int64),
                ("resid", C.c_void_p), ("ldres", C.c_int64)]


LIPSCHITZ_MLP_MAX_LAYERS = 8
SWISH_DUAL_PARTIALS = 1024


class LipschitzMlpDesc(C.Structure):
    _fields_ = [("num_layers", C.c_int32), ("widths", C.c_int32 * (LIPSCHITZ_MLP_MAX_LAYERS + 1)),
                ("w", C.c_void_p * LIPSCHITZ_MLP_MAX_LAYERS), ("bias", C.c_void_p * LIPSCHITZ_MLP_MAX_LAYERS),
                ("b", C.c_float * LIPSCHITZ_MLP_MAX_LAYERS)]


DENSITY_MAX_TERMS = 4
STOCHASTIC_MAX_DIM = 64


class DensityTerm(C.Structure):
    _fields_ = [("n_modes", C.c_int32), ("loc", C.c_void_p), ("log_scale", C.c_void_p), ("weight_scores", C.c_void_p)]


class DensityDesc(C.Structure):
    _fields_ = [("n_terms", C.c_int32), ("dim", C.c_int32), ("term", DensityTerm * DENSITY_MAX_TERMS)]


# every symbol include/nfb200.h declares: (restype, argtypes)
_VP, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float
SYMBOLS = {
    "nfb_abi_version": (C.c_int, []),
    "nfb_last_error": (C.c_char_p, []),
    "nfb_device_info": (C.c_int, [_I32P, _I32P, _I32P]),
    "nfb_rqs_spline": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I32, _I32, _F, _F, _I32, _I32, _VP]),
    "nfb_rqs_spline_tails": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _VP, _VP, _F, _I32, _I32, _VP]),
    "nfb_periodic_features": (C.c_int, [_VP, _VP, _I64, _I32, _VP, _VP, _VP, _VP, _VP]),
    "nfb_rqs_spline_backward": (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _F, _F, _VP]),
    "nfb_rqs_spline_tails_backward": (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _VP, _VP, _F,
                                                _VP]),
    "nfb_periodic_features_backward": (C.c_int, [_VP, _VP, _I64, _I32, _VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP]),
    "nfb_glu_residual_backward": (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, _VP, _VP]),
    "nfb_resnet_backward_workspace_bytes": (_I64, [C.POINTER(ResnetCtxDesc), _I64]),
    "nfb_resnet_backward": (C.c_int, [C.POINTER(ResnetCtxDesc), _VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP,
                                      C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), _VP]),
    "nfb_maf_inverse_backward_workspace_bytes": (_I64, [C.POINTER(ResnetCtxDesc), _I32, _I64]),
    "nfb_maf_inverse_backward": (C.c_int, [C.POINTER(ResnetCtxDesc), _I32, _VP, _VP, _VP, _VP, _VP, _I64, _VP, _I64, _VP,
                                           _VP, C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), _VP]),
    "nfb_rqs_spline_inverse_backward": (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _F, _F, _VP]),
    "nfb_rqs_spline_tails_inverse_backward": (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _VP,
                                                        _VP, _F, _VP]),
    "nfb_ar_rqs_sampling_backward_workspace_bytes": (_I64, [C.POINTER(ResnetCtxDesc), _I32, _I32, _I32, _I64]),
    "nfb_ar_rqs_sampling_backward": (C.c_int, [C.POINTER(ResnetCtxDesc), _I32, _I32, _I32, _F, _VP, _VP, _VP, _VP, _VP,
                                               _VP, _I32, _VP, _VP, _VP, _VP, _VP, _I64, _VP, _I64, _VP, _VP,
                                               C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), C.POINTER(_VP), _VP, _VP,
                                               _VP]),
    "nfb_mlp_backward_workspace_bytes": (_I64, [C.POINTER(MlpDesc), _I64]),
    "nfb_mlp_backward": (C.c_int, [C.POINTER(MlpDesc), _VP, _VP, _I64, _VP, _I64, _VP, C.POINTER(_VP), C.POINTER(_VP),
                                   _VP]),
    "nfb_diag_gaussian_log_prob": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I32, _I32, _VP]),
    "nfb_swish": (C.c_int, [_VP, _F, _I64, _VP, _VP, _VP]),
    "nfb_mul_rows": (C.c_int, [_VP, _VP, _I64, _I32, _VP, _VP]),
    "nfb_logabsdet_i_plus_j_2x2": (C.c_int, [_VP, _I64, _VP, _VP]),
    "nfb_glu_residual": (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP]),
    "nfb_rowdot": (C.c_int, [_VP, _VP, _I64, _I32, _F, _I32, _VP, _VP]),
    "nfb_lipschitz_mlp_dual_backward_workspace_bytes": (_I64, [C.POINTER(LipschitzMlpDesc), _I32, _I64]),
    "nfb_lipschitz_mlp_dual_backward": (C.c_int, [C.POINTER(LipschitzMlpDesc), _VP, _VP, _I32, _VP, _VP, _I64, _VP, _I64,
                                                  _VP, C.POINTER(_VP), C.POINTER(_VP), _VP, _VP]),
    "nfb_swish_dual": (C.c_int, [_VP, _VP, _F, _I64, _I32, _I32, _VP, _VP]),
    "nfb_swish_dual_adjoint": (C.c_int, [_VP, _VP, _F, _I64, _I32, _I32, _VP, _VP, _VP, _VP, _VP, _VP]),
    "nfb_logabsdet_i_plus_j_2x2_backward": (C.c_int, [_VP, _VP, _I64, _VP, _VP]),
    "nfb_maf_affine": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _VP]),
    "nfb_logit_transform": (C.c_int, [_VP, _VP, _VP, _I64, _I64, _F, _I32, _I32, _VP]),
    "nfb_gemm_f32": (C.c_int, [C.POINTER(GemmDesc), _VP]),
    "nfb_conv2d": (C.c_int, [_VP, _I32, _I32, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _I32, _F, _VP]),
    "nfb_glow_conditioner": (C.c_int, [_VP, _I32, _I32, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32,
                                       _F, _VP]),
    "nfb_glow_conditioner_packed_bytes": (C.c_int64, [_I32, _I32, _I32]),
    "nfb_glow_conditioner_pack": (C.c_int, [_VP, _VP, _VP, _I32, _I32, _I32, _VP, _VP]),
    "nfb_glow_conditioner_packed": (C.c_int, [_VP, _I32, _I32, _I32, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _F, _VP]),
    "nfb_affine_coupling_image_taps": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "nfb_affine_coupling_image_taps_supported": (C.c_int32, [_I32, _I32, _I32, _I32]),
    "nfb_glow_block": (C.c_int, [_VP] * 12 + [_I64, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _F, _I32, _VP]),
    "nfb_tap_shift_add": (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _VP]),
    "nfb_glow_fold_actnorm_conv1x1": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP]),
    "nfb_glow_fold_conv1x1_actnorm_forward": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP]),
    "nfb_affine_coupling_image": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "nfb_squeeze": (C.c_int, [_VP, _VP, _I64, _I32, _I32, _I32, _I32, _VP]),
    "nfb_copy_channels": (C.c_int, [_VP, _VP, _I64, _I32, _I32, _I32, _I32, _VP]),
    "nfb_paste_channels": (C.c_int, [_VP, _VP, _I64, _I32, _I32, _I32, _I32, _VP]),
    "nfb_class_cond_diag_gaussian_log_prob": (C.c_int, [_VP, _VP, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _VP]),
    "nfb_conv2d_wgrad": (C.c_int, [_VP, _I32, _I32, _VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _I32, _I32, _VP]),
    "nfb_conv2d_dgrad": (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I32, _I32, _I32, _I32, _VP, _F, _I32, _VP]),
    "nfb_affine_coupling_image_backward": (C.c_int, [_VP] * 6 + [_I64, _I32, _I32, _I32, _I32, _I32, _VP]),
    "nfb_gaussian_table_log_prob_backward": (C.c_int, [_VP] * 8 + [_I64, _I32, _I32, _I32, _VP]),
    "nfb_logit_transform_backward": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _I64, _F, _VP]),
    "nfb_gaussian_mixture_log_prob": (C.c_int, [_VP] * 5 + [_I64, _I32, _I32, _I32, _VP]),
    "nfb_gaussian_mixture_log_prob_backward_workspace_bytes": (_I64, [_I64, _I32, _I32]),
    "nfb_gaussian_mixture_log_prob_backward": (C.c_int, [_VP] * 5 + [_I64, _I32, _I32, _VP, _I64] + [_VP] * 5),
    "nfb_vae_reparam_sample": (C.c_int, [_VP, _VP, _I64, _I32, _VP, _I64, _I32, _I32, _VP, _VP, _VP]),
    "nfb_vae_reparam_sample_backward": (C.c_int, [_VP, _VP, _I64, _I32, _VP, _VP, _VP, _I64, _I32, _I32, _VP, _VP, _VP]),
    "nfb_vae_gaussian_log_prob": (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I64, _I32, _I64, _I64, _F, _VP, _VP]),
    "nfb_vae_gaussian_log_prob_backward": (C.c_int, [_VP, _VP, _VP, _I64, _I32, _VP, _I64, _I32, _I64, _I64, _VP, _VP,
                                                     _VP, _VP]),
    "nfb_bernoulli_log_prob": (C.c_int, [_VP, _VP, _I64, _I32, _I64, _VP, _VP]),
    "nfb_bernoulli_log_prob_backward": (C.c_int, [_VP, _VP, _VP, _I64, _I32, _I64, _VP, _VP, _VP]),
    "nfb_sigmoid": (C.c_int, [_VP, _VP, _I64, _VP]),
    "nfb_sigmoid_backward": (C.c_int, [_VP, _VP, _VP, _I64, _VP]),
    "nfb_hmc_chain": (C.c_int, [C.POINTER(DensityDesc), _I64, _I32, _I32, _F] + [_VP] * 10),
    "nfb_hmc_backward_workspace_bytes": (_I64, [_I64, _I32]),
    "nfb_hmc_backward": (C.c_int, [C.POINTER(DensityDesc), _I64, _I32, _F] + [_VP] * 7 + [_VP, _I64, _VP, _VP, _VP]),
    "nfb_mh_chain": (C.c_int, [C.POINTER(DensityDesc), _I64, _I32] + [_VP] * 9),
    "nfb_flow_create": (C.c_int, [C.POINTER(_VP), _I32]),
    "nfb_flow_destroy": (C.c_int, [_VP]),
    "nfb_flow_add_ar_rqs": (C.c_int, [_VP, C.POINTER(ArRqsDesc)]),
    "nfb_flow_add_coupled_rqs": (C.c_int, [_VP, C.POINTER(CoupledRqsDesc)]),
    "nfb_flow_add_lu_linear_permute": (C.c_int, [_VP, C.POINTER(LuDesc)]),
    "nfb_flow_add_masked_affine": (C.c_int, [_VP, C.POINTER(MaskedAffineDesc)]),
    "nfb_flow_add_affine_coupling": (C.c_int, [_VP, C.POINTER(AffineCouplingDesc)]),
    "nfb_flow_add_affine_const": (C.c_int, [_VP, C.POINTER(AffineConstDesc)]),
    "nfb_flow_add_permute": (C.c_int, [_VP, C.POINTER(PermuteDesc)]),
    "nfb_flow_add_planar": (C.c_int, [_VP, C.POINTER(PlanarDesc)]),
    "nfb_flow_add_radial": (C.c_int, [_VP, C.POINTER(RadialDesc)]),
    "nfb_flow_set_base_diag_gaussian": (C.c_int, [_VP, _VP, _VP]),
    "nfb_flow_set_base_gaussian_mixture": (C.c_int, [_VP, _I32, _VP, _VP, _VP]),
    "nfb_flow_finalize": (C.c_int, [_VP, _I32, _VP]),
    "nfb_flow_repack": (C.c_int, [_VP, _VP]),
    "nfb_flow_num_layers": (C.c_int, [_VP]),
    "nfb_flow_last_launch_count": (_I64, [_VP]),
    "nfb_flow_layer_is_fused": (C.c_int, [_VP, _I32]),
    "nfb_flow_sampling_units": (C.c_int, [_VP]),
    "nfb_flow_layer_apply": (C.c_int, [_VP, _I32, _I32, _VP, _VP, _VP, _I64, _I32, _VP]),
    "nfb_flow_transform": (C.c_int, [_VP, _I32, _VP, _VP, _VP, _I64, _VP]),
    "nfb_flow_log_prob": (C.c_int, [_VP, _VP, _VP, _I64, _VP]),
    "nfb_flow_forward_kld": (C.c_int, [_VP, _VP, _I64, _VP, _VP, _VP]),
    "nfb_flow_num_grad_slots": (C.c_int, [_VP]),
    "nfb_flow_grad_slot_numel": (_I64, [_VP, _I32]),
    "nfb_flow_log_prob_backward": (C.c_int, [_VP, _VP, _VP, _I64, _VP, _VP, C.POINTER(_VP), _VP]),
    "nfb_flow_sampling_backward_workspace_bytes": (_I64, [_VP, _I64]),
    "nfb_flow_sampling_backward": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _VP, _I64, _VP, C.POINTER(_VP), _VP]),
    "nfb_flow_density_backward_workspace_bytes": (_I64, [_VP, _I64]),
    "nfb_flow_density_backward": (C.c_int, [_VP, _VP, _VP, _VP, _I64, _VP, _I64, _VP, C.POINTER(_VP), _VP]),
    "nfb_flow_log_prob_host": (C.c_int, [_VP, _VP, _VP, _I64]),
    "nfb_flow_forward_kld_host": (C.c_int, [_VP, _VP, _I64, _VP]),
}

_lib = None


class NativeError(RuntimeError):
    pass


def lib():
    """Load libnfb200.so (built in-tree by `__graft_entry__.build()` / csrc/Makefile)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeError(
                f"{LIB_PATH} is missing: build it with `make -C normalizing-flows_b200/csrc` "
                "(or __graft_entry__.build()).  normflows-b200 has no eager/CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)  # AttributeError here = header/library mismatch
            fn.restype, fn.argtypes = res, args
        _lib = handle
    return _lib


_ERRORS = {2: ValueError, 3: NotImplementedError}


def check(rc):
    if rc != 0:
        msg = lib().nfb_last_error().decode("utf-8", "replace")
        raise _ERRORS.get(rc, NativeError)(msg)


def ptr(t):
    """Device pointer of a contiguous CUDA tensor (or None)."""
    return None if t is None else C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
