"""Neural spline flow layers (reference: normflows/flows/neural_spline/wrapper.py:14-85,186-244,
coupling.py:16-362, autoregressive.py:17-134, flows/affine/autoregressive.py:10-47).

Module trees mirror the reference so `state_dict()` keys match:
  AutoregressiveRationalQuadraticSpline.mprqat.autoregressive_net.{initial_layer,blocks,final_layer}
  CoupledRationalQuadraticSpline.prqct.{identity_features,transform_features,transform_net,
                                        unconditional_transform.unnormalized_*}
NOTE the wrappers swap directions (wrapper.py:79-85,238-244): `inverse()` is the density direction
(one conditioner pass), `forward()` is sampling (D passes for the autoregressive layer).  The stand-alone layers (the
context-conditioned and circular ones) are differentiable in both directions (_standalone.ModuleFn / SamplingFn)."""
import ctypes as C

import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .._image_autograd import wants_grad
from .._native import resnet_desc
from ..nets.made import MADE
from ..nets.resnet import ResidualNet
from .base import Flow, NativeFlow

_BOUNDARY = float(np.log(np.exp(1 - 1e-3) - 1))  # utils/splines.py:36 with min_derivative 1e-3


def _check_bins(num_bins):
    if 1e-3 * num_bins > 1.0:
        raise ValueError("Minimal bin width too large for the number of bins")


class _ARTransform(nn.Module):
    """Holds `autoregressive_net` under the reference's attribute name (`mprqat`)."""

    def __init__(self, features, hidden_features, num_bins, num_blocks, permute_mask, activation,
                 dropout_probability, init_identity, context_features=None, output_multiplier=None,
                 preprocessing=None):
        super().__init__()
        self.autoregressive_net = MADE(features, hidden_features, context_features, num_blocks,
                                       output_multiplier=output_multiplier or 3 * num_bins - 1, use_residual_blocks=True,
                                       random_mask=False, permute_mask=permute_mask, activation=activation,
                                       dropout_probability=dropout_probability, use_batch_norm=False,
                                       preprocessing=preprocessing)
        if init_identity:
            nn.init.constant_(self.autoregressive_net.final_layer.weight, 0.0)
            nn.init.constant_(self.autoregressive_net.final_layer.bias, _BOUNDARY)


class AutoregressiveRationalQuadraticSpline(NativeFlow):
    def __init__(self, num_input_channels, num_blocks, num_hidden_channels, num_context_channels=None,
                 num_bins=8, tail_bound=3, activation=nn.ReLU, dropout_probability=0.0,
                 permute_mask=False, init_identity=True):
        super().__init__()
        if torch.is_tensor(tail_bound):
            raise NotImplementedError("per-feature tail bounds are not on the CUDA path")
        _check_bins(num_bins)
        self.features, self.num_bins, self.tail_bound = num_input_channels, num_bins, float(tail_bound)
        self.num_context_channels = num_context_channels
        self.mprqat = _ARTransform(num_input_channels, num_hidden_channels, num_bins, num_blocks,
                                   permute_mask, activation(), dropout_probability, init_identity,
                                   context_features=num_context_channels)

    # Context-conditioned layer (ConditionalNormalizingFlow, core.py:216-366): the conditioner takes the context through
    # the MADE's context layers + GLU gates, so it runs as stand-alone tensor-core GEMMs (nets.MADE.forward) and the
    # spline as the stand-alone HBM-bound kernel (csrc/nfb_kernels.cu rqs_rows_kernel) instead of the fused block.
    # The density direction trains through _standalone.ModuleFn (_value / _adjoint below), the sampling direction
    # through _standalone.SamplingFn (_sampling_value / _sampling_adjoint: the fixed-point adjoint of the D-pass loop).
    def _conditional(self, z, context, sampling):
        from .._standalone import apply_module, apply_sampling
        if not sampling:  # wrapper.inverse -> Autoregressive.forward: one pass (affine/autoregressive.py:24-27)
            return apply_module(self, z, context)
        return apply_sampling(self, z, context)

    def _sampling_value(self, z, context, keep):
        from .._native import rqs_spline
        net = self.mprqat.autoregressive_net
        out, ld = torch.zeros_like(z), None  # D passes (:29-38)
        for _ in range(self.features):
            out, ld = rqs_spline(z, net._value(out, context, None), self.num_bins, self.tail_bound, 1.0, True)
        return out, ld

    def _sampling_adjoint(self, z, x, context, keep, g_x, g_ld, need_z, need_ctx):
        from .._standalone import ar_rqs_sampling_backward
        return ar_rqs_sampling_backward(self.mprqat.autoregressive_net, self.features, self.num_bins, self.num_bins - 1,
                                        self.tail_bound, None, None, z, x, context, g_x, g_ld, need_z, need_ctx)

    def _sampling_differentiable(self, context=None):
        """The stand-alone (context) path is differentiable in the sampling direction; the fused path is not."""
        return self.num_context_channels is not None or context is not None

    def _value(self, z, context, keep):
        from .._native import rqs_spline
        params = self.mprqat.autoregressive_net._value(z, context, None)
        if keep is not None:
            keep["params"] = params
        return rqs_spline(z, params, self.num_bins, self.tail_bound, 1.0, False)

    def _adjoint(self, z, context, keep, grads, need_x, need_ctx):
        from .._standalone import conditioner_backward, spline_backward
        gz, g_params = spline_backward(z, keep["params"], False, self.num_bins, grads[0], grads[1], 1.0,
                                       tail_bound=self.tail_bound)
        g_net, g_ctx, gmap = conditioner_backward(self.mprqat.autoregressive_net, True, z, context, g_params,
                                                  need_ctx=need_ctx)
        return gz + g_net, g_ctx, gmap

    def forward(self, z, context=None):
        if self.num_context_channels is not None or context is not None:
            return self._conditional(z, context, True)
        return super().forward(z)

    def inverse(self, z, context=None):
        if self.num_context_channels is not None or context is not None:
            return self._conditional(z, context, False)
        return super().inverse(z)

    def _native_tensors(self):
        net = self.mprqat.autoregressive_net
        return list(net.parameters()) + [b for n, b in net.named_buffers() if n.endswith("mask")]

    def _native_add(self, handle, features):
        if features != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, features))
        d = L.ArRqsDesc()
        d.features, d.num_bins, d.tail_bound = self.features, self.num_bins, self.tail_bound
        d.net, keep = resnet_desc(self.mprqat.autoregressive_net, masked=True)
        L.check(L.lib().nfb_flow_add_ar_rqs(handle, C.byref(d)))
        del keep


class _UnconditionalCDF(nn.Module):
    def __init__(self, features, num_bins):
        super().__init__()
        self.unnormalized_widths = nn.Parameter(torch.zeros(features, num_bins))
        self.unnormalized_heights = nn.Parameter(torch.zeros(features, num_bins))
        self.unnormalized_derivatives = nn.Parameter(_BOUNDARY * torch.ones(features, num_bins - 1))


class _CoupledTransform(nn.Module):
    """`prqct`: feature index buffers, the conditioner and the unconditional transform."""

    def __init__(self, features, hidden_features, num_blocks, num_bins, reverse_mask, activation,
                 dropout_probability, init_identity, context_features=None):
        super().__init__()
        idx = torch.arange(features)
        start = 0 if reverse_mask else 1  # utils/masks.py:14-16 with even=reverse_mask
        transform = (idx % 2 == start % 2) if features > 1 else idx == start
        mask = torch.zeros(features, dtype=torch.bool)
        mask[start::2] = True
        self.register_buffer("identity_features", idx[~mask])
        self.register_buffer("transform_features", idx[mask])
        n_id, n_tr = int((~mask).sum()), int(mask.sum())
        if n_id == 0 or n_tr == 0:
            raise ValueError("Mask can't be empty.")
        self.transform_net = ResidualNet(n_id, n_tr * (3 * num_bins - 1), hidden_features, context_features, num_blocks,
                                         activation, dropout_probability, False)
        if init_identity:
            nn.init.constant_(self.transform_net.final_layer.weight, 0.0)
            nn.init.constant_(self.transform_net.final_layer.bias, _BOUNDARY)
        self.unconditional_transform = _UnconditionalCDF(n_id, num_bins)
        del transform


class CoupledRationalQuadraticSpline(NativeFlow):
    def __init__(self, num_input_channels, num_blocks, num_hidden_channels, num_context_channels=None,
                 num_bins=8, tails="linear", tail_bound=3.0, activation=nn.ReLU, dropout_probability=0.0,
                 reverse_mask=False, init_identity=True):
        super().__init__()
        if tails != "linear":
            raise NotImplementedError("only tails='linear' is on the CUDA path")
        if torch.is_tensor(tail_bound):
            raise NotImplementedError("per-feature tail bounds are not on the CUDA path")
        _check_bins(num_bins)
        self.features, self.num_bins, self.tail_bound = num_input_channels, num_bins, float(tail_bound)
        self.num_context_channels = num_context_channels
        self.prqct = _CoupledTransform(num_input_channels, num_hidden_channels, num_blocks, num_bins,
                                       reverse_mask, activation(), dropout_probability, init_identity,
                                       context_features=num_context_channels)

    def _conditional(self, z, context, sampling):
        """Context-conditioned coupling layer outside the fused block (see AutoregressiveRationalQuadraticSpline):
        Coupling.forward / .inverse of neural_spline/coupling.py:71-128 with the unconditional CDF of :221-253."""
        from .._standalone import apply_module, apply_sampling
        if not sampling:
            return apply_module(self, z, context)
        return apply_sampling(self, z, context)

    def _sampling_value(self, z, context, keep):
        from .._native import rqs_spline
        p, k = self.prqct, self.num_bins
        ident, trans = z[:, p.identity_features].contiguous(), z[:, p.transform_features].contiguous()
        wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
        yi, ldi = rqs_spline(ident, _uncond_rows(p.unconditional_transform, z.shape[0]), k, self.tail_bound, 1.0, True)
        params = p.transform_net._value(yi, context, None)
        if keep is not None:
            keep["params"], keep["yi"] = params, yi
        yt, ld = rqs_spline(trans, params, k, self.tail_bound, wh, True)
        return _merge(z, p, yi, yt), ld + ldi

    def _sampling_adjoint(self, z, x, context, keep, g_x, g_ld, need_z, need_ctx):
        from .._standalone import spline_inverse_backward
        spline = lambda zz, params, shared, wh, gx, gld: spline_inverse_backward(
            zz, params, shared, self.num_bins, gx, gld, wh, tail_bound=self.tail_bound, need_z=need_z)
        return _coupling_sampling_adjoint(self.prqct, z, context, keep, g_x, g_ld, spline, need_z, need_ctx)

    def _sampling_differentiable(self, context=None):
        """The stand-alone (context) path, and the native one with 8 bins (nfb_flow_sampling_backward on the layer's own
        handle)."""
        return self.num_context_channels is not None or context is not None or self.num_bins == 8

    def _value(self, z, context, keep):
        from .._native import rqs_spline
        p, k = self.prqct, self.num_bins
        ident, trans = z[:, p.identity_features].contiguous(), z[:, p.transform_features].contiguous()
        wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
        params = p.transform_net._value(ident, context, None)
        if keep is not None:
            keep["params"] = params
        yt, ld = rqs_spline(trans, params, k, self.tail_bound, wh, False)
        yi, ldi = rqs_spline(ident, _uncond_rows(p.unconditional_transform, z.shape[0]), k, self.tail_bound, 1.0, False)
        return _merge(z, p, yi, yt), ld + ldi

    def _adjoint(self, z, context, keep, grads, need_x, need_ctx):
        from .._standalone import spline_backward
        spline = lambda x, params, shared, wh, gy, gld: spline_backward(x, params, shared, self.num_bins, gy, gld, wh,
                                                                        tail_bound=self.tail_bound)
        return _coupling_adjoint(self.prqct, z, context, keep["params"], grads, spline, need_ctx)

    def forward(self, z, context=None):
        if self.num_context_channels is not None or context is not None:
            return self._conditional(z, context, True)
        if self.num_bins == 8 and wants_grad(self, z):   # the one-layer stack's native sampling backward
            from .._standalone import stack_sampling
            return stack_sampling(self._single(), [self], z, list(self.parameters()))
        return super().forward(z)

    def inverse(self, z, context=None):
        if self.num_context_channels is not None or context is not None:
            return self._conditional(z, context, False)
        return super().inverse(z)

    def _native_tensors(self):
        p = self.prqct
        return list(p.parameters()) + [p.identity_features, p.transform_features]

    def _native_add(self, handle, features):
        if features != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, features))
        p = self.prqct
        d = L.CoupledRqsDesc()
        d.features, d.num_bins, d.tail_bound = self.features, self.num_bins, self.tail_bound
        d.num_identity, d.num_transform = len(p.identity_features), len(p.transform_features)
        d.identity_features = p.identity_features.data_ptr()
        d.transform_features = p.transform_features.data_ptr()
        d.net, keep = resnet_desc(p.transform_net, masked=False)
        u = p.unconditional_transform
        d.uncond_widths = u.unnormalized_widths.data_ptr()
        d.uncond_heights = u.unnormalized_heights.data_ptr()
        d.uncond_derivatives = u.unnormalized_derivatives.data_ptr()
        L.check(L.lib().nfb_flow_add_coupled_rqs(handle, C.byref(d)))
        del keep


def _uncond_rows(u, rows):
    """The unconditional CDF's table [n_id, P] repeated for every row (_share_across_batch, coupling.py:217-219)."""
    up = torch.cat([u.unnormalized_widths, u.unnormalized_heights, u.unnormalized_derivatives], dim=1)
    return up.reshape(1, -1).expand(rows, -1).contiguous()


def _merge(z, p, yi, yt):
    out = torch.empty_like(z)
    out[:, p.identity_features] = yi
    out[:, p.transform_features] = yt
    return out


def _coupling_adjoint(p, z, context, params, grads, spline, need_ctx):
    """Backward of a coupling layer's density pass (Coupling.forward, neural_spline/coupling.py:71-98):
    transform features = spline adjoint; identity features = unconditional-CDF adjoint + the conditioner's data
    gradient.  spline(x, params, shared, wh_scale, g_y, g_log_det) -> (g_x, g_params)."""
    from .._standalone import conditioner_backward
    idf, trf = p.identity_features, p.transform_features
    g_out, g_ld = grads
    ident, trans = z[:, idf].contiguous(), z[:, trf].contiguous()
    u = p.unconditional_transform
    k = u.unnormalized_widths.shape[1]
    table = torch.cat([u.unnormalized_widths, u.unnormalized_heights, u.unnormalized_derivatives], dim=1).contiguous()
    wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
    g_tr, g_params = spline(trans, params, False, wh, g_out[:, trf].contiguous(), g_ld)
    g_id, g_table = spline(ident, table, True, 1.0, g_out[:, idf].contiguous(), g_ld)
    g_net, g_ctx, gmap = conditioner_backward(p.transform_net, False, ident, context, g_params, need_ctx=need_ctx)
    gz = torch.empty_like(z)
    gz[:, idf] = g_id + g_net
    gz[:, trf] = g_tr
    gmap[u.unnormalized_widths] = g_table[:, :k]
    gmap[u.unnormalized_heights] = g_table[:, k:2 * k]
    gmap[u.unnormalized_derivatives] = g_table[:, 2 * k:]
    return gz, g_ctx, gmap


def _coupling_sampling_adjoint(p, z, context, keep, g_out, g_ld, spline, need_z, need_ctx):
    """Backward of a coupling layer's sampling pass (Coupling.inverse, neural_spline/coupling.py:100-128): the inverse
    unconditional CDF gives yi on the identity features, the conditioner reads yi, the inverse spline maps the transform
    features.  Transform features: inverse-spline adjoint; then the conditioner's backward at yi (periodic features
    included); identity features: the unconditional CDF's inverse adjoint on g_yi = g_out[idf] + the conditioner's data
    gradient.  spline(z, params, shared, wh_scale, g_x, g_log_det) -> (g_z | None, g_params)."""
    from .._standalone import conditioner_backward
    idf, trf = p.identity_features, p.transform_features
    if g_out is None:
        g_out = torch.zeros_like(z)
    ident, trans = z[:, idf].contiguous(), z[:, trf].contiguous()
    u = p.unconditional_transform
    k = u.unnormalized_widths.shape[1]
    table = torch.cat([u.unnormalized_widths, u.unnormalized_heights, u.unnormalized_derivatives], dim=1).contiguous()
    wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
    g_tr, g_params = spline(trans, keep["params"], False, wh, g_out[:, trf].contiguous(), g_ld)
    g_net, g_ctx, gmap = conditioner_backward(p.transform_net, False, keep["yi"], context, g_params, need_ctx=need_ctx)
    g_id, g_table = spline(ident, table, True, 1.0, (g_out[:, idf] + g_net).contiguous(), g_ld)
    gz = None
    if need_z:
        gz = torch.empty_like(z)
        gz[:, idf] = g_id
        gz[:, trf] = g_tr
    gmap[u.unnormalized_widths] = g_table[:, :k]
    gmap[u.unnormalized_heights] = g_table[:, k:2 * k]
    gmap[u.unnormalized_derivatives] = g_table[:, 2 * k:]
    return gz, g_ctx, gmap


# ---------------------------------------------------------------------------------------------------------------
# Circular variants (reference: flows/neural_spline/wrapper.py:88-183, 247-311): `tails` is a per-feature list, so every
# knot has a derivative parameter (3K+1 per feature; utils/splines.py:48-57) and the bound may differ per feature.
# They run outside the fused block: conditioner = stand-alone tensor-core GEMMs (nets.*.forward), spline =
# csrc/nfb_kernels.cu rqs_rows_tails_kernel.
# ---------------------------------------------------------------------------------------------------------------
def _tail_tensors(tail_bound, feature_idx, ind_circ, n_features, device):
    """float32 tail bound and int32 circular flag per listed feature, on `device`."""
    idx = torch.as_tensor(feature_idx, dtype=torch.long).cpu()
    tb = tail_bound.detach().cpu().float()[idx] if torch.is_tensor(tail_bound) else \
        torch.full((len(idx),), float(tail_bound))
    circ = torch.zeros(n_features, dtype=torch.int32)
    circ[torch.as_tensor(list(ind_circ), dtype=torch.long)] = 1
    return tb.contiguous().to(device), circ[idx].contiguous().to(device)


class _CircularCoupledTransform(nn.Module):
    """`prqct` of the circular coupling layer: index buffers, conditioner (with periodic features), unconditional CDF."""

    def __init__(self, features, hidden_features, num_blocks, num_bins, ind_circ, tail_bound, mask, activation,
                 dropout_probability, init_identity, context_features=None):
        super().__init__()
        idx = torch.arange(features)
        self.register_buffer("identity_features", idx[mask <= 0])
        self.register_buffer("transform_features", idx[mask > 0])
        n_id, n_tr = len(self.identity_features), len(self.transform_features)
        if n_id == 0 or n_tr == 0:
            raise ValueError("Mask can't be empty.")
        circ = set(int(i) for i in ind_circ)
        ind_circ_id = [i for i, f in enumerate(self.identity_features.tolist()) if f in circ]
        if torch.is_tensor(tail_bound):   # wrapper.py:134-138: indexed by the position among the identity features
            scale_pf = np.pi / tail_bound[ind_circ_id] if ind_circ_id else 1.0
        else:
            scale_pf = np.pi / tail_bound
        from ..utils.nn import PeriodicFeaturesElementwise
        pf = PeriodicFeaturesElementwise(n_id, ind_circ_id, scale_pf) if ind_circ_id else None
        self.transform_net = ResidualNet(n_id, n_tr * (3 * num_bins + 1), hidden_features, context_features, num_blocks,
                                         activation, dropout_probability, False, preprocessing=pf)
        if init_identity:
            nn.init.constant_(self.transform_net.final_layer.weight, 0.0)
            nn.init.constant_(self.transform_net.final_layer.bias, _BOUNDARY)
        u = nn.Module()   # PiecewiseRationalQuadraticCDF with a tails list: K + 1 derivatives (coupling.py:194-200)
        u.unnormalized_widths = nn.Parameter(torch.zeros(n_id, num_bins))
        u.unnormalized_heights = nn.Parameter(torch.zeros(n_id, num_bins))
        u.unnormalized_derivatives = nn.Parameter(_BOUNDARY * torch.ones(n_id, num_bins + 1))
        if torch.is_tensor(tail_bound):
            u.register_buffer("tail_bound", tail_bound[self.identity_features])      # coupling.py:210-213
        self.unconditional_transform = u
        if torch.is_tensor(tail_bound):
            self.register_buffer("tail_bound", tail_bound[self.transform_features])   # coupling.py:317-318


class CircularCoupledRationalQuadraticSpline(Flow):
    def __init__(self, num_input_channels, num_blocks, num_hidden_channels, ind_circ, num_context_channels=None,
                 num_bins=8, tail_bound=3.0, activation=nn.ReLU, dropout_probability=0.0, reverse_mask=False,
                 mask=None, init_identity=True):
        super().__init__()
        _check_bins(num_bins)
        if mask is None:   # utils/masks.py:5-17 create_alternating_binary_mask(features, even=reverse_mask)
            mask = torch.zeros(num_input_channels, dtype=torch.uint8)
            mask[(0 if reverse_mask else 1)::2] = 1
        self.features, self.num_bins = num_input_channels, num_bins
        self.ind_circ = [int(i) for i in ind_circ]
        self._tail_bound = tail_bound
        self.prqct = _CircularCoupledTransform(num_input_channels, num_hidden_channels, num_blocks, num_bins,
                                               self.ind_circ, tail_bound, torch.as_tensor(mask), activation(),
                                               dropout_probability, init_identity, context_features=num_context_channels)

    def _tails(self, p, device):
        return (_tail_tensors(self._tail_bound, p.identity_features, self.ind_circ, self.features, device),
                _tail_tensors(self._tail_bound, p.transform_features, self.ind_circ, self.features, device))

    def _run(self, z, context, sampling):
        from .._standalone import apply_module, apply_sampling
        if not sampling:   # Coupling.forward (coupling.py:71-98)
            return apply_module(self, z, context)
        return apply_sampling(self, z, context)   # Coupling.inverse (:100-128)

    def _sampling_value(self, z, context, keep):
        from .._native import rqs_spline_tails
        p, k = self.prqct, self.num_bins
        (tb_id, c_id), (tb_tr, c_tr) = self._tails(p, z.device)
        ident, trans = z[:, p.identity_features].contiguous(), z[:, p.transform_features].contiguous()
        wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
        yi, ldi = rqs_spline_tails(ident, _uncond_rows(p.unconditional_transform, z.shape[0]), k, k + 1, tb_id, c_id,
                                   1.0, True)
        params = p.transform_net._value(yi, context, None)
        if keep is not None:
            keep["params"], keep["yi"] = params, yi
        yt, ld = rqs_spline_tails(trans, params, k, k + 1, tb_tr, c_tr, wh, True)
        return _merge(z, p, yi, yt), ld + ldi

    def _sampling_adjoint(self, z, x, context, keep, g_x, g_ld, need_z, need_ctx):
        from .._standalone import spline_inverse_backward
        p, k = self.prqct, self.num_bins
        (tb_id, c_id), (tb_tr, c_tr) = self._tails(p, z.device)

        def spline(zz, params, shared, wh, gx, gld):
            tb, circ = (tb_id, c_id) if shared else (tb_tr, c_tr)
            return spline_inverse_backward(zz, params, shared, k, gx, gld, wh, num_derivatives=k + 1, tails=tb,
                                           circular=circ, need_z=need_z)
        return _coupling_sampling_adjoint(p, z, context, keep, g_x, g_ld, spline, need_z, need_ctx)

    def _sampling_differentiable(self, context=None):
        return True

    def _value(self, z, context, keep):
        from .._native import rqs_spline_tails
        p, k = self.prqct, self.num_bins
        (tb_id, c_id), (tb_tr, c_tr) = self._tails(p, z.device)
        ident, trans = z[:, p.identity_features].contiguous(), z[:, p.transform_features].contiguous()
        wh = 1.0 / float(np.sqrt(p.transform_net.hidden_features))
        params = p.transform_net._value(ident, context, None)
        if keep is not None:
            keep["params"] = params
        yt, ld = rqs_spline_tails(trans, params, k, k + 1, tb_tr, c_tr, wh, False)
        yi, ldi = rqs_spline_tails(ident, _uncond_rows(p.unconditional_transform, z.shape[0]), k, k + 1, tb_id, c_id,
                                   1.0, False)
        return _merge(z, p, yi, yt), ld + ldi

    def _adjoint(self, z, context, keep, grads, need_x, need_ctx):
        from .._standalone import spline_backward
        p, k = self.prqct, self.num_bins
        (tb_id, c_id), (tb_tr, c_tr) = self._tails(p, z.device)

        def spline(x, params, shared, wh, gy, gld):
            tb, circ = (tb_id, c_id) if shared else (tb_tr, c_tr)
            return spline_backward(x, params, shared, k, gy, gld, wh, num_derivatives=k + 1, tails=tb, circular=circ)
        return _coupling_adjoint(p, z, context, keep["params"], grads, spline, need_ctx)

    def forward(self, z, context=None):   # wrapper.py:177-179: forward = prqct.inverse
        return self._run(z, context, True)

    def inverse(self, z, context=None):
        return self._run(z, context, False)


class CircularAutoregressiveRationalQuadraticSpline(Flow):
    def __init__(self, num_input_channels, num_blocks, num_hidden_channels, ind_circ, num_context_channels=None,
                 num_bins=8, tail_bound=3, activation=nn.ReLU, dropout_probability=0.0, permute_mask=True,
                 init_identity=True):
        super().__init__()
        _check_bins(num_bins)
        self.features, self.num_bins = num_input_channels, num_bins
        self.ind_circ = [int(i) for i in ind_circ]
        self._tail_bound = tail_bound
        from ..utils.nn import PeriodicFeaturesElementwise
        # neural_spline/autoregressive.py:44-53: periodic features of the circular coordinates in front of the MADE
        scale_pf = np.pi / tail_bound[self.ind_circ] if torch.is_tensor(tail_bound) else np.pi / tail_bound
        pf = PeriodicFeaturesElementwise(num_input_channels, self.ind_circ, scale_pf)
        self.mprqat = _ARTransform(num_input_channels, num_hidden_channels, num_bins, num_blocks, permute_mask,
                                   activation(), dropout_probability, init_identity,
                                   context_features=num_context_channels, output_multiplier=3 * num_bins + 1,
                                   preprocessing=pf)
        if torch.is_tensor(tail_bound):
            self.mprqat.register_buffer("tail_bound", tail_bound)    # neural_spline/autoregressive.py:82-83

    def _run(self, z, context, sampling):
        from .._standalone import apply_module, apply_sampling
        if not sampling:   # one MADE pass (affine/autoregressive.py:24-27)
            return apply_module(self, z, context)
        return apply_sampling(self, z, context)

    def _sampling_value(self, z, context, keep):
        from .._native import rqs_spline_tails
        k, net = self.num_bins, self.mprqat.autoregressive_net
        tb, circ = _tail_tensors(self._tail_bound, range(self.features), self.ind_circ, self.features, z.device)
        out, ld = torch.zeros_like(z), None   # D passes (:29-38)
        for _ in range(self.features):
            out, ld = rqs_spline_tails(z, net._value(out, context, None), k, k + 1, tb, circ, 1.0, True)
        return out, ld

    def _sampling_adjoint(self, z, x, context, keep, g_x, g_ld, need_z, need_ctx):
        from .._standalone import ar_rqs_sampling_backward
        k = self.num_bins
        tb, circ = _tail_tensors(self._tail_bound, range(self.features), self.ind_circ, self.features, z.device)
        return ar_rqs_sampling_backward(self.mprqat.autoregressive_net, self.features, k, k + 1, 0.0, tb, circ, z, x,
                                        context, g_x, g_ld, need_z, need_ctx)

    def _sampling_differentiable(self, context=None):
        return True

    def _value(self, z, context, keep):   # MADE has no hidden_features: no 1/sqrt(H)
        from .._native import rqs_spline_tails
        k = self.num_bins
        tb, circ = _tail_tensors(self._tail_bound, range(self.features), self.ind_circ, self.features, z.device)
        params = self.mprqat.autoregressive_net._value(z, context, None)
        if keep is not None:
            keep["params"] = params
        return rqs_spline_tails(z, params, k, k + 1, tb, circ, 1.0, False)

    def _adjoint(self, z, context, keep, grads, need_x, need_ctx):
        from .._standalone import conditioner_backward, spline_backward
        k = self.num_bins
        tb, circ = _tail_tensors(self._tail_bound, range(self.features), self.ind_circ, self.features, z.device)
        gz, g_params = spline_backward(z, keep["params"], False, k, grads[0], grads[1], 1.0, num_derivatives=k + 1,
                                       tails=tb, circular=circ)
        g_net, g_ctx, gmap = conditioner_backward(self.mprqat.autoregressive_net, True, z, context, g_params,
                                                  need_ctx=need_ctx)
        return gz + g_net, g_ctx, gmap

    def forward(self, z, context=None):   # wrapper.py:305-307: forward = mprqat.inverse
        return self._run(z, context, True)

    def inverse(self, z, context=None):
        return self._run(z, context, False)
