"""Host-side glue between the nn.Module shims and the C ABI (include/nfb200.h).

`FlowHandle` owns one `nfb_flow_t`: the packed device image of an ordered list of layers (plus an
optional DiagGaussian or GaussianMixture base).  It re-reads the parameters when they change (optimizer step,
load_state_dict, .to()) by comparing (data_ptr, _version) signatures -- the same idea as the
reference's cache invalidation in `_Linear.train()` (normflows/flows/mixing.py:328-332)."""
import ctypes as C

import torch

import operator

from . import _lib as L

_VERSION = operator.attrgetter("_version")

# Packed-weight caches are keyed on (data_ptr, Tensor._version).  `p.data.add_()` / `.data.copy_()` (older
# optimizers, EMA/SWA swaps, weight clipping) change the values WITHOUT bumping the version the Parameter
# reports, so the caches also watch a process-wide generation counter that is bumped by
#   * every torch optimizer step (global post-hook below),
#   * load_state_dict / train() / eval() on a NormalizingFlow (core.py),
#   * an explicit `normflows.invalidate_packed_weights()` (or `model.repack()`),
# which is the documented call after any other out-of-band `.data` mutation.  `cached` below applies this to the
# image path's caches; FlowHandle keeps its own split signature.
_GENERATION = [0]


def invalidate_packed_weights():
    """Force every packed device image (bf16 split weight streams, folded Glow convolutions) to be rebuilt from
    the current parameter values on its next use."""
    _GENERATION[0] += 1


def generation():
    return _GENERATION[0]


def cached(owner, key, tensors, extra, build):
    """build() once per parameter version: the value is kept in owner.__dict__[key] under the signature of `tensors`
    ((data_ptr, _version) each), `extra` and the generation, and rebuilt when that signature changes."""
    sig = tuple((t.data_ptr(), t._version) for t in tensors) + tuple(extra) + (_GENERATION[0],)
    hit = owner.__dict__.get(key)
    if hit is None or hit[0] != sig:
        hit = (sig, build())
        owner.__dict__[key] = hit
    return hit[1]


try:  # torch >= 2.0
    from torch.optim.optimizer import register_optimizer_step_post_hook as _reg_post

    _reg_post(lambda opt, args, kwargs: invalidate_packed_weights())
except Exception:  # pragma: no cover
    pass


def require_cuda_f32(t, what="input"):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(
            f"{what} is on {t.device}: normflows-b200 runs the transform stack as sm_90a CUDA kernels "
            "only; there is no CPU/eager fallback. Move the model and data to a CUDA device.")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{what} has dtype {t.dtype}; the CUDA path computes in float32 only")
    return t.contiguous()


class FlowHandle:
    def __init__(self, layers, base=None, use_tensor_cores=True):
        self.layers = list(layers)
        self.base = base
        self.use_tc = bool(use_tensor_cores)
        self._h = None
        self._sig_ptr = None
        self._sig_ver = None
        self._features = None
        self._slots = None
        self._calls = 0
        self._gen = -1

    def invalidate(self):
        self._gen = -1

    # -- lifetime -------------------------------------------------------------------------
    def close(self):
        if self._h is not None:
            L.lib().nfb_flow_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _tensors_slow(self):
        ts = []
        for layer in self.layers:
            ts.extend(layer._native_tensors())
        if self.base is not None:
            ts.extend(self.base._native_tensors())
        return ts

    def _build_slots(self):
        """Walking the module tree through nn.Module.__getattr__ costs ~1.3 ms for a 32-block stack -- more than
        a fifth of the fused kernel's run time and fully exposed on the synchronous host path.  Remember WHERE
        each tensor lives instead ((module._parameters | module._buffers, name) pairs): a per-call refresh is
        then one dict lookup per tensor (~40 us) and still sees `.to()`, `load_state_dict`, optimizer steps and
        re-registered parameters, because it re-reads the dict entries rather than caching the tensors."""
        ts = self._tensors_slow()
        where = {}
        mods = list(self.layers) + ([self.base] if self.base is not None else [])
        for root in mods:
            for m in root.modules():
                for d in (m._parameters, m._buffers):
                    for k, v in d.items():
                        if v is not None:
                            where.setdefault(id(v), (d, k))
        slots = [where.get(id(t)) for t in ts]
        self._slots = None if any(sl is None for sl in slots) else slots  # plain-attribute tensor: slow path
        self._calls = 0
        return ts

    def _tensors(self):
        self._calls += 1
        if self._slots is None or self._calls & 255 == 0:
            # every 256th call re-derive the list the slow way: catches a sub-module OBJECT that was swapped
            # out after the first call (the only change the dict slots cannot see)
            ts = self._tensors_slow()
            if self._slots is not None and any(d[k] is not t for (d, k), t in zip(self._slots, ts)):
                ts = self._build_slots()
            return ts
        return [d[k] for d, k in self._slots]

    def ensure(self, features, device):
        if self._h is None and self._slots is None:
            ts = self._build_slots()
        else:
            ts = self._tensors()
        sig_ptr = (*map(torch.Tensor.data_ptr, ts), features, device.index)
        sig_ver = tuple(map(_VERSION, ts))
        gen = _GENERATION[0]
        if sig_ptr == self._sig_ptr and sig_ver == self._sig_ver and gen == self._gen and self._h is not None:
            return self._h
        for t in ts:  # validated whenever anything changed (new tensors, new device, first call)
            if t.device != device:
                raise RuntimeError(f"parameter on {t.device} but input on {device}: call model.to(device)")
            if t.dtype.is_floating_point and t.dtype != torch.float32:
                raise RuntimeError(f"parameter dtype {t.dtype}: the CUDA path computes in float32 only")
            if not t.is_contiguous():
                raise RuntimeError("non-contiguous parameter")
        lib = L.lib()
        with torch.cuda.device(device):
            if self._h is None or sig_ptr != self._sig_ptr:
                self.close()
                h = C.c_void_p()
                L.check(lib.nfb_flow_create(C.byref(h), features))
                self._h = h
                try:
                    for layer in self.layers:
                        layer._native_add(self._h, features)
                    if self.base is not None:
                        self.base._native_attach(self._h, features)
                    L.check(lib.nfb_flow_finalize(self._h, int(self.use_tc), L.stream_ptr()))
                except Exception:
                    self.close()
                    raise
                self._sig_ptr, self._sig_ver, self._features = sig_ptr, sig_ver, features
            elif sig_ver != self._sig_ver or gen != self._gen:
                L.check(lib.nfb_flow_repack(self._h, L.stream_ptr()))
                self._sig_ver = sig_ver
            self._gen = gen
        return self._h

    # -- operations -------------------------------------------------------------------------
    def _prep(self, z):
        z = require_cuda_f32(z)
        if z.dim() != 2:
            raise ValueError("Inputs must be a 2D tensor [batch, features] on the CUDA path.")
        return z, self.ensure(z.shape[1], z.device)

    def layer_apply(self, index, direction, z):
        z, h = self._prep(z)
        out = torch.empty_like(z)
        ld = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        if z.shape[0] == 0:
            return out, ld
        with torch.cuda.device(z.device):
            L.check(L.lib().nfb_flow_layer_apply(h, index, direction, L.ptr(z), L.ptr(out), L.ptr(ld),
                                                 z.shape[0], 0, L.stream_ptr()))
        return out, ld

    def transform(self, direction, z):
        z, h = self._prep(z)
        out = torch.empty_like(z)
        ld = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
        if z.shape[0] == 0:
            return out, ld
        with torch.cuda.device(z.device):
            L.check(L.lib().nfb_flow_transform(h, direction, L.ptr(z), L.ptr(out), L.ptr(ld), z.shape[0],
                                               L.stream_ptr()))
        return out, ld

    def log_prob(self, x):
        x, h = self._prep(x)
        lq = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
        if x.shape[0] == 0:
            return lq
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_flow_log_prob(h, L.ptr(x), L.ptr(lq), x.shape[0], L.stream_ptr()))
        return lq

    def forward_kld(self, x, want_sum=False, sum_out=None):
        """-mean(log_q) as a 0-dim fp32 tensor; optionally also sum(log_q) (fp64) -- either returned
        (want_sum) or written into the caller's 1-element fp64 tensor `sum_out` (data-parallel callers)."""
        x, h = self._prep(x)
        loss = torch.empty((), dtype=torch.float32, device=x.device)
        s = sum_out if sum_out is not None else (
            torch.empty(2, dtype=torch.float64, device=x.device) if want_sum else None)
        if s is not None and (s.dtype != torch.float64 or s.device != x.device or s.numel() < 2
                              or not s.is_contiguous()):
            raise ValueError("sum_out must be a contiguous float64 tensor [sum, rows] on the input's device")
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_flow_forward_kld(h, L.ptr(x), x.shape[0], L.ptr(loss), L.ptr(s),
                                                 L.stream_ptr()))
        return (loss, s) if want_sum else loss

    def forward_kld_host(self, x_host, device):
        """x_host: pinned (or pageable) CPU float32 tensor [B, D]; H2D + D2H copies are inside the call."""
        if x_host.is_cuda or x_host.dtype != torch.float32 or x_host.dim() != 2:
            raise ValueError("forward_kld_host expects a CPU float32 [batch, features] tensor")
        x_host = x_host.contiguous()
        h = self.ensure(x_host.shape[1], device)
        out = C.c_float()
        with torch.cuda.device(device):
            L.check(L.lib().nfb_flow_forward_kld_host(h, C.c_void_p(x_host.data_ptr()), x_host.shape[0],
                                                      C.byref(out)))
        return out.value

    def log_prob_host(self, x_host, device):
        if x_host.is_cuda or x_host.dtype != torch.float32 or x_host.dim() != 2:
            raise ValueError("log_prob_host expects a CPU float32 [batch, features] tensor")
        x_host = x_host.contiguous()
        h = self.ensure(x_host.shape[1], device)
        out = torch.empty(x_host.shape[0], dtype=torch.float32)
        with torch.cuda.device(device):
            L.check(L.lib().nfb_flow_log_prob_host(h, C.c_void_p(x_host.data_ptr()), C.c_void_p(out.data_ptr()),
                                                   x_host.shape[0]))
        return out

    def launch_count(self):
        return int(L.lib().nfb_flow_last_launch_count(self._h)) if self._h is not None else 0

    def sampling_units(self):
        """Units of the whole-stack sampling plan (0: the sampling direction runs layer by layer)."""
        return int(L.lib().nfb_flow_sampling_units(self._h)) if self._h is not None else 0

    def fused_layers(self):
        if self._h is None:
            return []
        return [i for i in range(len(self.layers)) if L.lib().nfb_flow_layer_is_fused(self._h, i)]


def linear(x, weight, bias=None, a_relu=False, relu_out=False, resid=None):
    """act(x) @ weight.T + bias (+ resid) on the tensor core (csrc/nfb_gemm_tc.cu through nfb_gemm_f32).
    x: [M, K] CUDA float32 (row stride free), weight: [N, K]; returns a new [M, N] tensor."""
    x = require_cuda_f32(x)
    if x.dim() != 2:
        raise ValueError("linear expects a 2-D input")
    weight = weight.contiguous()
    M, K = x.shape
    N = weight.shape[0]
    out = torch.empty(M, N, dtype=torch.float32, device=x.device)
    if M == 0:
        return out
    d = L.GemmDesc()
    d.A, d.B, d.C = x.data_ptr(), weight.data_ptr(), out.data_ptr()
    d.lda, d.ldb, d.ldc, d.M, d.N, d.K = x.stride(0), K, N, M, N, K
    d.a_relu, d.relu_out = int(a_relu), int(relu_out)
    if bias is not None:
        d.bias = bias.contiguous().data_ptr()
    if resid is not None:
        resid = resid.contiguous()
        d.resid, d.ldres = resid.data_ptr(), resid.stride(0)
    with torch.cuda.device(x.device):
        L.check(L.lib().nfb_gemm_f32(C.byref(d), L.stream_ptr()))
    return out


def linear_t(x, weight):
    """x @ weight for weight [K, N] row-major (the dgrad / vector-Jacobian layout: no transpose in memory)."""
    x = require_cuda_f32(x)
    weight = weight.contiguous()
    M, K = x.shape
    N = weight.shape[1]
    out = torch.empty(M, N, dtype=torch.float32, device=x.device)
    if M == 0:
        return out
    d = L.GemmDesc()
    d.A, d.B, d.C = x.data_ptr(), weight.data_ptr(), out.data_ptr()
    d.lda, d.ldb, d.ldc, d.M, d.N, d.K, d.b_mn = x.stride(0), N, N, M, N, K, 1
    with torch.cuda.device(x.device):
        L.check(L.lib().nfb_gemm_f32(C.byref(d), L.stream_ptr()))
    return out


def swish(x, b, want_derivative=False):
    """(x sigmoid(b x) / 1.1, derivative or None) -- nets/lipschitz.py:642-648 with b = softplus(beta)."""
    x = require_cuda_f32(x)
    a = torch.empty_like(x)
    da = torch.empty_like(x) if want_derivative else None
    if x.numel():
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_swish(L.ptr(x), float(b), x.numel(), L.ptr(a), L.ptr(da), L.stream_ptr()))
    return a, da


def mul_rows(src, m, nt):
    """src: [nt, ...] stacked tensors, m: [...]; returns src * m broadcast over the leading dim."""
    out = torch.empty_like(src)
    if src.numel():
        with torch.cuda.device(src.device):
            L.check(L.lib().nfb_mul_rows(L.ptr(src), L.ptr(m), m.numel(), int(nt), L.ptr(out), L.stream_ptr()))
    return out


def rowdot(a, b, c=1.0, out=None):
    """out[r] (+)= c * sum_j a[r, j] b[r, j]"""
    acc = out is not None
    if out is None:
        out = torch.empty(a.shape[0], dtype=torch.float32, device=a.device)
    if a.shape[0]:
        with torch.cuda.device(a.device):
            L.check(L.lib().nfb_rowdot(L.ptr(a), L.ptr(b), a.shape[0], a.shape[1], float(c), int(acc), L.ptr(out),
                                       L.stream_ptr()))
    return out


def glu_residual(h, t, c):
    out = torch.empty_like(h)
    if h.numel():
        with torch.cuda.device(h.device):
            L.check(L.lib().nfb_glu_residual(L.ptr(h), L.ptr(t), L.ptr(c), h.numel(), L.ptr(out), L.stream_ptr()))
    return out


def resnet_forward(net, x, masked, context=None):
    """ResidualNet.forward (nets/resnet.py:92-104) / MADE.forward (nets/made.py:296-304) outside the fused kernel
    (stand-alone call of the module, or a context-conditioned layer): pre-activation residual blocks, every Linear one
    tensor-core GEMM with fused bias / ReLU / residual; with a context the blocks end in the GLU gate
    h + t * sigmoid(context_layer(context)) (csrc/nfb_residual.cu)."""
    eff = (lambda l: l.weight * l.mask) if masked else (lambda l: l.weight)
    if context is not None:
        context = require_cuda_f32(context, "context")
    if context is None:
        h = linear(x, eff(net.initial_layer), net.initial_layer.bias)
    elif masked:   # MADE: initial_layer(inputs) + context_layer(context)   (made.py:297-300)
        h = linear(x, eff(net.initial_layer), net.initial_layer.bias)
        h = linear(context, net.context_layer.weight, net.context_layer.bias, resid=h)
    else:          # ResidualNet: initial_layer(cat(inputs, context))        (resnet.py:98-99)
        h = linear(torch.cat((require_cuda_f32(x), context), dim=1), net.initial_layer.weight, net.initial_layer.bias)
    for blk in net.blocks:
        l0, l1 = blk.linear_layers
        t = linear(h, eff(l0), l0.bias, a_relu=True)
        if context is None:
            h = linear(t, eff(l1), l1.bias, a_relu=True, resid=h)
        else:
            t = linear(t, eff(l1), l1.bias, a_relu=True)
            h = glu_residual(h, t, linear(context, blk.context_layer.weight, blk.context_layer.bias))
    return linear(h, eff(net.final_layer), net.final_layer.bias)


def rqs_spline(x, params, num_bins, tail_bound, wh_scale, inverse):
    """utils/splines.py:16-97 on contiguous [rows, feats] inputs with per-element parameters (csrc/nfb_kernels.cu)."""
    x = require_cuda_f32(x)
    params = params.contiguous()
    y = torch.empty_like(x)
    ld = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    if x.shape[0]:
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_rqs_spline(L.ptr(x), L.ptr(params), L.ptr(y), L.ptr(ld), x.shape[0], x.shape[1],
                                           num_bins, C.c_float(tail_bound), C.c_float(wh_scale), int(inverse), 0,
                                           L.stream_ptr()))
    return y, ld


def rqs_spline_tails(x, params, num_bins, num_derivatives, tail_bound, circular, wh_scale, inverse):
    """utils/splines.py:16-97 with per-feature tails (:42-57): tail_bound float32 [feats] and circular int32 [feats] on
    the device, params [rows, feats * (2 K + num_derivatives)] (csrc/nfb_kernels.cu rqs_rows_tails_kernel)."""
    x = require_cuda_f32(x)
    params = params.contiguous()
    y = torch.empty_like(x)
    ld = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    if x.shape[0]:
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_rqs_spline_tails(L.ptr(x), L.ptr(params), L.ptr(y), L.ptr(ld), x.shape[0], x.shape[1],
                                                 num_bins, num_derivatives, L.ptr(tail_bound), L.ptr(circular),
                                                 C.c_float(wh_scale), int(inverse), 0, L.stream_ptr()))
    return y, ld


def periodic_features(x, slot, weights, scale, bias=None):
    """utils/nn.py:64-130 PeriodicFeaturesElementwise.forward on the device (csrc/nfb_kernels.cu)."""
    x = require_cuda_f32(x)
    y = torch.empty_like(x)
    if x.numel():
        with torch.cuda.device(x.device):
            L.check(L.lib().nfb_periodic_features(L.ptr(x), L.ptr(y), x.shape[0], x.shape[1], L.ptr(slot),
                                                  L.ptr(weights), L.ptr(scale), L.ptr(bias) if bias is not None else None,
                                                  L.stream_ptr()))
    return y


def resnet_desc(net, masked):
    """Fill an nfb_resnet_desc_t from a ResidualNet / MADE shim; returns (desc, keepalive)."""
    nb = len(net.blocks)
    VP = C.c_void_p
    wb = (VP * max(1, 2 * nb))()
    bb = (VP * max(1, 2 * nb))()
    mb = (VP * max(1, 2 * nb))()
    for i, blk in enumerate(net.blocks):
        for j in range(2):
            lin = blk.linear_layers[j]
            wb[2 * i + j] = lin.weight.data_ptr()
            bb[2 * i + j] = lin.bias.data_ptr()
            mb[2 * i + j] = lin.mask.data_ptr() if masked else None
    d = L.ResnetDesc()
    d.in_features = net.initial_layer.in_features
    d.hidden_features = net.initial_layer.out_features
    d.out_features = net.final_layer.out_features
    d.num_blocks = nb
    d.w_initial, d.b_initial = net.initial_layer.weight.data_ptr(), net.initial_layer.bias.data_ptr()
    d.m_initial = net.initial_layer.mask.data_ptr() if masked else None
    d.w_blocks = C.cast(wb, C.POINTER(VP))
    d.b_blocks = C.cast(bb, C.POINTER(VP))
    d.m_blocks = C.cast(mb, C.POINTER(VP)) if masked else None
    d.w_final, d.b_final = net.final_layer.weight.data_ptr(), net.final_layer.bias.data_ptr()
    d.m_final = net.final_layer.mask.data_ptr() if masked else None
    return d, (wb, bb, mb)


def mlp_desc(mlp):
    d = L.MlpDesc()
    if mlp is None:
        d.num_layers = 0
        return d
    lins = mlp.linear_layers()
    if len(lins) > 6:
        raise NotImplementedError("MLP with more than 6 Linear layers is not supported by the CUDA path")
    d.num_layers = len(lins)
    d.sizes[0] = lins[0].in_features
    for i, lin in enumerate(lins):
        d.sizes[i + 1] = lin.out_features
        d.w[i] = lin.weight.data_ptr()
        d.b[i] = lin.bias.data_ptr()
    d.leaky = float(mlp.leaky)
    return d
