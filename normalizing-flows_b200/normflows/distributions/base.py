"""Base distributions: only what the density pass ends in (reference:
normflows/distributions/base.py:8-49 BaseDistribution, :53-103 DiagGaussian, :573-659 GaussianMixture)."""
import numpy as np
import torch
from torch import nn

from .. import _lib as L
from .._image_autograd import gaussian_table_log_prob
from .._native import require_cuda_f32


def _tempered(log_scale, temperature):
    """Temperature annealing: log_scale + log T (base.py:318-319, 339-340)."""
    return log_scale if temperature is None else log_scale + np.log(temperature)


def _labels(y, device):
    """int64 class indices on `device`; one-hot rows select their class (base.py:336-337, 403-411)."""
    return (y if y.dim() == 1 else torch.argmax(y, dim=1)).to(device=device, dtype=torch.int64).contiguous()


class BaseDistribution(nn.Module):
    def forward(self, num_samples=1):
        raise NotImplementedError

    def log_prob(self, z):
        raise NotImplementedError

    def sample(self, num_samples=1, **kwargs):
        z, _ = self.forward(num_samples, **kwargs)
        return z


class DiagGaussian(BaseDistribution):
    def __init__(self, shape, trainable=True):
        super().__init__()
        if isinstance(shape, int):
            shape = (shape,)
        shape = tuple(shape)
        self.shape, self.n_dim, self.d = shape, len(shape), int(np.prod(shape))
        if trainable:
            self.loc = nn.Parameter(torch.zeros(1, *shape))
            self.log_scale = nn.Parameter(torch.zeros(1, *shape))
        else:
            self.register_buffer("loc", torch.zeros(1, *shape))
            self.register_buffer("log_scale", torch.zeros(1, *shape))
        self.temperature = None

    def forward(self, num_samples=1, context=None):
        # sampling from the base is off the hot path (core.py:167-180): plain torch RNG
        eps = torch.randn((num_samples,) + self.shape, dtype=self.loc.dtype, device=self.loc.device)
        ls = _tempered(self.log_scale, self.temperature)
        z = self.loc + torch.exp(ls) * eps
        log_p = -0.5 * self.d * np.log(2 * np.pi) - torch.sum(ls + 0.5 * eps ** 2,
                                                              list(range(1, self.n_dim + 1)))
        return z, log_p

    def log_prob(self, z, context=None):
        z = require_cuda_f32(z)
        ls = _tempered(self.log_scale, self.temperature)
        return gaussian_table_log_prob(z, self.loc.reshape(self.d, 1), ls.reshape(self.d, 1), None, 1)

    # the base of a flow object (_native.FlowHandle): its tensors, in the order of its gradient slots, and its setter
    def _native_tensors(self):
        return [self.loc, self.log_scale]

    def _native_attach(self, handle, features):
        L.check(L.lib().nfb_flow_set_base_diag_gaussian(handle, L.ptr(self.loc), L.ptr(self.log_scale)))


class GaussianMixture(BaseDistribution):
    """Mixture of Gaussians with diagonal covariances (reference: distributions/base.py:573-659): the same parameters
    (or buffers, trainable=False) `loc` [1, K, D], `log_scale` [1, K, D], `weight_scores` [1, K] and the same seeded
    construction (a `loc=None` default is drawn with np.random.randn).  The tensors are float32 (the CUDA path computes in
    float32 only); a reference state_dict (float64) loads with strict=True, converted on load.  `log_prob` is the CUDA
    kernel (csrc/nfb_mixture.cu) with its native backward, gradients to z and all three parameters; with log_softmax
    in place of log(softmax), a weight that underflows gives a finite, negligible term instead of -inf.  Sampling draws
    the modes with torch.multinomial and eps with torch.randn (plumbing RNG, like the other bases) and is
    reparameterised: z = loc[m] + exp(log_scale[m]) eps in differentiable torch."""

    def __init__(self, n_modes, dim, loc=None, scale=None, weights=None, trainable=True):
        super().__init__()
        self.n_modes = n_modes
        self.dim = dim
        if loc is None:
            loc = np.random.randn(self.n_modes, self.dim)
        loc = np.array(loc)[None, ...]
        if scale is None:
            scale = np.ones((self.n_modes, self.dim))
        scale = np.array(scale)[None, ...]
        if weights is None:
            weights = np.ones(self.n_modes)
        weights = np.array(weights)[None, ...]
        weights = weights / weights.sum(1)
        f32 = lambda v: torch.tensor(v, dtype=torch.float32)
        tensors = {"loc": f32(1.0 * loc), "log_scale": f32(np.log(1.0 * scale)),
                   "weight_scores": f32(np.log(1.0 * weights))}
        for name, t in tensors.items():
            if trainable:
                setattr(self, name, nn.Parameter(t))
            else:
                self.register_buffer(name, t)

    def forward(self, num_samples=1):
        dev = self.loc.device
        weights = torch.softmax(self.weight_scores.detach(), 1)
        mode = torch.multinomial(weights[0, :], num_samples, replacement=True)
        eps = torch.randn(num_samples, self.dim, dtype=self.loc.dtype, device=dev)
        z = self.loc[0, mode] + torch.exp(self.log_scale[0, mode]) * eps
        return z, self.log_prob(z)

    def log_prob(self, z):
        from .._standalone import MixtureLogProbFn
        z = require_cuda_f32(z)
        if z.dim() != 2 or z.shape[1] != self.dim:
            raise ValueError(f"GaussianMixture.log_prob expects [batch, {self.dim}], got {list(z.shape)}")
        return MixtureLogProbFn.apply(z, *(require_cuda_f32(t, "GaussianMixture parameter")
                                           for t in self._native_tensors()))

    def _native_tensors(self):
        return [self.loc, self.log_scale, self.weight_scores]

    def _native_attach(self, handle, features):
        if features != self.dim:
            raise ValueError(f"GaussianMixture of dim {self.dim} as the base of a {features}-feature flow")
        L.check(L.lib().nfb_flow_set_base_gaussian_mixture(handle, self.n_modes, L.ptr(self.loc), L.ptr(self.log_scale),
                                                           L.ptr(self.weight_scores)))


class UniformGaussian(BaseDistribution):
    """Uniform on the features `ind` (width scale[ind], centred at 0), Gaussian with standard deviation scale on the
    others (reference: distributions/base.py:198-270); the base of examples/paper_example_nsf.ipynb.  Same buffers
    (`ind`, `ind_`, `inv_perm`, `scale`).  Sampling is torch RNG, reparameterised like DiagGaussian.forward; the density is
    the diagonal-Gaussian kernel on the Gaussian columns plus the uniform part's constant.  Like the reference it does
    not check the uniform support."""

    def __init__(self, ndim, ind, scale=None):
        super().__init__()
        self.ndim = ndim
        if isinstance(ind, int):
            ind = [ind]
        if torch.is_tensor(ind):
            self.register_buffer("ind", ind.long())
        else:
            self.register_buffer("ind", torch.tensor(ind, dtype=torch.long))
        uniform = set(self.ind.tolist())
        self.register_buffer("ind_", torch.tensor([i for i in range(ndim) if i not in uniform], dtype=torch.long))
        perm_ = torch.cat((self.ind, self.ind_))
        inv_perm_ = torch.zeros_like(perm_)
        inv_perm_[perm_] = torch.arange(ndim)
        self.register_buffer("inv_perm", inv_perm_)
        self.register_buffer("scale", torch.ones(ndim) if scale is None else scale)

    def forward(self, num_samples=1, context=None):
        z = self.sample(num_samples)
        return z, self.log_prob(z)

    def sample(self, num_samples=1, context=None):
        eps_u = torch.rand((num_samples, len(self.ind)), dtype=self.scale.dtype, device=self.scale.device) - 0.5
        eps_g = torch.randn((num_samples, len(self.ind_)), dtype=self.scale.dtype, device=self.scale.device)
        z = torch.cat((eps_u, eps_g), -1)
        return self.scale * z[..., self.inv_perm]

    def log_prob(self, z, context=None):
        z = require_cuda_f32(z)
        const = -torch.sum(torch.log(self.scale[self.ind]))
        if len(self.ind_) == 0:
            return const.expand(z.shape[0]).to(torch.float32)
        zg = z[:, self.ind_].contiguous()
        ls = torch.log(self.scale[self.ind_]).float().reshape(-1, 1)
        return gaussian_table_log_prob(zg, torch.zeros_like(ls), ls, None, 1) + const


class ClassCondDiagGaussian(BaseDistribution):
    """Class-conditional diagonal Gaussian (reference: distributions/base.py:281-344); `log_prob(z, y)` with
    integer labels runs in csrc/nfb_glow.cu."""

    def __init__(self, shape, num_classes):
        super().__init__()
        if isinstance(shape, int):
            shape = (shape,)
        shape = tuple(shape)
        self.shape, self.n_dim, self.d, self.num_classes = shape, len(shape), int(np.prod(shape)), num_classes
        self.loc = nn.Parameter(torch.zeros(*shape, num_classes))
        self.log_scale = nn.Parameter(torch.zeros(*shape, num_classes))
        self.temperature = None

    def forward(self, num_samples=1, y=None):
        """distributions/base.py:302-325: z = loc[..., y] + exp(log_scale[..., y]) * eps and its log-density.
        The random draws (labels, eps) and the per-class parameter gather are torch device ops (plumbing; the
        reference's generator stream cannot be reproduced anyway), the density is the CUDA kernel."""
        dev = self.loc.device
        if y is not None:
            num_samples = len(y)
            y = _labels(y, dev)
        else:
            y = torch.randint(self.num_classes, (num_samples,), device=dev)
        with torch.no_grad():
            eps = torch.randn((num_samples,) + self.shape, dtype=self.loc.dtype, device=dev)
            loc = self.loc.detach().movedim(-1, 0)[y]
            log_scale = _tempered(self.log_scale, self.temperature).detach().movedim(-1, 0)[y]
            z = (loc + torch.exp(log_scale) * eps).contiguous()
        return z, self.log_prob(z, y)

    def log_prob(self, z, y):
        z = require_cuda_f32(z)
        K, ls = self.num_classes, _tempered(self.log_scale, self.temperature)
        return gaussian_table_log_prob(z, self.loc.reshape(self.d, K), ls.reshape(self.d, K), _labels(y, z.device), 1)


class ConditionalDiagGaussian(BaseDistribution):
    """Diagonal Gaussian whose mean / log-scale come from a context encoder (distributions/base.py:106-155): the
    encoder output's first half is the mean, the second half the log standard deviation.  The per-sample density is a
    row-wise kernel launch on the standardised residual."""

    def __init__(self, shape, context_encoder):
        super().__init__()
        if isinstance(shape, int):
            shape = (shape,)
        shape = tuple(shape)
        self.shape, self.n_dim, self.d = shape, len(shape), int(np.prod(shape))
        self.context_encoder = context_encoder

    def _params(self, context):
        enc = self.context_encoder(context)
        split = enc.shape[-1] // 2
        return enc[..., :split], enc[..., split:]

    def forward(self, num_samples=1, context=None):
        mean, log_scale = self._params(context)
        eps = torch.randn((num_samples,) + self.shape, dtype=mean.dtype, device=mean.device)
        z = mean + torch.exp(log_scale) * eps
        log_p = -0.5 * self.d * np.log(2 * np.pi) - torch.sum(log_scale + 0.5 * eps ** 2, list(range(1, self.n_dim + 1)))
        return z, log_p

    def log_prob(self, z, context=None):
        z = require_cuda_f32(z)
        mean, log_scale = self._params(context)
        # standardise per sample, then the unit-Gaussian density kernel (differentiable in u, so in z and the encoder
        # output); the log-scale term is a row sum
        from .._standalone import UnitGaussianFn
        u = ((z - mean) * torch.exp(-log_scale)).contiguous().reshape(z.shape[0], -1)
        out = UnitGaussianFn.apply(u)
        return out - torch.sum(log_scale.reshape(z.shape[0], -1), dim=1)


class GlowBase(BaseDistribution):
    """Base distribution of the Glow model (reference: distributions/base.py:347-471): diagonal Gaussian with one mean
    and one log-scale per CHANNEL (`loc * exp(loc_logs * f)`, `log_scale * exp(log_scale_logs * f)`), optionally shifted
    per class (`loc_cc`, `log_scale_cc`).  The per-channel / per-class parameter tables are a few hundred numbers and are
    assembled with torch on the device (parameter preparation, like the reference); the density of the batch is the CUDA
    kernel (csrc/nfb_kernels.cu diag_gauss_kernel / csrc/nfb_glow.cu class-conditional twin)."""

    def __init__(self, shape, num_classes=None, logscale_factor=3.0):
        super().__init__()
        if isinstance(shape, int):
            shape = (shape,)
        shape = tuple(shape)
        self.shape, self.n_dim = shape, len(shape)
        self.num_pix = int(np.prod(shape[1:]))
        self.d = int(np.prod(shape))
        self.num_classes = num_classes
        self.class_cond = num_classes is not None
        self.logscale_factor = logscale_factor
        one = (1, shape[0]) + (1,) * (self.n_dim - 1)
        self.loc = nn.Parameter(torch.zeros(*one))
        self.loc_logs = nn.Parameter(torch.zeros(*one))
        self.log_scale = nn.Parameter(torch.zeros(*one))
        self.log_scale_logs = nn.Parameter(torch.zeros(*one))
        if self.class_cond:
            self.loc_cc = nn.Parameter(torch.zeros(num_classes, shape[0]))
            self.log_scale_cc = nn.Parameter(torch.zeros(num_classes, shape[0]))
        self.temperature = None

    def _channel_params(self):
        """([1, C] or [K, C]) mean and log-scale per channel (per class), base.py:397-424 / 438-461."""
        loc = (self.loc * torch.exp(self.loc_logs * self.logscale_factor)).reshape(1, -1)
        ls = (self.log_scale * torch.exp(self.log_scale_logs * self.logscale_factor)).reshape(1, -1)
        if self.class_cond:
            loc = loc + self.loc_cc
            ls = ls + self.log_scale_cc
        return loc, _tempered(ls, self.temperature)

    def forward(self, num_samples=1, y=None):
        dev = self.loc.device
        view = (-1, self.shape[0]) + (1,) * (self.n_dim - 1)
        with torch.no_grad():
            loc, ls = self._channel_params()
            if self.class_cond:
                if y is not None:
                    num_samples = len(y)
                    y = _labels(y, dev)
                else:
                    y = torch.randint(self.num_classes, (num_samples,), device=dev)
                loc, ls = loc[y], ls[y]                                     # [B, C]
            eps = torch.randn((num_samples,) + self.shape, dtype=self.loc.dtype, device=dev)
            z = (loc.reshape(view) + torch.exp(ls.reshape(view)) * eps).contiguous()
        return z, self.log_prob(z, y)

    def log_prob(self, z, y=None):
        z = require_cuda_f32(z)
        loc, ls = self._channel_params()   # tables [C, K]: element i of a sample uses channel i // num_pix
        return gaussian_table_log_prob(z, loc.t(), ls.t(), _labels(y, z.device) if self.class_cond else None,
                                       self.num_pix)
