"""Shared by tests/golden/make_affine_fkl_grads.py (run against the reference) and tests/test_affine_fkl_training.py
(run against this package): the models and stored inputs of the forward-KL cases of the affine family.  `nf` is whichever
package is passed in; only constructor arguments the reference and this package share are used."""
import torch

import helpers_affine_rkl as A
import helpers_rkl as R

CASES = ["colab", "realnvp", "every", "mixed", "cond"]
SEEDS = {"colab": 31, "realnvp": 32, "every": 33, "mixed": 34, "cond": 35}
DIMS = {"colab": 2, "realnvp": 2, "every": 5, "mixed": 2, "cond": 2}
# perturbation of the weights off their init: 32 blocks at 0.05 overflow the log-det in float32 and in the reference
SIGMA = {"colab": 0.01}


def colab(nf, num_layers=32):
    """examples/real_nvp_colab.ipynb (and the first model of change_base_distribution.ipynb) as written."""
    base = nf.distributions.base.DiagGaussian(2)
    flows = []
    for i in range(num_layers):
        param_map = nf.nets.MLP([1, 64, 64, 2], init_zeros=True)
        flows.append(nf.flows.AffineCouplingBlock(param_map))
        flows.append(nf.flows.Permute(2, mode='swap'))
    return nf.NormalizingFlow(base, flows)


def build(nf, name):
    if name == "colab":
        torch.manual_seed(SEEDS[name])
        return colab(nf)
    if name == "realnvp":
        return A.build(nf, "m")
    if name == "every":
        return A.build(nf, "p")
    if name == "cond":
        return A.build(nf, "q")
    torch.manual_seed(SEEDS[name])   # mixed: affine groups on both sides of a spline block + LU pair
    b = torch.Tensor([1, 0])
    flows = [nf.flows.MaskedAffineFlow(b, nf.nets.MLP([2, 8, 2]), nf.nets.MLP([2, 8, 2], leaky=0.2)), nf.flows.ActNorm(2),
             nf.flows.AutoregressiveRationalQuadraticSpline(2, 1, 32), nf.flows.LULinearPermute(2),
             nf.flows.AffineCouplingBlock(nf.nets.MLP([1, 16, 2]), True, "sigmoid"), nf.flows.Permute(2, "swap")]
    return nf.NormalizingFlow(nf.distributions.DiagGaussian(2), flows)


def data(name, n=512):
    """The stored inputs x of case `name` (float32): standard normal draws scaled to the two-moons range."""
    g = torch.Generator().manual_seed(200 + SEEDS[name])
    return 1.5 * torch.randn(n, DIMS[name], generator=g)


def context_of(n=512):
    return R.context_of(n)


mark_actnorm_done = A.mark_actnorm_done
