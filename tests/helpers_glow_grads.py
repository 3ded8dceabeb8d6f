"""The seeded projections of the Glow gradient goldens (tests/golden/make_glow_grads.py), shared by the minting script
and tests/test_glow_training.py."""
import hashlib

import numpy as np
import torch


def grad_projections(name, shape):
    """(v [prod(shape[1:])], u [shape[0]]) fp64 draws: the goldens store G v and u G with G = the gradient reshaped to
    [shape[0], -1]; seeded by the parameter name, so the order of the parameters does not matter."""
    g = torch.Generator().manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:8], 16))
    rest = int(np.prod(shape[1:])) if len(shape) > 1 else 1
    return (torch.randn(rest, generator=g, dtype=torch.float64), torch.randn(shape[0], generator=g, dtype=torch.float64))
