from .base import Flow, NativeFlow, Reverse, Composite, zero_log_det_like_z
from .neural_spline import (AutoregressiveRationalQuadraticSpline, CoupledRationalQuadraticSpline,
                            CircularAutoregressiveRationalQuadraticSpline, CircularCoupledRationalQuadraticSpline)
from .mixing import LULinearPermute, Permute, InvertibleAffine
from .autoregressive import Autoregressive, MaskedAffineAutoregressive
from .affine import (AffineConstFlow, ActNorm, MaskedAffineFlow, AffineCouplingBlock, AffineCoupling,
                     Split, Merge)
from .glow import GlowBlock, Invertible1x1Conv, Squeeze, ImageMerge
from .residual import Residual, iResBlock
from .planar import Planar
from .radial import Radial
from .stochastic import MetropolisHastings, HamiltonianMonteCarlo
