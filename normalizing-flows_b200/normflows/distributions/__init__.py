from .base import (BaseDistribution, DiagGaussian, ClassCondDiagGaussian, ConditionalDiagGaussian, GaussianMixture,
                   GlowBase, UniformGaussian)
from .encoder import BaseEncoder, Dirac, Uniform, NNDiagGaussian
from .decoder import BaseDecoder, NNDiagGaussianDecoder, NNBernoulliDecoder
from .prior import TwoModes, Sinusoidal, Sinusoidal_gap, Sinusoidal_split, Smiley
from .target import Target, TwoIndependent, TwoMoons
from .mh_proposal import MHProposal, DiagGaussianProposal
from .linear_interpolation import LinearInterpolation
