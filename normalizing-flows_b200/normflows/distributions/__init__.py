from .base import (BaseDistribution, DiagGaussian, ClassCondDiagGaussian, ConditionalDiagGaussian, GaussianMixture,
                   GlowBase, UniformGaussian)
from .prior import TwoModes, Sinusoidal, Sinusoidal_gap, Sinusoidal_split, Smiley
from .target import Target, TwoIndependent, TwoMoons
