from .base import (BaseDistribution, DiagGaussian, ClassCondDiagGaussian, ConditionalDiagGaussian, GlowBase,
                   UniformGaussian)
from .prior import TwoModes
from .target import Target, TwoIndependent, TwoMoons
