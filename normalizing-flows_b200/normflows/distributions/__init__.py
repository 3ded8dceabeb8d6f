from .base import (BaseDistribution, DiagGaussian, ClassCondDiagGaussian, ConditionalDiagGaussian, GlowBase,
                   UniformGaussian)
from .target import Target, TwoMoons
