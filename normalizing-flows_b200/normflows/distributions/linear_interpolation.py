class LinearInterpolation:
    """Linear interpolation of two distributions in log space (reference: distributions/linear_interpolation.py):
    log p = alpha log p_1 + (1 - alpha) log p_2.  Like the reference, a plain object, not a module.  When both are
    native densities (a flat DiagGaussian, a GaussianMixture, or another such interpolation), the HMC and MH layers
    evaluate it inside their kernels (normflows/_stochastic.py)."""

    def __init__(self, dist1, dist2, alpha):
        self.alpha = alpha
        self.dist1 = dist1
        self.dist2 = dist2

    def log_prob(self, z):
        return self.alpha * self.dist1.log_prob(z) + (1 - self.alpha) * self.dist2.log_prob(z)
