// Compiles the HMC kernels' density element (csrc/nfb_mixture.cuh mixture_row_log_prob_grad: log p and c grad log p
// of one row, the feature loops unrolled over a compile-time bound) for the HOST, so that the `not gpu` suite can check
// it against central differences and the mixture's own row formula.  Test-only object.
#include "../../normalizing-flows_b200/csrc/nfb_mixture.cuh"

// rows z [n, D <= 16], one mixture term loc / log_scale [K, D], weight_scores [K], coefficient c -> log p [n] and
// c grad log p [n, D]
extern "C" __attribute__((visibility("default")))
void stochastic_grad_check(int K, int D, int n, double c, const double* z, const double* mu, const double* ls,
                           const double* ws, double* lp, double* grad) {
    for (int r = 0; r < n; ++r) {
        double g[16] = {0};
        lp[r] = nfb::mixture_row_log_prob_grad<16, double>(z + r * D, D, mu, ls, ws, K, c, g);
        for (int d = 0; d < D; ++d) grad[r * D + d] = g[d];
    }
}
