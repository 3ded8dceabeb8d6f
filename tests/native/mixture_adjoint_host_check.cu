// Compiles the Gaussian-mixture element math (csrc/nfb_mixture.cuh) for the HOST, so that the `not gpu` suite can check
// the log-density and its adjoint against fp64 autograd and central differences.  Test-only object; the product library
// never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_mixture.cuh"

#include <vector>

template <typename T>
static void run(int K, int D, int n, const double* z, const double* mu, const double* ls, const double* ws,
                const double* g, double* lp, double* gz, double* gmu, double* gls, double* gws) {
    std::vector<T> m(K * D), l(K * D), w(K), zr(D), gzr(D), gm(K * D, (T)0), gl(K * D, (T)0), gw(K, (T)0);
    for (int i = 0; i < K * D; ++i) { m[i] = (T)mu[i]; l[i] = (T)ls[i]; }
    for (int k = 0; k < K; ++k) w[k] = (T)ws[k];
    for (int r = 0; r < n; ++r) {
        for (int d = 0; d < D; ++d) zr[d] = (T)z[r * D + d];
        lp[r] = (double)nfb::mixture_row_log_prob<T>(zr.data(), m.data(), l.data(), w.data(), K, D);
        nfb::mixture_row_adjoint<T>(zr.data(), m.data(), l.data(), w.data(), K, D, (T)g[r], gzr.data(), gm.data(),
                                    gl.data(), gw.data());
        for (int d = 0; d < D; ++d) gz[r * D + d] = (double)gzr[d];
    }
    for (int i = 0; i < K * D; ++i) { gmu[i] = (double)gm[i]; gls[i] = (double)gl[i]; }
    for (int k = 0; k < K; ++k) gws[k] = (double)gw[k];
}

// rows z [n, D], loc / log_scale [K, D], weight_scores [K], row cotangents g [n] -> log p [n], g_z [n, D] and the
// parameter gradients summed over the rows
extern "C" __attribute__((visibility("default")))
void mixture_adjoint_check(int K, int D, int n, int use_float, const double* z, const double* mu, const double* ls,
                           const double* ws, const double* g, double* lp, double* gz, double* gmu, double* gls,
                           double* gws) {
    if (use_float) run<float>(K, D, n, z, mu, ls, ws, g, lp, gz, gmu, gls, gws);
    else run<double>(K, D, n, z, mu, ls, ws, g, lp, gz, gmu, gls, gws);
}
