// Compiles the generalised spline adjoint (csrc/nfb_spline_bwd.cuh rqs_adjoint_params: any K <= 32, linear /
// circular / per-feature tails) for the HOST, so that the `not gpu` suite can check it against fp64 autograd and
// finite differences.  Test-only object; the product library never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_spline_bwd.cuh"
void nfb_set_error(const char*, ...) {}

template <typename T>
static void run(int n, int K, int nd, const int* circ, const double* x, const double* p, double wh, const double* tail,
                const double* gy, const double* gl, double* y, double* lad, double* gx, double* gp) {
    const int P = 2 * K + nd;
    for (int i = 0; i < n; ++i) {
        T pp[3 * 32 + 1], g[3 * 32 + 1], yy, ll, gxx;
        for (int k = 0; k < P; ++k) pp[k] = (T)p[(size_t)i * P + k];
        nfb::rqs_adjoint_params<32, T>(K, nd, circ[i] != 0, (T)x[i], pp, (T)wh, (T)tail[i], (T)gy[i], (T)gl[i], yy, ll,
                                       gxx, g);
        y[i] = yy; lad[i] = ll; gx[i] = gxx;
        for (int k = 0; k < P; ++k) gp[(size_t)i * P + k] = g[k];
    }
}

extern "C" __attribute__((visibility("default")))
void spline_adjoint_check(int n, int K, int nd, const int* circ, const double* x, const double* p, double wh,
                          const double* tail, const double* gy, const double* gl, int use_float, double* y, double* lad,
                          double* gx, double* gp) {
    if (use_float) run<float>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
    else run<double>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
}
