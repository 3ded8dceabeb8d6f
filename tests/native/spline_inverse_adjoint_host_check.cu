// Compiles the inverse-spline adjoint (csrc/nfb_spline_bwd.cuh rqs_inverse_adjoint_params) and the forward one it is
// checked against (rqs_adjoint_params) for the HOST, so that the `not gpu` suite can check it in double precision
// against finite differences of the oracle's inverse spline (tests/test_reverse_kld_training.py).  Test-only object;
// the product library never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_spline_bwd.cuh"
void nfb_set_error(const char*, ...) {}

template <bool INV, typename T>
static void run(int n, int K, int nd, const int* circ, const double* x, const double* p, double wh, const double* tail,
                const double* gy, const double* gl, double* y, double* lad, double* gx, double* gp) {
    const int P = 2 * K + nd;
    for (int i = 0; i < n; ++i) {
        T pp[3 * 32 + 1], g[3 * 32 + 1], yy, ll, gxx;
        for (int k = 0; k < P; ++k) pp[k] = (T)p[(size_t)i * P + k];
        if (INV)
            nfb::rqs_inverse_adjoint_params<32, T>(K, nd, circ[i] != 0, (T)x[i], pp, (T)wh, (T)tail[i], (T)gy[i],
                                                   (T)gl[i], yy, ll, gxx, g);
        else
            nfb::rqs_adjoint_params<32, T>(K, nd, circ[i] != 0, (T)x[i], pp, (T)wh, (T)tail[i], (T)gy[i], (T)gl[i], yy,
                                           ll, gxx, g);
        y[i] = yy; lad[i] = ll; gx[i] = gxx;
        for (int k = 0; k < P; ++k) gp[(size_t)i * P + k] = g[k];
    }
}

// inverse = 1: z in x, (x, ld) out in (y, lad), g_z out in gx; inverse = 0: the forward element.
extern "C" __attribute__((visibility("default")))
void spline_inverse_adjoint_check(int n, int K, int nd, const int* circ, const double* x, const double* p, double wh,
                                  const double* tail, const double* gy, const double* gl, int use_float, int inverse,
                                  double* y, double* lad, double* gx, double* gp) {
    if (inverse) {
        if (use_float) run<true, float>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
        else run<true, double>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
    } else {
        if (use_float) run<false, float>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
        else run<false, double>(n, K, nd, circ, x, p, wh, tail, gy, gl, y, lad, gx, gp);
    }
}
