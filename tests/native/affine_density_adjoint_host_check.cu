// Compiles the affine family's density-direction element adjoints (csrc/nfb_affine_bwd.cuh) for the HOST, so that the
// `not gpu` suite can check them against fp64 autograd and central differences.  Test-only object; the product library
// never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_affine_bwd.cuh"

template <typename T>
static void run(int op, int scale, int smap, int n, const double* a, const double* b, const double* c, const double* d,
                const double* g, const double* gam, double* o0, double* o1, double* o2) {
    for (int i = 0; i < n; ++i) {
        T r0, r1, r2;
        if (op == 0) nfb::masked_affine_density_adjoint<T>((T)a[i], (T)b[i], (T)c[i], (T)d[i], (T)g[i], (T)gam[i], r0, r1, r2);
        else if (op == 1) nfb::affine_const_density_adjoint<T>((T)a[i], (T)c[i], (T)d[i], (T)g[i], (T)gam[i], r0, r1, r2);
        else nfb::coupling_density_adjoint<T>(scale, smap, (T)a[i], (T)b[i], (T)c[i], (T)g[i], (T)gam[i], r0, r1, r2);
        o0[i] = r0; o1[i] = r1; o2[i] = r2;
    }
}

// op 0 masked  : (a, b, c, d) = (z, b, s, t)     -> (s_hat, t_hat, g_z direct)
// op 1 const   : (a, c, d) = (z, s, t)           -> (g_z, cs, ct)
// op 2 coupling: (a, b, c) = (v, shift, sc)      -> (g_v, g_shift, g_sc)
extern "C" __attribute__((visibility("default")))
void affine_density_adjoint_check(int op, int scale, int smap, int n, int use_float, const double* a, const double* b,
                                  const double* c, const double* d, const double* g, const double* gam, double* o0,
                                  double* o1, double* o2) {
    if (use_float) run<float>(op, scale, smap, n, a, b, c, d, g, gam, o0, o1, o2);
    else run<double>(op, scale, smap, n, a, b, c, d, g, gam, o0, o1, o2);
}
