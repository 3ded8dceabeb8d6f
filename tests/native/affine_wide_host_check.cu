// Compiles the wide affine path's element formulas (csrc/nfb_affine_wide.cuh) for the HOST, so that the `not gpu` suite
// can check them against fp64 torch and the existing adjoints.  Test-only object; the product library never contains or
// calls this.
#include "../../normalizing-flows_b200/csrc/nfb_affine_wide.cuh"

template <typename T>
static void run(int op, int dir, int scale, int smap, int n, const double* a, const double* b, const double* c,
                const double* d, double* x, double* ld) {
    for (int i = 0; i < n; ++i) {
        T r0, r1;
        if (op == 0) nfb::masked_affine_elem<T>(dir, (T)a[i], (T)b[i], (T)c[i], (T)d[i], r0, r1);
        else if (op == 1) nfb::affine_const_elem<T>(dir, (T)a[i], (T)b[i], (T)c[i], r0, r1);
        else nfb::coupling_elem<T>(dir, scale, smap, (T)a[i], (T)b[i], (T)c[i], r0, r1);
        x[i] = r0; ld[i] = r1;
    }
}

// op 0 masked  : (a, b, c, d) = (z, b, s, t)
// op 1 const   : (a, b, c) = (z, s, t)
// op 2 coupling: (a, b, c) = (v, shift, sc)        -> (x, log-det term)
extern "C" __attribute__((visibility("default")))
void affine_wide_elem_check(int op, int dir, int scale, int smap, int n, int use_float, const double* a, const double* b,
                            const double* c, const double* d, double* x, double* ld) {
    if (use_float) run<float>(op, dir, scale, smap, n, a, b, c, d, x, ld);
    else run<double>(op, dir, scale, smap, n, a, b, c, d, x, ld);
}
