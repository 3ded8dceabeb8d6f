// Compiles the MAF density-pass element adjoint (csrc/nfb_maf_bwd.cuh maf_affine_adjoint) for the HOST, so that the
// `not gpu` suite can check it against fp64 autograd and finite differences.  Test-only object; the product library
// never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_maf_bwd.cuh"

template <typename T>
static void run(int n, const double* x, const double* u, const double* shift, const double* lam, const double* gld,
                double* pbar_u, double* pbar_shift, double* gx) {
    for (int i = 0; i < n; ++i) {
        T gu, gs, g;
        nfb::maf_affine_adjoint<T>((T)x[i], (T)u[i], (T)shift[i], (T)lam[i], (T)gld[i], gu, gs, g);
        pbar_u[i] = gu; pbar_shift[i] = gs; gx[i] = g;
    }
}

extern "C" __attribute__((visibility("default")))
void maf_adjoint_check(int n, int use_float, const double* x, const double* u, const double* shift, const double* lam,
                       const double* gld, double* pbar_u, double* pbar_shift, double* gx) {
    if (use_float) run<float>(n, x, u, shift, lam, gld, pbar_u, pbar_shift, gx);
    else run<double>(n, x, u, shift, lam, gld, pbar_u, pbar_shift, gx);
}
