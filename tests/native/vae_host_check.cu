// Compiles the flow-VAE element math (csrc/nfb_vae.cuh) for the HOST, so that the `not gpu` suite can check the draw,
// the Gaussian density and the Bernoulli likelihood, and their adjoints, against fp64 autograd and central differences.
// Test-only object; the product library never contains or calls this.
#include "../../normalizing-flows_b200/csrc/nfb_vae.cuh"

template <typename T>
static void gauss(int kind, int n, const double* m, const double* p, const double* e, const double* gz,
                  const double* g, double* z, double* nlq, double* g_m, double* g_p, double* dens, double* gd_v,
                  double* gd_m, double* gd_p) {
    for (int i = 0; i < n; ++i) {
        T sd, lsd, t, gm, gsd, gv;
        nfb::vae_std<T>((T)p[i], kind, sd, lsd);
        z[i] = (double)nfb::vae_draw<T>((T)m[i], sd, lsd, (T)e[i], t);
        nlq[i] = (double)t;
        nfb::vae_draw_adjoint<T>(sd, (T)e[i], (T)gz[i], (T)g[i], gm, gsd);
        g_m[i] = (double)gm;
        g_p[i] = (double)(gsd * nfb::vae_dstd<T>(sd, kind));
        // density of the value e[i] under (m, p)
        dens[i] = (double)nfb::vae_density_term<T>((T)e[i], (T)m[i], sd, lsd);
        nfb::vae_density_adjoint<T>((T)e[i], (T)m[i], sd, (T)g[i], gv, gm, gsd);
        gd_v[i] = (double)gv;
        gd_m[i] = (double)gm;
        gd_p[i] = (double)(gsd * nfb::vae_dstd<T>(sd, kind));
    }
}

template <typename T>
static void bern(int n, const double* s, const double* x, double* term, double* ds, double* sig) {
    for (int i = 0; i < n; ++i) {
        term[i] = (double)nfb::vae_bernoulli_term<T>((T)s[i], (T)x[i]);
        ds[i] = (double)nfb::vae_bernoulli_dscore<T>((T)s[i], (T)x[i]);
        sig[i] = (double)nfb::vae_sigmoid<T>((T)s[i]);
    }
}

// elementwise over n entries: the draw z = m + sd e with its share nlq of -log q and its adjoint (cotangents gz of z,
// g of log q) to m and the scale column p; the density share of the value e under (m, p) and its adjoint (cotangent g
// of log p) to e, m and p
extern "C" __attribute__((visibility("default")))
void vae_gauss_check(int kind, int n, int use_float, const double* m, const double* p, const double* e,
                     const double* gz, const double* g, double* z, double* nlq, double* g_m, double* g_p, double* dens,
                     double* gd_v, double* gd_m, double* gd_p) {
    if (use_float) gauss<float>(kind, n, m, p, e, gz, g, z, nlq, g_m, g_p, dens, gd_v, gd_m, gd_p);
    else gauss<double>(kind, n, m, p, e, gz, g, z, nlq, g_m, g_p, dens, gd_v, gd_m, gd_p);
}

// elementwise: the Bernoulli term x log_sig(s) + (1 - x) log_sig(-s), its derivative in s, and sigmoid(s)
extern "C" __attribute__((visibility("default")))
void vae_bernoulli_check(int n, int use_float, const double* s, const double* x, double* term, double* ds,
                         double* sig) {
    if (use_float) bern<float>(n, s, x, term, ds, sig);
    else bern<double>(n, s, x, term, ds, sig);
}
