// Compiles the planar / radial flows' per-layer constants, element adjoints and parameter chains
// (csrc/nfb_planar_bwd.cuh) for the HOST, so that the `not gpu` suite can check them against fp64 autograd and central
// differences.  Test-only object; the product library never contains or calls this.
#include <vector>

#include "../../normalizing-flows_b200/csrc/nfb_planar_bwd.cuh"

#define EXPORT extern "C" __attribute__((visibility("default")))

template <typename T>
static void planar_layer(int act, double slope, int n, int d, const double* z, const double* u, const double* w, double b,
                         const double* g, const double* gam, double* gz, double* gu, double* gw, double* gb,
                         double* consts) {
    std::vector<T> uu(u, u + d), ww(w, w + d), Sz(d, 0), Sg(d, 0), ou(d), ow(d);
    T k, psi, Sc = 0, Se = 0, ob;
    nfb::planar_consts<T>(uu.data(), ww.data(), d, k, psi);
    consts[0] = k; consts[1] = psi;
    for (int r = 0; r < n; ++r) {
        T lin = 0, gdu = 0;
        for (int j = 0; j < d; ++j) { lin += ww[j] * (T)z[r * d + j]; gdu += (T)g[r * d + j] * (uu[j] + k * ww[j]); }
        lin += (T)b;
        T c, hv, e;
        nfb::planar_row_adjoint<T>(act, (T)slope, lin, psi, gdu, (T)gam[r], c, hv, e);
        for (int j = 0; j < d; ++j) {
            gz[r * d + j] = (T)g[r * d + j] + c * ww[j];
            Sz[j] += c * (T)z[r * d + j];
            Sg[j] += hv * (T)g[r * d + j];
        }
        Sc += c; Se += e;
    }
    nfb::planar_param_chain<T>(uu.data(), ww.data(), d, Sz.data(), Sc, Sg.data(), Se, ou.data(), ow.data(), &ob);
    for (int j = 0; j < d; ++j) { gu[j] = ou[j]; gw[j] = ow[j]; }
    *gb = ob;
}

template <typename T>
static void radial_layer(int n, int d, const double* z, const double* z0, double alpha, double beta, const double* g,
                         const double* gam, double* gz, double* gz0, double* gbeta, double* galpha, double* consts) {
    T ah, bh, Sbh = 0, Sah = 0;
    nfb::radial_consts<T>((T)alpha, (T)beta, ah, bh);
    consts[0] = ah; consts[1] = bh;
    std::vector<T> S(d, 0);
    for (int r = 0; r < n; ++r) {
        T r2 = 0, gdot = 0;
        for (int j = 0; j < d; ++j) {
            const T dz = (T)z[r * d + j] - (T)z0[j];
            r2 += dz * dz; gdot += (T)g[r * d + j] * dz;
        }
        T h, cr, gbh, gah;
        nfb::radial_row_adjoint<T>(nfb::pl_sqrt(r2), ah, bh, (T)(d - 1), gdot, (T)gam[r], h, cr, gbh, gah);
        for (int j = 0; j < d; ++j) {
            const T gdz = h * (T)g[r * d + j] + cr * ((T)z[r * d + j] - (T)z0[j]);
            gz[r * d + j] = (T)g[r * d + j] + gdz;
            S[j] += gdz;
        }
        Sbh += gbh; Sah += gah;
    }
    for (int j = 0; j < d; ++j) gz0[j] = -S[j];
    T gb, ga;
    nfb::radial_param_chain<T>((T)alpha, (T)beta, Sbh, Sah, gb, ga);
    *gbeta = gb; *galpha = ga;
}

// one planar layer over n rows: g_z [n, d], g_u, g_w [d], g_b and the constants (k, psi)
EXPORT void planar_layer_check(int use_float, int act, double slope, int n, int d, const double* z, const double* u,
                               const double* w, double b, const double* g, const double* gam, double* gz, double* gu,
                               double* gw, double* gb, double* consts) {
    if (use_float) planar_layer<float>(act, slope, n, d, z, u, w, b, g, gam, gz, gu, gw, gb, consts);
    else planar_layer<double>(act, slope, n, d, z, u, w, b, g, gam, gz, gu, gw, gb, consts);
}

// one radial layer over n rows: g_z [n, d], g_z0 [d], g_beta, g_alpha and the constants (alpha_hat, beta_hat)
EXPORT void radial_layer_check(int use_float, int n, int d, const double* z, const double* z0, double alpha, double beta,
                               const double* g, const double* gam, double* gz, double* gz0, double* gbeta,
                               double* galpha, double* consts) {
    if (use_float) radial_layer<float>(n, d, z, z0, alpha, beta, g, gam, gz, gz0, gbeta, galpha, consts);
    else radial_layer<double>(n, d, z, z0, alpha, beta, g, gam, gz, gz0, gbeta, galpha, consts);
}

// the planar row adjoint alone: (c, h, e) per element
EXPORT void planar_row_check(int use_float, int act, double slope, int n, const double* lin, const double* psi,
                             const double* gu, const double* gam, double* c, double* hv, double* e) {
    for (int i = 0; i < n; ++i) {
        if (use_float) {
            float a, b2, e2;
            nfb::planar_row_adjoint<float>(act, (float)slope, (float)lin[i], (float)psi[i], (float)gu[i], (float)gam[i],
                                           a, b2, e2);
            c[i] = a; hv[i] = b2; e[i] = e2;
        } else {
            nfb::planar_row_adjoint<double>(act, slope, lin[i], psi[i], gu[i], gam[i], c[i], hv[i], e[i]);
        }
    }
}
