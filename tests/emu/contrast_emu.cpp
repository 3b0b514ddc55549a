// contrast_emu.cpp -- HOST EMULATOR of k_wald_contrasts.  TEST INFRASTRUCTURE ONLY.
//
// The whole host emulator (pdq_emu.cpp: the lane team, the design pack, every emu_* entry) plus emu_wald_contrasts, which runs
// wald_contrasts_gene -- the exact source of the sm_90a kernel -- with 1..32 lanes per gene (emu_set_lanes).  Built by
// tests/emu/contrast_ops.py into tests/emu/_build/ as a library of its own, so the emulator the other tests load is unchanged.
#include "pdq_emu.cpp"

extern "C" {

// pdq_wald_contrasts: K contrasts of fitted coefficients, mu built from them (wald_contrasts_gene); outputs (K, ld_out).
// -2 (PDQ_ERR_INVALID) for K <= 0, ld_out < G or an unknown alternative, -3 for p > 16.
int emu_wald_contrasts(const double* X, const double* sf, int N, int p, const double* disp, const double* lfc, int G, const double* ridge,
                       int K, const double* contrasts, const double* lfc_null, const int* alt, double* pv, double* stat, double* se,
                       int64_t ld_out) {
    if (K <= 0 || ld_out < G) return -2;
    std::vector<double> tab((size_t)K * (p + 2));
    for (int k = 0; k < K; ++k) {
        if (alt[k] < 0 || alt[k] > 4) return -2;
        for (int j = 0; j < p; ++j) tab[(size_t)k * (p + 2) + j] = contrasts[(size_t)k * p + j];
        tab[(size_t)k * (p + 2) + p] = lfc_null[k];
        tab[(size_t)k * (p + 2) + p + 1] = (double)alt[k];
    }
    Pack k = make_pack(X, sf, N, p);
    EMU_DISPATCH(p, {
        for (int g = 0; g < G; ++g)
            with_lanes([&](const Group& grp) {
                wald_contrasts_gene<P>(grp, k.d, ridge, disp[g], lfc + (size_t)g * P, K, tab.data(), pv + g, stat + g, se + g, ld_out, true);
            });
    });
    return 0;
}

}  // extern "C"
