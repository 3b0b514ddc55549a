// sf_emu.cpp -- HOST EMULATOR of the size-factor kernels.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the per-entry functions of k_log_means / k_size_factor_median (log_mean_term, kept_logmean, log_ratio_entry in
// pydeseq2_b200/csrc/pdq_trend.cuh) and the median selection -- the exact sources of the sm_90a kernels -- with g++, one "thread",
// so that the CPU test-suite can check pdq_size_factors_ex (median of ratios and poscounts, over every gene or control genes)
// against the reference.  Built by tests/emu/sf_ops.py into tests/emu/_build/.
#include <stdint.h>

#include <vector>

#include "../../pydeseq2_b200/csrc/pdq_trend.cuh"

using namespace pdq;

extern "C" {

// pdq_size_factors_ex: `control` may be NULL, `logmeans` (G,) receives the raw log means; -2 (PDQ_ERR_INVALID) for an unknown kind
int emu_size_factors_ex(const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control, double* sf, double* logmeans) {
    if (kind != kSfRatio && kind != kSfPoscounts) return -2;
    std::vector<double> kept((size_t)G), row((size_t)G);
    for (int g = 0; g < G; ++g) {  // k_log_means
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += log_mean_term(counts[(size_t)n * ld + g], kind);
        logmeans[g] = s / (double)N;
        kept[g] = kept_logmean(logmeans[g], kind, control == nullptr || control[g] != 0);
    }
    unsigned hist[514];
    SerialReducer red;
    for (int n = 0; n < N; ++n) {  // k_size_factor_median
        size_t cnt = 0;
        for (int g = 0; g < G; ++g) {
            bool keep;
            row[g] = log_ratio_entry(counts[(size_t)n * ld + g], kept[g], keep, kind == kSfPoscounts);
            cnt += keep;
        }
        sf[n] = exp(median_of(red, row.data(), (size_t)G, cnt, false, 0.0, hist));
    }
    if (kind == kSfPoscounts) {  // k_size_factor_geomean
        double s = 0.0;
        for (int n = 0; n < N; ++n) s += log(sf[n]);
        const double gm = exp(s / (double)N);
        for (int n = 0; n < N; ++n) sf[n] = sf[n] / gm;
    }
    return 0;
}

}  // extern "C"
