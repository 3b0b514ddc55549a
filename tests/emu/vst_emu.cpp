// vst_emu.cpp -- HOST EMULATOR of the variance-stabilising transform kernels.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the per-element function of k_vst_transform (pydeseq2_b200/csrc/pdq_vst.cuh) and the median selection of
// k_size_factor_median (pdq_trend.cuh) -- the exact sources of the sm_90a kernels -- with g++, so that the CPU test-suite can
// check them against the reference's numpy expressions.  Built by tests/emu/vst_ops.py into tests/emu/_build/.
#include <stdint.h>

#include <vector>

#include "../../pydeseq2_b200/csrc/pdq_trend.cuh"
#include "../../pydeseq2_b200/csrc/pdq_vst.cuh"

using namespace pdq;

extern "C" {

int emu_vst_transform(const int64_t* counts, int64_t ld, int N, int G, const double* sf, int kind, double c0, double c1, double* out,
                      int64_t ld_out) {
    if (kind != kVstParametric && kind != kVstMean) return -2;
    const VstParams prm{kind, c0, c1};
    for (int n = 0; n < N; ++n)
        for (int g = 0; g < G; ++g) out[(size_t)n * ld_out + g] = vst_value(counts[(size_t)n * ld + g], sf[n], prm);
    return 0;
}

// held-out size factors with the device's selection code (k_size_factor_median on the caller's log means, one "thread")
int emu_size_factors_from_logmeans(const int64_t* counts, int64_t ld, int N, int G, const double* lm, double* sf) {
    std::vector<double> row((size_t)G);
    unsigned hist[514];
    SerialReducer red;
    for (int n = 0; n < N; ++n) {
        size_t cnt = 0;
        for (int g = 0; g < G; ++g) {
            bool keep;
            row[g] = log_ratio_entry(counts[(size_t)n * ld + g], lm[g], keep);
            cnt += keep;
        }
        sf[n] = exp(median_of(red, row.data(), (size_t)G, cnt, false, 0.0, hist));
    }
    return 0;
}

}  // extern "C"
