// padj_emu.cpp -- HOST EMULATOR of pdq_padj_rejections / pdq_padj_bh.  TEST INFRASTRUCTURE ONLY.
//
// Compiles pydeseq2_b200/csrc/pdq_padj.cuh (the exact source the sm_90a kernels of pdq_padj.cu are built from: np.quantile's
// linear method, scipy's BH value, the comparison with alpha, the clip) with g++, and puts std::sort where the device has its
// radix sort -- ties in p cannot change any output.  The same statuses as the C ABI: -2 for bad shapes or a p-value outside
// [0, 1].  Built by tests/emu/padj_emu.py into tests/emu/_build/ and loaded only by tests/.
#include <math.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "../../pydeseq2_b200/csrc/pdq_padj.cuh"

using namespace pdq;

namespace {
bool args_bad(const double* pv, int64_t ld, int K, int G) {
    if (G <= 0 || K <= 0 || ld < G) return true;
    for (int k = 0; k < K; ++k)
        for (int g = 0; g < G; ++g) {
            const double p = pv[k * ld + g];
            if (!std::isnan(p) && !(p >= 0.0 && p <= 1.0)) return true;
        }
    return false;
}

// genes of one row in the set (padj_in_set), by ascending p
std::vector<int> sorted_set(const double* bm, int G, const double* row, double cutoff) {
    std::vector<int> idx;
    for (int g = 0; g < G; ++g)
        if (padj_in_set(row[g], bm[g], cutoff)) idx.push_back(g);
    std::sort(idx.begin(), idx.end(), [&](int a, int b) { return row[a] < row[b]; });
    return idx;
}
}  // namespace

extern "C" {

int emu_padj_rejections(const double* bm, int G, const double* pv, int64_t ld, int K, const double* theta, int n_theta, double alpha,
                        double* cutoffs_out, int* num_rej_out) {
    if (args_bad(pv, ld, K, G) || n_theta <= 0 || n_theta > kPadjMaxTheta) return -2;
    std::vector<double> sorted(bm, bm + G);
    bool any_nan = false;
    for (double v : sorted) any_nan |= std::isnan(v);
    if (!any_nan) std::sort(sorted.begin(), sorted.end());
    for (int i = 0; i < n_theta; ++i) cutoffs_out[i] = quantile_linear(sorted.data(), G, theta[i], any_nan);
    std::vector<uint64_t> mask(G);
    for (int g = 0; g < G; ++g) mask[g] = padj_member_mask(bm[g], cutoffs_out, n_theta);
    for (int k = 0; k < K; ++k) {
        const double* row = pv + k * ld;
        const std::vector<int> idx = sorted_set(bm, G, row, -INFINITY);
        for (int i = 0; i < n_theta; ++i) {
            int64_t m = 0, r = 0;
            int best = 0;
            for (int g : idx) m += (mask[g] >> i) & 1;
            for (int g : idx)
                if ((mask[g] >> i) & 1 && bh_below(row[g], ++r, m, alpha)) best = (int)r;
            num_rej_out[k * n_theta + i] = best;
        }
    }
    return 0;
}

int emu_padj_bh(const double* bm, int G, const double* pv, int64_t ld, int K, const double* cutoff, double* padj_out, int64_t ld_out) {
    if (args_bad(pv, ld, K, G) || ld_out < G) return -2;
    for (int k = 0; k < K; ++k) {
        const double* row = pv + k * ld;
        double* out = padj_out + k * ld_out;
        for (int g = 0; g < G; ++g) out[g] = NAN;
        const std::vector<int> idx = sorted_set(bm, G, row, cutoff[k]);
        const int64_t m = (int64_t)idx.size();
        double run = INFINITY;
        for (int64_t t = m - 1; t >= 0; --t) {
            const double q = bh_value(row[idx[t]], t + 1, m);
            run = q < run ? q : run;
            out[idx[t]] = m > 1 ? clip01(run) : run;
        }
    }
    return 0;
}

}  // extern "C"
