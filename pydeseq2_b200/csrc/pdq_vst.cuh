// pdq_vst.cuh -- per-element variance-stabilising transform (DeseqDataSet.vst_transform, dds.py:438-514).
// Compiled for the device (k_vst_transform) and for the host emulator of the test-suite (same source).
//
// q = y / sf is a true IEEE division, not a multiply by 1/sf, so that q is bit-identical to the reference's normed_counts
// (`X / size_factors`, dds.py:676-678); the operations are grouped as numpy evaluates the reference's expressions, and the
// transcendentals are the libdevice / libm ones (log2, asinh, sqrt), not the table-driven fast logarithm of pdq_fast.cuh.
#pragma once

#include <math.h>
#include <stdint.h>

#include "pdq_math.cuh"

namespace pdq {

enum { kVstParametric = 0, kVstMean = 1 };

// kind kVstParametric: c0 = a0, c1 = a1 of the dispersion trend a0 + a1 / mean (uns["vst_trend_coeffs"]);
// kind kVstMean: c0 = the trimmed mean of the genewise dispersions (dds.py:503-505), c1 unused
struct VstParams {
    int kind;
    double c0, c1;
};

PDQ_HD double vst_value(int64_t y, double sf, const VstParams& p) {
    const double q = (double)y / sf;
    if (p.kind == kVstParametric) {
        // log2((1 + a1 + 2 a0 q + 2 sqrt(a0 q (1 + a1 + a0 q))) / (4 a0))   (dds.py:492-501)
        const double a0 = p.c0, k1 = 1.0 + p.c1;
        return log2((k1 + (2.0 * a0) * q + 2.0 * sqrt((a0 * q) * (k1 + a0 * q))) / (4.0 * a0));
    }
    // (2 asinh(sqrt(d q)) - log d - log 4) / log 2   (dds.py:502-510)
    const double d = p.c0;
    return (2.0 * asinh(sqrt(d * q)) - log(d) - log(4.0)) / log(2.0);
}

}  // namespace pdq
