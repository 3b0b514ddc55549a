// math_ops.h -- TEST INFRASTRUCTURE.  One elementwise entry per FP64 primitive of pdq_fast.cuh / pdq_math.cuh and one call of
// the per-gene table builders of pdq_gene.cuh, shared by the GPU probe (pdq_probe.cu, device branches) and the host emulator
// (tests/emu/pdq_emu.cpp, host branches), so that both are driven with the same op codes (tests/math_checks.py: OPS).
#pragma once

#include "../../pydeseq2_b200/csrc/pdq_gene.cuh"

namespace pdq_probe {

enum Op {
    kFastRcp,       // fast_rcp(x)
    kFastDiv,       // fast_div(x, y)
    kFastLog,       // fast_log(x)
    kFastLogNb,     // fast_log_nb(x)
    kFastExp,       // fast_exp(x)
    kFastExpNb,     // fast_exp_nb(x)
    kTlog,          // tlog(x, tab)
    kTlogNb,        // tlog_nb(x, tab)
    kTexp,          // texp(x, tab)
    kTexpNb,        // texp_nb(x, tab)
    kLgamma,        // lgamma_pos(x)
    kDigamma,       // digamma_pos(x)
    kTrigamma,      // trigamma_pos(x)
    kLgDgLg,        // lgamma_digamma_pos(x): the lgamma output
    kLgDgDg,        // lgamma_digamma_pos(x): the digamma output
    kLgammaAsym,    // lgamma_asym(x, y = log x), x >= 10
    kDigammaAsym,   // digamma_asym(x, y = log x), x >= 10
    kTrigammaAsym,  // trigamma_asym(x), x >= 10
    kNormSf,        // norm_sf(x)
    kNumOps
};

PDQ_HD double apply(int op, double x, double y, const double* tab) {
    using namespace pdq;
    double lg, dg;
    switch (op) {
        case kFastRcp: return fast_rcp(x);
        case kFastDiv: return fast_div(x, y);
        case kFastLog: return fast_log(x);
        case kFastLogNb: return fast_log_nb(x);
        case kFastExp: return fast_exp(x);
        case kFastExpNb: return fast_exp_nb(x);
        case kTlog: return tlog(x, tab);
        case kTlogNb: return tlog_nb(x, tab);
        case kTexp: return texp(x, tab);
        case kTexpNb: return texp_nb(x, tab);
        case kLgamma: return lgamma_pos(x);
        case kDigamma: return digamma_pos(x);
        case kTrigamma: return trigamma_pos(x);
        case kLgDgLg: lgamma_digamma_pos(x, lg, dg); return lg;
        case kLgDgDg: lgamma_digamma_pos(x, lg, dg); return dg;
        case kLgammaAsym: return lgamma_asym(x, y);
        case kDigammaAsym: return digamma_asym(x, y);
        case kTrigammaAsym: return trigamma_asym(x);
        case kNormSf: return norm_sf(x);
        default: return __builtin_nan("");
    }
}

// the per-gene tables at r, into `tab` (4 * kPsiK doubles, shared by the lanes of the gene): lgamma(r + k) from
// build_lgamma_table, psi(r + k) from build_psi_table, then psi(r + k) and psi'(r + k) from build_psi_tri_tables
constexpr int kTabOut = 4 * pdq::kPsiK;

PDQ_HD void build_tables(const pdq::Group& grp, double* tab, double r, const double* mtab) {
    pdq::build_lgamma_table(grp, tab, r, mtab);
    pdq::build_psi_table(grp, tab + pdq::kPsiK, r);
    pdq::build_psi_tri_tables(grp, tab + 2 * pdq::kPsiK, r);
}

}  // namespace pdq_probe
