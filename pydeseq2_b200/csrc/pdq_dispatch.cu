// pdq_dispatch.cu -- routes a launch to the translation unit that owns the design's width.
//
// pdq_kernels.cu holds the per-gene kernels and is compiled once for p = 1..8 (p x p algebra unrolled in registers) and once per
// wide width p = 9..16 (same source, the small matrices in local memory): see the note at the top of that file and
// pydeseq2_b200/build.py.  Every unit exports its launchers under a suffixed name; the per-gene launchers declared in
// pdq_internal.h live here (those that do not depend on the design width are in pdq_common.cu).  Designs of 17..128
// columns (only created on contexts that opted in: 65..128 columns are a second opt-in) go to pdq_wide.cu's launchers (`_wide`),
// which pick the team width from the design.  The fused MAP -> LFC pair has none and reports PDQ_ERR_UNSUPPORTED for them;
// apeGLM shrinkage reaches its wide launcher only on a context that also opted in to wide shrinkage (pdq_set_wide_shrink,
// checked in pdq_api.cu), and above PDQ_MAX_P_WIDE columns only with large shrinkage on as well (pdq_set_large_shrink).
#include "pdq_internal.h"

namespace pdq {

#define PDQ_UNITS(X) X(_p1to8) X(_p9) X(_p10) X(_p11) X(_p12) X(_p13) X(_p14) X(_p15) X(_p16)

#define PDQ_ROUTE(name, p, ...)                                   \
    switch (p) {                                                  \
        case 1: case 2: case 3: case 4: case 5: case 6: case 7:   \
        case 8: return name##_p1to8(__VA_ARGS__);                 \
        case 9: return name##_p9(__VA_ARGS__);                    \
        case 10: return name##_p10(__VA_ARGS__);                  \
        case 11: return name##_p11(__VA_ARGS__);                  \
        case 12: return name##_p12(__VA_ARGS__);                  \
        case 13: return name##_p13(__VA_ARGS__);                  \
        case 14: return name##_p14(__VA_ARGS__);                  \
        case 15: return name##_p15(__VA_ARGS__);                  \
        case 16: return name##_p16(__VA_ARGS__);                  \
        default: return PDQ_ERR_UNSUPPORTED;                      \
    }

#define PDQ_ROUTE_WIDE(name, p, ...)                                                                     \
    if ((p) > PDQ_MAX_P) return (p) <= PDQ_MAX_P_LARGE ? name##_wide(__VA_ARGS__) : PDQ_ERR_UNSUPPORTED; \
    PDQ_ROUTE(name, p, __VA_ARGS__)

#define PDQ_UNITS_ALL(X) PDQ_UNITS(X) X(_wide)

#define DECL_LIN(sfx) int launch_lin_reg_mu##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, double, double*, int64_t);
PDQ_UNITS_ALL(DECL_LIN)
int launch_lin_reg_mu(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_mu, double* mu_out,
                      int64_t ld_out) {
    PDQ_ROUTE_WIDE(launch_lin_reg_mu, d.p, c, d, counts, ld, G, min_mu, mu_out, ld_out)
}

#define DECL_IRLS(sfx)                                                                                                           \
    int launch_irls##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, const double*, const IrlsHost&, double*, \
                         double*, double*, int64_t, double*, int*, int*, const WaldHost*);
PDQ_UNITS_ALL(DECL_IRLS)
int launch_irls(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* disp, const IrlsHost& prm,
                double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status, int* n_fallback, const WaldHost* wald) {
    PDQ_ROUTE_WIDE(launch_irls, d.p, c, d, counts, ld, G, disp, prm, beta, mu, hat, ld_out, conv, status, n_fallback, wald)
}

#define DECL_ALPHA(sfx)                                                                                                          \
    int launch_alpha_mle##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, const double*, int64_t, const double*, \
                              double, double, double, const double*, int, int, double*, double*, int*, const double*, double*);
PDQ_UNITS_ALL(DECL_ALPHA)
int launch_alpha_mle(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, int64_t ld_mu,
                     const double* alpha_hat, double min_disp, double max_disp, double prior_var, const double* prior_var_dev, int cr_reg,
                     int prior_reg, double* alpha, double* conv, int* status, const double* hint_in, double* hint_out) {
    PDQ_ROUTE_WIDE(launch_alpha_mle, d.p, c, d, counts, ld, G, mu, ld_mu, alpha_hat, min_disp, max_disp, prior_var, prior_var_dev, cr_reg,
              prior_reg, alpha, conv, status, hint_in, hint_out)
}

#define DECL_TAIL(sfx) \
    int launch_map_irls##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, const TailHost&, const IrlsHost&, const WaldHost&);
PDQ_UNITS(DECL_TAIL)
int launch_map_irls(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const TailHost& t, const IrlsHost& prm,
                    const WaldHost& wald) {
    PDQ_ROUTE(launch_map_irls, d.p, c, d, counts, ld, G, t, prm, wald)
}

#define DECL_WALD(sfx)                                                                                                         \
    int launch_wald##sfx(const LaunchCfg&, const DesignDev&, const double*, const double*, const double*, int64_t, int, const double*, \
                         const double*, double, int, double*, double*, double*);
PDQ_UNITS_ALL(DECL_WALD)
int launch_wald(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, const double* mu, int64_t ld_mu, int G,
                const double* ridge, const double* contrast, double lfc_null, int alt, double* pv, double* stat, double* se) {
    PDQ_ROUTE_WIDE(launch_wald, d.p, c, d, disp, lfc, mu, ld_mu, G, ridge, contrast, lfc_null, alt, pv, stat, se)
}

#define DECL_WALDK(sfx)                                                                                                \
    int launch_wald_contrasts##sfx(const LaunchCfg&, const DesignDev&, const double*, const double*, int, const double*, int, \
                                   const double*, double*, double*, double*, int64_t);
PDQ_UNITS_ALL(DECL_WALDK)
int launch_wald_contrasts(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, int G, const double* ridge, int K,
                          const double* tab, double* pv, double* stat, double* se, int64_t ld_out) {
    PDQ_ROUTE_WIDE(launch_wald_contrasts, d.p, c, d, disp, lfc, G, ridge, K, tab, pv, stat, se, ld_out)
}

#define DECL_ROUGH(sfx) int launch_rough##sfx(const LaunchCfg&, const DesignDev&, const double*, int64_t, int, double*);
PDQ_UNITS_ALL(DECL_ROUGH)
int launch_rough(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha) {
    PDQ_ROUTE_WIDE(launch_rough, d.p, c, d, normed, ld, G, alpha)
}

#define DECL_MOMENTS(sfx) int launch_moments##sfx(const LaunchCfg&, const DesignDev&, const double*, int64_t, int, double*, double*);
PDQ_UNITS_ALL(DECL_MOMENTS)
int launch_moments(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha, double* all_zero) {
    PDQ_ROUTE_WIDE(launch_moments, d.p, c, d, normed, ld, G, alpha, all_zero)
}

#define DECL_MOM(sfx)                                                                                                       \
    int launch_mom_from_counts##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, double, double, double*, \
                                    double*, double, double*, int64_t);
PDQ_UNITS_ALL(DECL_MOM)
int launch_mom_from_counts(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_disp,
                           double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat, int64_t ld_mu) {
    PDQ_ROUTE_WIDE(launch_mom_from_counts, d.p, c, d, counts, ld, G, min_disp, max_disp, alpha, normed_mean, min_mu, mu_hat, ld_mu)
}

#define DECL_MOMALPHA(sfx)                                                                                                \
    int launch_mom_alpha##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, double, double, double, double*, \
                              double*, double*, int64_t, double*, double*, int*, double*);
PDQ_UNITS(DECL_MOMALPHA)
int launch_mom_alpha(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_disp, double max_disp,
                     double min_mu, double* mom, double* normed_mean, double* mu_hat, int64_t ld_mu, double* alpha, double* conv,
                     int* status, double* hint_out) {
    if (d.p > PDQ_MAX_P) {  // the wide-design kernels have no fold: the two launches, same results
        const int n1 = launch_mom_from_counts(c, d, counts, ld, G, min_disp, max_disp, mom, normed_mean, min_mu, mu_hat, ld_mu);
        if (n1 < 0) return n1;
        const int n2 = launch_alpha_mle(c, d, counts, ld, G, mu_hat, ld_mu, mom, min_disp, max_disp, 1.0, nullptr, 1, 0, alpha, conv,
                                        status, nullptr, hint_out);
        return n2 < 0 ? n2 : n1 + n2;
    }
    PDQ_ROUTE(launch_mom_alpha, d.p, c, d, counts, ld, G, min_disp, max_disp, min_mu, mom, normed_mean, mu_hat, ld_mu, alpha, conv, status,
              hint_out)
}

#define DECL_MULFC(sfx) int launch_mu_from_lfc##sfx(const LaunchCfg&, const DesignDev&, const double*, int, double*, int64_t);
PDQ_UNITS_ALL(DECL_MULFC)
int launch_mu_from_lfc(const LaunchCfg& c, const DesignDev& d, const double* lfc, int G, double* mu, int64_t ld_out) {
    PDQ_ROUTE_WIDE(launch_mu_from_lfc, d.p, c, d, lfc, G, mu, ld_out)
}

#define DECL_COOKS(sfx)                                                                                                          \
    int launch_cooks##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, const double*, const double*, int64_t, \
                          double, double*, int64_t, double*, double*, double*, double*);
PDQ_UNITS_ALL(DECL_COOKS)
int launch_cooks(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                 int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced, double* ws) {
    PDQ_ROUTE_WIDE(launch_cooks, d.p, c, d, counts, ld, G, mu, hat, ld2, cutoff, cooks, ld_out, disp, outlier, replaced, ws)
}

#define DECL_SHRINK(sfx)                                                                                                      \
    int launch_lfc_shrink##sfx(const LaunchCfg&, const DesignDev&, const int64_t*, int64_t, int, const double*, double, double, \
                               int, double*, double*, double*, int*);
PDQ_UNITS_ALL(DECL_SHRINK)
int launch_lfc_shrink(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* size,
                      double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian, double* conv,
                      int* status) {
    PDQ_ROUTE_WIDE(launch_lfc_shrink, d.p, c, d, counts, ld, G, size, prior_no_shrink_scale, prior_scale, shrink_index, beta, inv_hessian,
                   conv, status)
}

}  // namespace pdq
