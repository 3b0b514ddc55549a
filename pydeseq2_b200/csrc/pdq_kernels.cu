// pdq_kernels.cu -- sm_90a kernels of the per-gene NB-GLM hot path and their launchers.
//
// Every kernel has the same skeleton (DESIGN.md §3):
//   1. one elected thread stages the design pack (X column-major, size factors, log size factors)
//      from global into shared memory with ONE TMA bulk copy (`cp.async.bulk`, SASS UBLKCP) whose
//      completion is signalled on an mbarrier; all threads wait on the barrier phase;
//   2. each warp owns 32/T adjacent genes, T lanes per gene; lanes stream the gene's samples from
//      the (N, G) sample-major arrays (coalesced across the adjacent genes of the warp, read-only
//      path) and keep all per-gene state (X^T W X, beta, ...) in registers;
//   3. cross-lane sums use xor-butterfly warp shuffles; p x p Cholesky solves run redundantly per lane.
// Tensor cores are deliberately not used: p <= 8, the work is FP64 transcendental + HBM streaming.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "pdq_gene.cuh"
#include "pdq_trend.cuh"
#include "pdq_shrink.cuh"
#include "pdq_internal.h"

// This file is compiled once per RANGE OF DESIGN WIDTHS (pydeseq2_b200/build.py): the base unit (PDQ_TU_P = 0) holds the kernels
// for p = 1..8 -- p x p algebra fully unrolled in registers -- and everything that does not depend on p; one further unit per
// wide design width p = 9..16 (PDQ_TU_P = p) holds that width's kernels, same source, loops over the design columns not
// unrolled.  The units compile in parallel; pdq_dispatch.cu routes a launch to the unit that owns the design's width.
#ifndef PDQ_TU_P
#define PDQ_TU_P 0
#endif
#define PDQ_CAT_(a, b) a##b
#define PDQ_CAT(a, b) PDQ_CAT_(a, b)
#if PDQ_TU_P == 0
#define PDQ_TUFN(name) name##_p1to8
#else
#define PDQ_TUFN(name) PDQ_CAT(name##_p, PDQ_TU_P)
#endif

namespace pdq {
namespace {

constexpr int kBlock = 128;
constexpr int kWarps = kBlock / 32;
// resident blocks per SM the two heavy kernels are compiled for (register cap = 65536 / (128 * blocks)).  The trade-off is set
// by the 64 K-register file per SM, which H100 has too: fewer resident blocks buy registers for the Newton-opening sweep of
// alpha_mle.  scripts/variants_sweep.sh times other values.
#ifndef PDQ_IRLS_MINB
#define PDQ_IRLS_MINB 4
#endif
#ifndef PDQ_ALPHA_MINB
#define PDQ_ALPHA_MINB 3
#endif

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// lookup tables of the table-driven log / exp (pdq_fast.cuh); staged into shared memory by the kernels that use them
__device__ const double g_math_tab[kMathTabLen] = {PDQ_MATH_TABLE_VALUES};
constexpr uint32_t kMathTabBytes = (uint32_t)kMathTabLen * 8u;
static_assert(kMathTabBytes % 16 == 0, "bulk copies are 16-byte granular");

// ---- TMA 1-D bulk copy global -> shared, mbarrier completion --------------------------------------
// Shared-memory layout: [ design pack (when staged) | mbarrier (16 B) | math table (kernels with TAB) | kernel-specific scratch ]
// Packs above the staging limit (pdq_api.cu: they would leave fewer than four blocks per SM) are NOT copied: the kernels then
// read the design rows straight from global memory -- every warp of the machine walks the same <= few-hundred-KB pack, so the
// rows live in L1 / L2 -- and shared memory no longer bounds the number of samples or resident blocks.
struct DesignView {
    const double* pack;
    int N;
    int pack_smem;  // bytes of the pack staged in shared memory; 0 = read it from global memory
};

// MODE: 1 = pack staged (shared-memory pointers, LDS), 0 = pack in global memory, -1 = decided at run time (generic loads)
template <bool TAB, int MODE>
__device__ __forceinline__ DesignS stage_design_t(const DesignView& dv, int P, unsigned char* smem) {
    double* s = reinterpret_cast<double*>(smem);
    const int RS = design_row_stride(P);
    const bool staged = MODE == 1 || (MODE == -1 && dv.pack_smem != 0);
    const uint32_t bytes = staged ? (uint32_t)((dv.N + 1) * RS) * 8u : 0u;  // N sample rows + the row of column maxima
    if (staged || TAB) {
        uint64_t* bar = reinterpret_cast<uint64_t*>(smem + bytes);
        const uint32_t bar_a = smem_u32(bar);
        if (threadIdx.x == 0) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a) : "memory");
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes + (TAB ? kMathTabBytes : 0u))
                         : "memory");
            if (TAB)
                asm volatile(
                    "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                        smem_u32(smem + bytes + 16)),
                    "l"(reinterpret_cast<const unsigned char*>(g_math_tab)), "r"(kMathTabBytes), "r"(bar_a)
                    : "memory");
            // chunked so a single descriptor never exceeds 32 KB; all chunks complete on the same barrier
            uint32_t off = 0;
            while (off < bytes) {
                const uint32_t n = (bytes - off > 32768u) ? 32768u : (bytes - off);
                asm volatile(
                    "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                        smem_u32(smem + off)),
                    "l"(reinterpret_cast<const unsigned char*>(dv.pack) + off), "r"(n), "r"(bar_a)
                    : "memory");
                off += n;
            }
        }
        uint32_t done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(bar_a), "r"(0u)
                : "memory");
        }
    }
    DesignS d;
    if (MODE == 1) d.X = s;
    else if (MODE == 0) d.X = dv.pack;
    else d.X = staged ? s : dv.pack;
    d.sf = d.X + P;
    d.lsf = d.X + P + 1;
    d.N = dv.N;
    d.RS = RS;
    d.mtab = TAB ? reinterpret_cast<const double*>(smem + bytes + 16) : nullptr;
    return d;
}

// the light kernels: staged or not is a run-time property of the design
__device__ __forceinline__ DesignS stage_design(const DesignView& dv, int P, unsigned char* smem) {
    return stage_design_t<false, -1>(dv, P, smem);
}
// offset of the kernel-specific scratch behind the pack + mbarrier (+ table)
__device__ __forceinline__ size_t scratch_off(const DesignView& dv, bool tab) { return (size_t)dv.pack_smem + 16 + (tab ? kMathTabBytes : 0u); }

__device__ __forceinline__ void map_lanes(int lgT, int G, Group& grp, int& gene, bool& valid, int block = -1) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    grp.T = 1 << lgT;
    grp.gpw = 32 >> lgT;
    grp.si = lane >> (5 - lgT);
    const int gi = lane & (grp.gpw - 1);
    const int gidx = ((block < 0 ? (int)blockIdx.x : block) * kWarps + warp) * grp.gpw + gi;
    valid = gidx < G;
    gene = valid ? gidx : (G - 1);
}

// Persistent scheduling for the two heavy kernels: the grid holds as many blocks as fit on the machine and every WARP
// draws gene tiles (32/T adjacent genes) from a global ticket counter until the tiles run out.  Genes differ in
// iteration count, so a static assignment leaves SMs idle at the tail (20 % of the cycles in the first profile).
// The ticket of the NEXT tile is drawn before the current tile is worked on (`ahead`), so the atomic's round trip to L2 is hidden.
__device__ __forceinline__ int draw_ticket(int* ticket) {
    int t = 0;
    if ((threadIdx.x & 31) == 0) t = atomicAdd(ticket, 1);
    return t;  // valid in lane 0; broadcast when consumed
}

// `descending` (experiment, see alpha_descending()): tickets walk the tiles from the last to the first
__device__ __forceinline__ bool next_tile(int* ticket, int lgT, int G, Group& grp, int& gene, bool& valid, int& ahead,
                                          bool descending = false) {
    const int lane = threadIdx.x & 31;
    grp.T = 1 << lgT;
    grp.gpw = 32 >> lgT;
    grp.si = lane >> (5 - lgT);
    int tile = __shfl_sync(0xffffffffu, ahead, 0);
    const int ntiles = (G + grp.gpw - 1) >> (5 - lgT);
    if (tile >= ntiles) return false;
    if (descending) tile = ntiles - 1 - tile;
    ahead = draw_ticket(ticket);
    const int gidx = tile * grp.gpw + (lane & (grp.gpw - 1));
    valid = gidx < G;
    gene = valid ? gidx : (G - 1);
    return true;
}

// ---- kernels --------------------------------------------------------------------------------------
template <int P>
struct LinMuArgs {
    DesignView dv;
    SmallMat<P> pinv;
    const int64_t* counts;
    int64_t ld;
    int G, lgT;
    double min_mu;
    double* mu;
    int64_t ld_out;
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_lin_reg_mu(const __grid_constant__ LinMuArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    linmu_gene<P>(grp, d, a.pinv, a.counts + g, a.ld, a.min_mu, a.mu + g, a.ld_out, valid);
}

template <int P>
struct IrlsArgs {
    DesignView dv;
    SmallMat<P> pinv;
    IrlsParams prm;
    const int64_t* counts;
    int64_t ld;
    int G, lgT;
    const double* disp;
    double *beta, *mu, *hat, *conv;
    int64_t ld_out;
    int* status;
    int* n_fallback;
    int* ticket;  // [0] tile counter of the persistent scheduler, [1] number of genes flagged for the optimiser branch (both
                  // zeroed before the launch)
    int force;    // test hook: flag every gene for the optimiser branch
    int with_wald;         // also the Wald test of the fit (resident pipeline): parameters and outputs below
    WaldParams<P> wald;
    double *wald_p, *wald_stat, *wald_se;
};

template <int P, bool STAGED>
__global__ void __launch_bounds__(kBlock, PDQ_IRLS_MINB) k_irls(const __grid_constant__ IrlsArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design_t<true, STAGED ? 1 : 0>(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    // behind the design pack, its mbarrier and the math table: log(k!) table, then one lgamma(r + k) table per gene of the warp's tile
    double* logfact = reinterpret_cast<double*>(smem + scratch_off(a.dv, true));
    if (threadIdx.x < kPsiK) logfact[threadIdx.x] = kLogFact[threadIdx.x];
    __syncthreads();
    const int gpw = 32 >> a.lgT;
    double* lg_tab = logfact + kPsiK + (size_t)((threadIdx.x >> 5) * gpw + ((threadIdx.x & 31) & (gpw - 1))) * kPsiK;
    int ahead = draw_ticket(a.ticket);
    while (next_tile(a.ticket, a.lgT, a.G, grp, g, valid, ahead)) {
        int st = 0;
        irls_gene<P>(grp, d, a.pinv, a.prm, a.counts + g, a.ld, a.disp[g], a.beta + (int64_t)g * P, a.mu + g, a.hat + g,
                     a.ld_out, a.conv + g, &st, valid, lg_tab, logfact, a.with_wald ? &a.wald : nullptr, a.wald_p + g,
                     a.wald_stat + g, a.wald_se + g);
        if (valid && grp.si == 0) {
            if (a.force) st = kIrlsNeedsOptimizer;
            a.status[g] = st;
            if (st != kIrlsOk) {
                atomicAdd(a.ticket + 1, 1);
                if (a.n_fallback) atomicAdd(a.n_fallback, 1);
            }
        }
    }
}

// optimiser branch for the genes k_irls flagged (utils.py:374-413).  Normally no gene is flagged: the launch is one wave of
// blocks that read the flagged-gene counter and exit; otherwise the blocks stride over the gene tiles and skip those without one.
template <int P>
__global__ void __launch_bounds__(kBlock) k_irls_optimizer(const __grid_constant__ IrlsArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    if (*reinterpret_cast<volatile const int*>(a.ticket + 1) == 0) return;
    const DesignS d = stage_design(a.dv, P, smem);
    const int per_block = kWarps * (32 >> a.lgT), nbt = (a.G + per_block - 1) / per_block;
    for (int bt = blockIdx.x; bt < nbt; bt += gridDim.x) {
        Group grp;
        int g;
        bool valid;
        map_lanes(a.lgT, a.G, grp, g, valid, bt);
        const bool run = valid && a.status[g] == kIrlsNeedsOptimizer;
        if (!__syncthreads_or(run)) continue;
        if (!__any_sync(0xffffffffu, run)) continue;
        irls_optimizer_gene<P>(grp, d, a.pinv, a.prm, a.counts + g, a.ld, a.disp[g], a.beta + (int64_t)g * P, a.mu + g,
                               a.hat + g, a.ld_out, a.conv + g, run, a.with_wald ? &a.wald : nullptr, a.wald_p + g,
                               a.wald_stat + g, a.wald_se + g);
    }
}

template <int P>
struct AlphaArgs {
    DesignView dv;
    AlphaParams prm;
    const int64_t* counts;
    int64_t ld;
    int G, lgT;
    const double* mu;
    int64_t ld_mu;
    const double* alpha_hat;
    double *alpha, *conv;
    int* status;
    const double* prior_var_dev;  // when set, overrides prm.prior_var (written by k_trend_prior on the same stream)
    int* ticket;                  // [0] tile counter of the persistent scheduler, [1] genes flagged for the grid (zeroed before)
    int force;                    // test hook: flag every gene for the grid fallback
    const double* hint_in;        // [G][2] (x*, h*) of the prior-free search on the same counts / means, or nullptr (alpha_gene)
    double* hint_out;             // [G][2] written by this search, or nullptr
    int descending;               // tile order of the persistent scheduler (next_tile)
};

template <int P, bool STAGED>
__global__ void __launch_bounds__(kBlock, PDQ_ALPHA_MINB) k_alpha_mle(const __grid_constant__ AlphaArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design_t<true, STAGED ? 1 : 0>(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    AlphaParams prm = a.prm;
    if (a.prior_var_dev) prm.prior_var = *a.prior_var_dev;
    const int gpw = 32 >> a.lgT;
    // per-gene psi(r + k) and psi'(r + k) tables live behind the design pack and its mbarrier (one slot of 2 * kPsiK doubles
    // per gene of the warp's tile)
    double* psi = reinterpret_cast<double*>(smem + scratch_off(a.dv, true)) +
                  (size_t)((threadIdx.x >> 5) * gpw + ((threadIdx.x & 31) & (gpw - 1))) * (2 * kPsiK);
    int ahead = draw_ticket(a.ticket);
    while (next_tile(a.ticket, a.lgT, a.G, grp, g, valid, ahead, a.descending != 0)) {
        alpha_gene<P>(grp, d, prm, a.counts + g, a.ld, a.mu + g, a.ld_mu, a.alpha_hat[g], a.alpha + g, a.conv + g,
                      a.status + g, valid, psi, a.hint_in ? a.hint_in + 2 * (int64_t)g : nullptr,
                      a.hint_out ? a.hint_out + 2 * (int64_t)g : nullptr);
        if (valid && grp.si == 0) {
            if (a.force) {
                a.status[g] = kAlphaNeedsGrid;
                a.conv[g] = 0.0;
            }
            if (a.status[g] == kAlphaNeedsGrid) atomicAdd(a.ticket + 1, 1);
        }
    }
}

// the reference's grid fallback for the genes k_alpha_mle flagged; same launch scheme as k_irls_optimizer
template <int P>
__global__ void __launch_bounds__(kBlock) k_alpha_grid(const __grid_constant__ AlphaArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    if (*reinterpret_cast<volatile const int*>(a.ticket + 1) == 0) return;
    const DesignS d = stage_design(a.dv, P, smem);
    const int per_block = kWarps * (32 >> a.lgT), nbt = (a.G + per_block - 1) / per_block;
    for (int bt = blockIdx.x; bt < nbt; bt += gridDim.x) {
        Group grp;
        int g;
        bool valid;
        map_lanes(a.lgT, a.G, grp, g, valid, bt);
        const bool run = valid && a.status[g] == kAlphaNeedsGrid;
        if (!__syncthreads_or(run)) continue;
        if (!__any_sync(0xffffffffu, run)) continue;
        alpha_grid_gene<P>(grp, d, a.prm.lo, a.prm.hi, a.counts + g, a.ld, a.mu + g, a.ld_mu, a.alpha + g, run);
    }
}

template <int P>
struct WaldArgs {
    DesignView dv;
    WaldParams<P> prm;
    const double *disp, *lfc, *mu;
    int64_t ld_mu;
    int G, lgT;
    double *pv, *stat, *se;
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_wald(const __grid_constant__ WaldArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    wald_gene<P>(grp, d, a.prm, a.disp[g], a.lfc + (int64_t)g * P, a.mu + g, a.ld_mu, a.pv + g, a.stat + g, a.se + g,
                 valid);
}

template <int P>
struct MomArgs {
    DesignView dv;
    SmallMat<P> pinv;
    const double* normed;    // plugin calls
    const int64_t* counts;   // resident pipeline
    int64_t ld;
    int G, lgT;
    double s_mean_inv, min_disp, max_disp;
    double *alpha, *aux;     // aux: all_zero flags (moments) or normalised means (fused)
    double min_mu;           // fused kernel only: also write mu_hat = max(sf * X beta, min_mu) when mu_hat != nullptr
    double* mu_hat;
    int64_t ld_mu;
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_rough(const __grid_constant__ MomArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    const double r = rough_disp_gene<P>(grp, d, a.pinv, NormedF64{a.normed + g, a.ld});
    if (valid && grp.si == 0) a.alpha[g] = r;
}

template <int P>
__global__ void __launch_bounds__(kBlock) k_moments(const __grid_constant__ MomArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    double mean;
    bool az;
    const double m = moments_disp_gene(grp, d, NormedF64{a.normed + g, a.ld}, a.s_mean_inv, mean, az);
    if (valid && grp.si == 0) {
        a.alpha[g] = m;
        a.aux[g] = az ? 1.0 : 0.0;
    }
}

template <int P>
__global__ void __launch_bounds__(kBlock) k_mom_from_counts(const __grid_constant__ MomArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    mom_fused_gene<P>(grp, d, a.pinv, a.counts + g, a.ld, a.s_mean_inv, a.min_disp, a.max_disp, a.min_mu, a.alpha + g, a.aux + g,
                      a.mu_hat ? a.mu_hat + g : nullptr, a.ld_mu, valid);
}

template <int P>
struct CooksArgs {
    DesignView dv;
    const int* plan;
    int plan_len, n_cells, n_in_cells;
    const int64_t* counts;
    int64_t ld;
    int G, lgT;
    const double *mu, *hat;
    int64_t ld2;
    double cutoff;
    double* cooks;
    int64_t ld_out;
    double *disp, *outlier, *replaced;
};

// Cook's distances + trimmed-moments dispersions (dds.py:986-1040); the gene's cell members are staged in shared memory
template <int P>
__global__ void __launch_bounds__(kBlock) k_cooks(const __grid_constant__ CooksArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    int* plan_s = reinterpret_cast<int*>(smem + scratch_off(a.dv, false));
    for (int i = threadIdx.x; i < a.plan_len; i += blockDim.x) plan_s[i] = a.plan[i];
    __syncthreads();
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    const CellPlan plan{plan_s + 2 + a.n_cells + 1, plan_s + 2, a.n_cells, plan_s[1]};
    const size_t plan_bytes = ((size_t)a.plan_len * 4 + 15) & ~(size_t)15;
    const int gslot = (threadIdx.x >> 5) * grp.gpw + ((threadIdx.x & 31) & (grp.gpw - 1));
    double* vals = reinterpret_cast<double*>(smem + scratch_off(a.dv, false) + plan_bytes) + (size_t)gslot * 2 * a.n_in_cells;
    cooks_gene<P>(grp, d, plan, a.counts + g, a.ld, a.mu + g, a.hat + g, a.ld2, a.cutoff, vals, vals + a.n_in_cells,
                  a.cooks ? a.cooks + g : nullptr, a.ld_out, a.disp + g, a.outlier + g, a.replaced + g, valid);
}

template <int P>
struct MuLfcArgs {
    DesignView dv;
    const double* lfc;
    int G, lgT;
    double* mu;
    int64_t ld_out;
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_mu_from_lfc(const __grid_constant__ MuLfcArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    if (!valid) return;
    double b[P];
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) b[j] = a.lfc[(int64_t)g * P + j];
    for (int n = grp.si; n < d.N; n += grp.T) {
        double x[P];
        load_x<P>(d, n, x);
        double eta = 0.0;
PDQ_UNROLL_P
        for (int j = 0; j < P; ++j) eta = fma(x[j], b[j], eta);
        a.mu[n * a.ld_out + g] = d.sf[n * d.RS] * exp(eta);  // ds.py:320-324
    }
}


#if PDQ_TU_P == 0
// ---- dispersion trend + prior: the whole gamma-GLM fit (all iterations, all outer rounds) and the MAD-based prior
// variance in ONE launch of one thread-block cluster.  Per iteration the blocks reduce their partial sums with warp
// shuffles + shared memory, exchange the block totals through distributed shared memory (DSMEM stores into every
// peer's slot table) and meet at one cluster barrier; all blocks then hold identical totals and take identical
// decisions, so no further communication is needed.
constexpr int kTrendK = 10;        // packed sums per reduction
constexpr int kTrendMaxCluster = 16;

struct ClusterReducer {
    double* warp_part;  // [32][kTrendK]
    double* slots;      // [2][kTrendMaxCluster][kTrendK], written by every block of the cluster (DSMEM)
    double* totals;     // [2][kTrendK]: the cluster-wide sums, broadcast to the block's threads
    unsigned rank, nblocks;
    int parity;
    __host__ __device__ int tid() const {
#if defined(__CUDA_ARCH__)
        return rank * blockDim.x + threadIdx.x;
#else
        return 0;
#endif
    }
    __host__ __device__ int nthreads() const {
#if defined(__CUDA_ARCH__)
        return nblocks * blockDim.x;
#else
        return 1;
#endif
    }
    __host__ __device__ int local_tid() const {
#if defined(__CUDA_ARCH__)
        return threadIdx.x;
#else
        return 0;
#endif
    }
    __host__ __device__ int local_nthreads() const {
#if defined(__CUDA_ARCH__)
        return blockDim.x;
#else
        return 1;
#endif
    }
    __host__ __device__ void local_sync() {
#if defined(__CUDA_ARCH__)
        __syncthreads();
#endif
    }
    __host__ __device__ void sync() {
#if defined(__CUDA_ARCH__)
        cooperative_groups::this_cluster().sync();
#endif
    }
    // cluster-wide maximum of one value per thread (same exchange pattern as sum_many)
    __host__ __device__ double max_one(double v) {
#if defined(__CUDA_ARCH__)
        namespace cg = cooperative_groups;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
        if (lane == 0) warp_part[warp * kTrendK] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            double m = warp_part[0];
            const int nw = blockDim.x >> 5;
            for (int w = 1; w < nw; ++w) m = fmax(m, warp_part[w * kTrendK]);
            if (nblocks > 1) {
                cg::cluster_group cluster = cg::this_cluster();
                for (unsigned r = 0; r < nblocks; ++r)
                    cluster.map_shared_rank(slots, r)[(parity * kTrendMaxCluster + rank) * kTrendK] = m;
            } else {
                slots[parity * kTrendMaxCluster * kTrendK] = m;
            }
        }
        if (nblocks > 1) cg::this_cluster().sync(); else __syncthreads();
        double m = slots[parity * kTrendMaxCluster * kTrendK];
        for (unsigned r = 1; r < nblocks; ++r) m = fmax(m, slots[(parity * kTrendMaxCluster + r) * kTrendK]);
        parity ^= 1;
        return m;
#else
        return v;
#endif
    }
    // histogram protocol of select_kth: zeroed bins become visible, blocks count disjoint slices, bins are merged
    __host__ __device__ void hist_begin() {
#if defined(__CUDA_ARCH__)
        if (nblocks > 1) cooperative_groups::this_cluster().sync(); else __syncthreads();
#endif
    }
    __host__ __device__ unsigned* hist_merge(unsigned* hist) {
#if defined(__CUDA_ARCH__)
        __syncthreads();  // local bins complete
        if (nblocks == 1) return hist;
        namespace cg = cooperative_groups;
        cg::cluster_group cluster = cg::this_cluster();
        if (threadIdx.x < 256) {
            const unsigned v = hist[threadIdx.x];
            if (v)
                for (unsigned r = 0; r < nblocks; ++r) atomicAdd(cluster.map_shared_rank(hist + 256, r) + threadIdx.x, v);
        }
        cluster.sync();
        return hist + 256;
#else
        return hist;
#endif
    }
    // warp 0 scans the 256-bin histogram (8 bins per lane + shuffle scan) and publishes digit / count-before in out[0..1]
    __host__ __device__ void find_bin(const unsigned* hist, unsigned* out, size_t k, int& d, size_t& cum) {
#if defined(__CUDA_ARCH__)
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            unsigned c[8], tot = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                c[j] = hist[lane * 8 + j];
                tot += c[j];
            }
            unsigned inc = tot;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {
                const unsigned t = __shfl_up_sync(0xffffffffu, inc, off);
                if (lane >= off) inc += t;
            }
            const unsigned before = inc - tot;
            const unsigned kk = (unsigned)k;
            if (before <= kk && kk < inc) {  // exactly one lane owns the crossing
                unsigned run = before;
                int j = 0;
                for (; j < 8; ++j) {
                    if (run + c[j] > kk) break;
                    run += c[j];
                }
                out[0] = (unsigned)(lane * 8 + j);
                out[1] = run;
            }
        }
        __syncthreads();
        d = (int)out[0];
        cum = out[1];
#else
        (void)hist; (void)out; (void)k; (void)d; (void)cum;
#endif
    }
    __host__ __device__ void sum_many(double* v, int k) {
#if defined(__CUDA_ARCH__)
        namespace cg = cooperative_groups;
        cg::cluster_group cluster = cg::this_cluster();
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int j = 0; j < k; ++j) {
            double w = v[j];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
            if (lane == 0) warp_part[warp * kTrendK + j] = w;
        }
        __syncthreads();
        if ((int)threadIdx.x < k) {
            double tot = 0.0;
            const int nw = blockDim.x >> 5;
            for (int w = 0; w < nw; ++w) tot += warp_part[w * kTrendK + threadIdx.x];
            if (nblocks > 1) {
                for (unsigned r = 0; r < nblocks; ++r) {
                    double* remote = cluster.map_shared_rank(slots, r);
                    remote[(parity * kTrendMaxCluster + rank) * kTrendK + threadIdx.x] = tot;
                }
            } else {
                slots[parity * kTrendMaxCluster * kTrendK + threadIdx.x] = tot;
            }
        }
        if (nblocks > 1) cluster.sync(); else __syncthreads();  // release the DSMEM stores / acquire the peers'
        // k threads add up the blocks' slots, everybody reads the k totals (broadcast reads).  Having EVERY thread
        // add nblocks * k slots itself would cost 160 shared-memory reads per thread and pass.
        if ((int)threadIdx.x < k) {
            double tot = 0.0;
            for (unsigned r = 0; r < nblocks; ++r) tot += slots[(parity * kTrendMaxCluster + r) * kTrendK + threadIdx.x];
            totals[parity * kTrendK + threadIdx.x] = tot;
        }
        __syncthreads();
        for (int j = 0; j < k; ++j) v[j] = totals[parity * kTrendK + j];
        parity ^= 1;
#else
        (void)v;
        (void)k;
#endif
    }
};

__global__ void __launch_bounds__(1024) k_trend_prior(const double* __restrict__ x, const double* __restrict__ t,
                                                      double* scratch /* 3 n doubles: xs | ts | res */, size_t n,
                                                      int x_is_mean, double lo, double hi, int outer, double min_disp,
                                                      double trigamma_c, int with_prior, TrendOut* out) {
    __shared__ double warp_part[32 * kTrendK];
    __shared__ double slots[2 * kTrendMaxCluster * kTrendK];
    __shared__ double totals[2 * kTrendK];
    __shared__ unsigned hist[514];
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    ClusterReducer red{warp_part, slots, totals, cluster.block_rank(), cluster.num_blocks(), 0};
    double *xs = scratch, *ts = scratch + n, *res = scratch + 2 * n;
    trend_prepare(red, x, t, n, x_is_mean != 0, lo, hi, xs, ts);
    TrendOut o = trend_fit_outer(red, xs, ts, n, outer != 0);
    if (with_prior && o.status == 0.0) trend_prior(red, x, t, n, lo, hi, min_disp, trigamma_c, res, hist, o);
    if (red.tid() == 0) *out = o;
    cluster.sync();  // no block may exit while peers can still address its shared memory
}

// ---- the same fit on the whole GPU (vectors of >= 64 k genes: the gathered vectors of many gene shards, one large shard).  One
// cooperative launch of one block per SM; the per-pass reductions go through a few hundred bytes of global memory (atomics) and a
// grid-wide barrier instead of DSMEM and a cluster barrier.  The accumulators rotate over three slots so that none is zeroed while
// another block may still read or add to it: pass p adds into slot p % 3, reads it behind the barrier, and block 0 then clears slot
// (p + 2) % 3, last read in pass p - 1 and next used in pass p + 1.
struct GridScratch {
    double acc[3][kTrendK];
    unsigned long long maxkey[3];
    unsigned hist[3][256];
};

struct GridReducer {
    double* warp_part;  // [32][kTrendK] shared
    double* totals;     // [kTrendK] shared
    GridScratch* gs;    // global, zeroed before the launch
    int p_sum, p_max, p_hist;
    __device__ int tid() const { return blockIdx.x * blockDim.x + threadIdx.x; }
    __device__ int nthreads() const { return gridDim.x * blockDim.x; }
    __device__ int local_tid() const { return threadIdx.x; }
    __device__ int local_nthreads() const { return blockDim.x; }
    __device__ void local_sync() { __syncthreads(); }
    __device__ void sync() { cooperative_groups::this_grid().sync(); }
    __device__ void sum_many(double* v, int k) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, slot = p_sum % 3;
        for (int j = 0; j < k; ++j) {
            double w = v[j];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
            if (lane == 0) warp_part[warp * kTrendK + j] = w;
        }
        __syncthreads();
        if ((int)threadIdx.x < k) {
            double tot = 0.0;
            const int nw = blockDim.x >> 5;
            for (int w = 0; w < nw; ++w) tot += warp_part[w * kTrendK + threadIdx.x];
            atomicAdd(&gs->acc[slot][threadIdx.x], tot);
        }
        cooperative_groups::this_grid().sync();
        if ((int)threadIdx.x < k) totals[threadIdx.x] = *reinterpret_cast<volatile double*>(&gs->acc[slot][threadIdx.x]);
        if (blockIdx.x == 0 && (int)threadIdx.x < kTrendK) gs->acc[(p_sum + 2) % 3][threadIdx.x] = 0.0;
        __syncthreads();
        for (int j = 0; j < k; ++j) v[j] = totals[j];
        __syncthreads();  // totals is overwritten by the next reduction
        ++p_sum;
    }
    __device__ double max_one(double v) {
        const int lane = threadIdx.x & 31, slot = p_max % 3;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
        if (lane == 0) atomicMax(&gs->maxkey[slot], (unsigned long long)f64_key(v));
        cooperative_groups::this_grid().sync();
        const double m = f64_from_key(*reinterpret_cast<volatile unsigned long long*>(&gs->maxkey[slot]));
        if (blockIdx.x == 0 && threadIdx.x == 0) gs->maxkey[(p_max + 2) % 3] = 0ull;
        ++p_max;
        return m;
    }
    __device__ void hist_begin() { __syncthreads(); }
    __device__ unsigned* hist_merge(unsigned* hist) {
        const int slot = p_hist % 3;
        __syncthreads();  // local bins complete
        if (threadIdx.x < 256) {
            const unsigned c = hist[threadIdx.x];
            if (c) atomicAdd(&gs->hist[slot][threadIdx.x], c);
        }
        cooperative_groups::this_grid().sync();
        if (threadIdx.x < 256) hist[256 + threadIdx.x] = *reinterpret_cast<volatile unsigned*>(&gs->hist[slot][threadIdx.x]);
        if (blockIdx.x == 0 && threadIdx.x < 256) gs->hist[(p_hist + 2) % 3][threadIdx.x] = 0u;
        __syncthreads();
        ++p_hist;
        return hist + 256;
    }
    __device__ void find_bin(const unsigned* hist, unsigned* out, size_t k, int& d, size_t& cum) {
        ClusterReducer tmp{nullptr, nullptr, nullptr, 0u, 1u, 0};  // the single-block scan of the 256 merged bins
        tmp.find_bin(hist, out, k, d, cum);
    }
};

__global__ void __launch_bounds__(1024) k_trend_prior_grid(const double* __restrict__ x, const double* __restrict__ t,
                                                           double* scratch /* 3 n doubles: xs | ts | res */, size_t n, int x_is_mean,
                                                           double lo, double hi, int outer, double min_disp, double trigamma_c,
                                                           int with_prior, TrendOut* out, GridScratch* gs) {
    __shared__ double warp_part[32 * kTrendK];
    __shared__ double totals[kTrendK];
    __shared__ unsigned hist[514];
    GridReducer red{warp_part, totals, gs, 0, 0, 0};
    double *xs = scratch, *ts = scratch + n, *res = scratch + 2 * n;
    trend_prepare(red, x, t, n, x_is_mean != 0, lo, hi, xs, ts);
    TrendOut o = trend_fit_outer(red, xs, ts, n, outer != 0);
    if (with_prior && o.status == 0.0) trend_prior(red, x, t, n, lo, hi, min_disp, trigamma_c, res, hist, o);
    if (red.tid() == 0) *out = o;
}

// ---- median-of-ratios size factors (preprocessing.py:31-102), SURVEY.md §8 f-2 -------------------------------------
// 1. per-gene mean of log counts (-inf when the gene holds a zero: such genes are filtered out, preprocessing.py:52-54)
__global__ void __launch_bounds__(kBlock) k_log_means(const int64_t* __restrict__ counts, int64_t ld, int N, int G, int lgT,
                                                      double* __restrict__ logmeans) {
    Group grp;
    int g;
    bool valid;
    map_lanes(lgT, G, grp, g, valid);
    const int64_t* yp = counts + g + (int64_t)grp.si * ld;
    double s = 0.0;
    for (int n = grp.si; n < N; n += grp.T, yp += (int64_t)grp.T * ld) s += log((double)*yp);  // libdevice log: log(0) = -inf
    s = grp.sum(s);
    if (valid && grp.si == 0) logmeans[g] = s / (double)N;
}

// 2. one block per sample: log ratios of the sample against the gene means, exact median by radix select
__global__ void __launch_bounds__(1024) k_size_factor_median(const int64_t* __restrict__ counts, int64_t ld, int G,
                                                             const double* __restrict__ logmeans, double* scratch,
                                                             double* sf_out) {
    __shared__ unsigned hist[514];
    __shared__ double warp_part[32 * kTrendK];
    __shared__ double slots[2 * kTrendMaxCluster * kTrendK];
    __shared__ double totals[2 * kTrendK];
    __shared__ unsigned cnt_s;
    const int n = blockIdx.x;
    double* row = scratch + (size_t)n * G;
    const int64_t* c = counts + (int64_t)n * ld;
    if (threadIdx.x == 0) cnt_s = 0;
    __syncthreads();
    unsigned cnt = 0;
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        const double lm = logmeans[g];
        const bool keep = fabs(lm) <= 1.7976931348623157e308;  // ~np.isinf(logmeans); NaN cannot occur for counts >= 0
        row[g] = keep ? log((double)c[g]) - lm : __longlong_as_double(0x7ff8000000000000ll);
        cnt += keep;
    }
    atomicAdd(&cnt_s, cnt);
    __syncthreads();
    ClusterReducer red{warp_part, slots, totals, 0u, 1u, 0};  // one block per sample: the single-block paths of the reducer
    const double med = median_of(red, row, (size_t)G, (size_t)cnt_s, false, 0.0, hist);
    if (threadIdx.x == 0) sf_out[n] = exp(med);
}

// fitted = c0 + c1 / mean (dds.py:1267-1275) from the device-resident coefficients
__global__ void k_trend_eval(const double* __restrict__ means, size_t n, const TrendOut* __restrict__ c, double* fitted) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fitted[i] = c->c0 + c->c1 / means[i];
}

// final dispersions (dds.py:918-932): clip the MAP estimate, but genes whose genewise estimate lies more than
// 2 sd of the log residuals above the trend keep their (clipped) genewise value
__global__ void k_select_disp(const double* __restrict__ gw, const double* __restrict__ mp, const double* __restrict__ fitted,
                              const TrendOut* __restrict__ c, size_t n, double lo, double hi, double* disp, double* outlier) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double g = gw[i], m = mp[i];
    g = (g < lo) ? lo : ((g > hi) ? hi : g);
    m = (m < lo) ? lo : ((m > hi) ? hi : m);
    const bool out = log(g) > log(fitted[i]) + 2.0 * sqrt(c->squared_logres);
    disp[i] = out ? g : m;
    if (outlier) outlier[i] = out ? 1.0 : 0.0;
}

#endif  // PDQ_TU_P == 0

// ---- launch helpers ---------------------------------------------------------------------------------
inline int grid_for(int G, int lgT) {
    const int genes_per_block = kWarps * (32 >> lgT);
    return (G + genes_per_block - 1) / genes_per_block;
}

inline int alpha_descending() {
    static int v = -1;
    if (v < 0) {
        // tuning hook, default off: with ascending counts the costly high-count tiles overlap the cheap ones' tail just as well
        const char* e = getenv("PDQ_ALPHA_DESCENDING");
        v = e ? (atoi(e) != 0) : 0;
    }
    return v;
}

// one wave of blocks for the (normally idle) fallback kernels
inline int fallback_grid(int sm_count, int G, int lgT) {
    const int need = grid_for(G, lgT);
    return need < 2 * sm_count ? need : 2 * sm_count;
}

template <class K>
int prep(K kernel, size_t smem) {
    if (smem > kMaxDynSmem) return PDQ_ERR_UNSUPPORTED;
    if (smem > 48 * 1024) {
        if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
            return PDQ_ERR_CUDA;
    }
    return 0;
}

// grid of a persistent kernel: every block the machine can hold at once, but no more blocks than warp tiles need
template <class K>
int persistent_grid(K kernel, size_t smem, int sm_count, int G, int lgT) {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBlock, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    const int need = grid_for(G, lgT);
    const int fit = per_sm * sm_count;
    return need < fit ? need : fit;
}

template <int P>
SmallMat<P> pinv_of(const DesignDev& d) {
    SmallMat<P> m;
    for (int i = 0; i < P * P; ++i) m.v[i] = d.pinv[i];
    return m;
}


// ---- apeGLM shrinkage (SURVEY.md §8 f-3) ----------------------------------------------------------------------------
template <int P>
struct ShrinkArgs {
    DesignView dv;
    ShrinkParams prm;
    const int64_t* counts;
    int64_t ld;
    int G, lgT;
    const double* size;
    double *beta, *ih, *conv;
    int* status;
    int force;  // test hook: send every gene of a two-column design through the grid fallback
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_lfc_shrink(const __grid_constant__ ShrinkArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    shrink_gene<P>(grp, d, a.prm, a.counts + g, a.ld, a.size[g], a.beta + (int64_t)g * P, a.ih + (int64_t)g * P * P, a.conv + g,
                   a.status + g, valid, a.force != 0);
}

#if PDQ_TU_P == 0
__global__ void __launch_bounds__(kBlock) k_lfc_shrink_grid(const __grid_constant__ ShrinkArgs<2> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    const bool run = valid && a.status[g] == kShrinkNeedsGrid;
    if (!__syncthreads_or(run)) return;
    const DesignS d = stage_design(a.dv, 2, smem);
    if (!__any_sync(0xffffffffu, run)) return;
    shrink_grid_gene(grp, d, a.prm, a.counts + g, a.ld, a.size[g], a.beta + (int64_t)g * 2, a.ih + (int64_t)g * 4, run);
}

#endif

#if PDQ_TU_P == 0
// ---- FP64 peak probe (bench.py: the second roofline of these kernels) ------------------------------------------------
// 8 independent DFMA chains per thread, 8 blocks of 256 threads per SM: enough independent work to saturate the FP64 pipe.
__global__ void __launch_bounds__(256) k_fp64_peak(double* out, int iters, double m, double c) {
    double a[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) a[k] = 1.0 + 1e-9 * (double)(threadIdx.x + k);
    for (int i = 0; i < iters; ++i) {
#pragma unroll
        for (int k = 0; k < 8; ++k) a[k] = fma(a[k], m, c);
    }
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) s += a[k];
    out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// ---- selected gene columns of a resident (N, G) array into a compact (N, R) array: the outlier refit works on the few replaced
// genes only (dds.py:1360-1458), so their mu / hat columns are all that has to leave the device
__global__ void k_gather_cols(const double* __restrict__ in, int64_t ld_in, int N, const int* __restrict__ idx, int R,
                              double* __restrict__ out, int64_t ld_out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, n = blockIdx.y;
    if (j < R && n < N) out[(int64_t)n * ld_out + j] = in[(int64_t)n * ld_in + idx[j]];
}

// ---- gene order of the resident pipeline.  IRLS iteration counts follow a gene's expression level, and the four genes of a warp
// run in lock step until the slowest stops: in the caller's gene order 22-24 % of the IRLS sweeps are repeats of finished genes,
// with the genes sorted by their total count 4-5 % (measured with the emulator on the synthetic cohorts).  ResidentFit therefore
// stores the shard's counts with the columns sorted by column sum (once, at upload) and returns every per-gene result to the
// caller's order with one scatter at the end of a pass.  Per-gene arithmetic does not depend on a gene's position: results are
// bit-identical to the unsorted pass.
__global__ void k_column_sums(const int64_t* __restrict__ counts, int64_t ld, int N, int G, double* __restrict__ sums) {
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    long long s = 0;
    for (int n = 0; n < N; ++n) s += counts[(int64_t)n * ld + g];
    sums[g] = (double)s;
}

// out[v][perm[j]][k] = in[v][j][k], v < nvec blocks of `stride` rows of `width` doubles (rows j < n)
__global__ void k_scatter_rows(const double* __restrict__ in, double* __restrict__ out, const int* __restrict__ perm, int n, int nvec,
                               int64_t stride, int width) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t per = (int64_t)n * width;
    if (t >= per * nvec) return;
    const int v = (int)(t / per);
    const int64_t r = t - (int64_t)v * per;
    const int j = (int)(r / width), k = (int)(r - (int64_t)j * width);
    out[((int64_t)v * stride + perm[j]) * width + k] = in[((int64_t)v * stride + j) * width + k];
}

// ---- content checksum of a device buffer: the device half of the residency cache of pdq_api.cu (host_hash there computes the
// same two wrapping sums with host threads).  HBM-bound.
__global__ void __launch_bounds__(256) k_hash(const uint64_t* __restrict__ w, size_t n, unsigned long long* out) {
    unsigned long long a = 0, b = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const uint64_t v = w[i];
        uint64_t t = (v + (i + 1) * 0x9E3779B97F4A7C15ull) * 0xBF58476D1CE4E5B9ull;
        a += t ^ (t >> 31);
        uint64_t u = (v ^ ((i + 1) * 0xD6E8FEB86659FD93ull)) * 0x94D049BB133111EBull;
        b += u ^ (u >> 29);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b += __shfl_xor_sync(0xffffffffu, b, off);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(out, a);
        atomicAdd(out + 1, b);
    }
}

#endif  // PDQ_TU_P == 0

#if PDQ_TU_P == 0
#define PDQ_DISPATCH_P(p, ...)             \
    switch (p) {                           \
        case 1: { constexpr int P = 1; __VA_ARGS__; } break; \
        case 2: { constexpr int P = 2; __VA_ARGS__; } break; \
        case 3: { constexpr int P = 3; __VA_ARGS__; } break; \
        case 4: { constexpr int P = 4; __VA_ARGS__; } break; \
        case 5: { constexpr int P = 5; __VA_ARGS__; } break; \
        case 6: { constexpr int P = 6; __VA_ARGS__; } break; \
        case 7: { constexpr int P = 7; __VA_ARGS__; } break; \
        case 8: { constexpr int P = 8; __VA_ARGS__; } break; \
        default: return PDQ_ERR_UNSUPPORTED; \
    }
#else
#define PDQ_DISPATCH_P(p, ...)                              \
    {                                                       \
        if ((p) != PDQ_TU_P) return PDQ_ERR_UNSUPPORTED;    \
        constexpr int P = PDQ_TU_P;                         \
        __VA_ARGS__;                                        \
    }
#endif

inline int check_launch() { return cudaGetLastError() == cudaSuccess ? 0 : PDQ_ERR_CUDA; }

}  // namespace

int PDQ_TUFN(launch_lin_reg_mu)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_mu,
                      double* mu_out, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        LinMuArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, pinv_of<P>(d), counts, ld, G, c.lgT, min_mu, mu_out, ld_out};
        if (int e = prep(k_lin_reg_mu<P>, d.smem_bytes)) return e;
        k_lin_reg_mu<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_irls)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* disp,
                const IrlsHost& h, double* beta, double* mu, double* hat, int64_t ld_out, double* conv, int* status,
                int* n_fallback, const WaldHost* w) {
    if (n_fallback && cudaMemsetAsync(n_fallback, 0, sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
    PDQ_DISPATCH_P(d.p, {
        IrlsArgs<P> a;
        a.dv = DesignView{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0};
        a.pinv = pinv_of<P>(d);
        a.prm = IrlsParams{h.min_mu, h.beta_tol, h.min_beta, h.max_beta, h.maxiter, d.full_rank, d.few_rows,
                           (c.debug & PDQ_DEBUG_FAIL_IRLS_OPTIMIZER) ? 1 : 0};
        a.counts = counts; a.ld = ld; a.G = G; a.lgT = c.lgT; a.disp = disp;
        a.beta = beta; a.mu = mu; a.hat = hat; a.conv = conv; a.ld_out = ld_out;
        a.status = status; a.n_fallback = n_fallback; a.ticket = c.tickets;
        a.force = (c.debug & PDQ_DEBUG_FORCE_IRLS_OPTIMIZER) ? 1 : 0;
        a.with_wald = w ? 1 : 0;
        a.wald_p = a.wald_stat = a.wald_se = nullptr;
        if (w) {
            for (int i = 0; i < P * P; ++i) a.wald.ridge[i] = w->ridge[i];
            for (int i = 0; i < P; ++i) a.wald.contrast[i] = w->contrast[i];
            a.wald.lfc_null = w->lfc_null;
            a.wald.alt = w->alt;
            a.wald_p = w->pv; a.wald_stat = w->stat; a.wald_se = w->se;
        }
        const size_t smem_irls = d.smem_bytes + kMathTabBytes + (size_t)(1 + kWarps * (32 >> c.lgT)) * kPsiK * sizeof(double);
        if (int e = prep(k_irls_optimizer<P>, d.smem_bytes)) return e;
        if (cudaMemsetAsync(c.tickets, 0, 2 * sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
        if (d.staged) {
            if (int e = prep(k_irls<P, true>, smem_irls)) return e;
            k_irls<P, true><<<persistent_grid(k_irls<P, true>, smem_irls, c.sm_count, G, c.lgT), kBlock, smem_irls, c.stream>>>(a);
        } else {
            if (int e = prep(k_irls<P, false>, smem_irls)) return e;
            k_irls<P, false><<<persistent_grid(k_irls<P, false>, smem_irls, c.sm_count, G, c.lgT), kBlock, smem_irls, c.stream>>>(a);
        }
        k_irls_optimizer<P><<<fallback_grid(c.sm_count, G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 2;
}

int PDQ_TUFN(launch_alpha_mle)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G,
                     const double* mu, int64_t ld_mu, const double* alpha_hat, double min_disp, double max_disp,
                     double prior_var, const double* prior_var_dev, int cr_reg, int prior_reg, double* alpha, double* conv,
                     int* status, const double* hint_in, double* hint_out) {
    PDQ_DISPATCH_P(d.p, {
        AlphaArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, AlphaParams{log(min_disp), log(max_disp), prior_var, cr_reg, prior_reg},
                       counts, ld, G, c.lgT, mu, ld_mu, alpha_hat, alpha, conv, status, prior_var_dev, c.tickets + 2,
                       (c.debug & PDQ_DEBUG_FORCE_ALPHA_GRID) ? 1 : 0, hint_in, hint_out, alpha_descending()};
        const size_t smem_alpha = d.smem_bytes + kMathTabBytes + (size_t)kWarps * (32 >> c.lgT) * 2 * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (cudaMemsetAsync(c.tickets + 2, 0, 2 * sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
        if (d.staged) {
            if (int e = prep(k_alpha_mle<P, true>, smem_alpha)) return e;
            k_alpha_mle<P, true><<<persistent_grid(k_alpha_mle<P, true>, smem_alpha, c.sm_count, G, c.lgT), kBlock, smem_alpha, c.stream>>>(a);
        } else {
            if (int e = prep(k_alpha_mle<P, false>, smem_alpha)) return e;
            k_alpha_mle<P, false><<<persistent_grid(k_alpha_mle<P, false>, smem_alpha, c.sm_count, G, c.lgT), kBlock, smem_alpha, c.stream>>>(a);
        }
        k_alpha_grid<P><<<fallback_grid(c.sm_count, G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 2;
}

int PDQ_TUFN(launch_wald)(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, const double* mu,
                int64_t ld_mu, int G, const double* ridge, const double* contrast, double lfc_null, int alt, double* pv,
                double* stat, double* se) {
    PDQ_DISPATCH_P(d.p, {
        WaldArgs<P> a;
        a.dv = DesignView{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0};
        for (int i = 0; i < P * P; ++i) a.prm.ridge[i] = ridge[i];
        for (int i = 0; i < P; ++i) a.prm.contrast[i] = contrast[i];
        a.prm.lfc_null = lfc_null;
        a.prm.alt = alt;
        a.disp = disp; a.lfc = lfc; a.mu = mu; a.ld_mu = ld_mu; a.G = G; a.lgT = c.lgT;
        a.pv = pv; a.stat = stat; a.se = se;
        if (int e = prep(k_wald<P>, d.smem_bytes)) return e;
        k_wald<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_rough)(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, pinv_of<P>(d), normed, nullptr, ld, G, c.lgT, d.s_mean_inv, 0.0, 0.0, alpha,
                     nullptr, 0.0, nullptr, 0};
        if (int e = prep(k_rough<P>, d.smem_bytes)) return e;
        k_rough<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_moments)(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha,
                   double* all_zero) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, pinv_of<P>(d), normed, nullptr, ld, G, c.lgT, d.s_mean_inv, 0.0, 0.0, alpha,
                     all_zero, 0.0, nullptr, 0};
        if (int e = prep(k_moments<P>, d.smem_bytes)) return e;
        k_moments<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_mom_from_counts)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G,
                           double min_disp, double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat,
                           int64_t ld_mu) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, pinv_of<P>(d), nullptr, counts, ld, G, c.lgT, d.s_mean_inv, min_disp,
                     max_disp, alpha, normed_mean, min_mu, mu_hat, ld_mu};
        if (int e = prep(k_mom_from_counts<P>, d.smem_bytes)) return e;
        k_mom_from_counts<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_mu_from_lfc)(const LaunchCfg& c, const DesignDev& d, const double* lfc, int G, double* mu, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        MuLfcArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, lfc, G, c.lgT, mu, ld_out};
        if (int e = prep(k_mu_from_lfc<P>, d.smem_bytes)) return e;
        k_mu_from_lfc<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}

#if PDQ_TU_P == 0
int launch_trend_fit(const LaunchCfg& c, const double* x, const double* t, double* scratch3n, size_t n, int x_is_mean,
                     double lo, double hi, int outer, double min_disp, double trigamma_c, int with_prior, double* out16) {
    // large vectors: one block per SM, cooperative launch (k_trend_prior_grid); PDQ_TREND_GRID=0/1 forces the choice
    {
        const char* e = getenv("PDQ_TREND_GRID");
        const int force = e ? atoi(e) : -1;
        const bool use_grid = force >= 0 ? force != 0 : n >= 65536;
        if (use_grid && c.grid_scratch) {
            if (cudaMemsetAsync(c.grid_scratch, 0, sizeof(GridScratch), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
            int blocks = (int)((n + 2047) / 2048);
            if (blocks > c.sm_count) blocks = c.sm_count;
            if (blocks < 1) blocks = 1;
            TrendOut* o16 = reinterpret_cast<TrendOut*>(out16);
            GridScratch* gs = reinterpret_cast<GridScratch*>(c.grid_scratch);
            void* args[] = {(void*)&x, (void*)&t, (void*)&scratch3n, (void*)&n, (void*)&x_is_mean, (void*)&lo, (void*)&hi, (void*)&outer,
                            (void*)&min_disp, (void*)&trigamma_c, (void*)&with_prior, (void*)&o16, (void*)&gs};
            if (cudaLaunchCooperativeKernel((const void*)k_trend_prior_grid, dim3(blocks), dim3(1024), args, 0, c.stream) == cudaSuccess) {
                if (int e = check_launch()) return e;
                return 1;
            }
            cudaGetLastError();  // cooperative launch not possible here: the cluster version below
        }
    }
    // cluster size: enough blocks for ~4 elements per thread; 8 is the portable maximum, 16 needs the opt-in attribute
    static int max_cluster = 0;
    if (!max_cluster) {
        max_cluster = 8;
        if (cudaFuncSetAttribute(k_trend_prior, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess)
            max_cluster = kTrendMaxCluster;
        else
            cudaGetLastError();
    }
    // threads per block: the per-pass cost of a small fit is the reduction (ten packed sums through warp shuffles and shared
    // memory per warp), not the arithmetic -- 256 threads per block (~5 genes per thread at 20 000 genes) instead of 1024 cut
    // it four-fold; large vectors keep 1024
    unsigned threads = n <= 24576 ? 256u : (n <= 49152 ? 512u : 1024u);
    if (const char* e = getenv("PDQ_TREND_THREADS")) {  // tuning hook
        const int v = atoi(e);
        if (v == 256 || v == 512 || v == 1024) threads = (unsigned)v;
    }
    unsigned nb = 1;
    while ((int)nb < max_cluster && (size_t)nb * threads * 4 < n) nb <<= 1;
    if (const char* e = getenv("PDQ_TREND_CLUSTER")) {  // tuning hook: force the cluster size (1, 2, 4, 8, 16)
        const int v = atoi(e);
        if (v >= 1 && v <= max_cluster && !(v & (v - 1))) nb = (unsigned)v;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(nb, 1, 1);
    cfg.blockDim = dim3(threads, 1, 1);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = c.stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = nb;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t err = cudaLaunchKernelEx(&cfg, k_trend_prior, x, t, scratch3n, n, x_is_mean, lo, hi, outer, min_disp, trigamma_c,
                                         with_prior, reinterpret_cast<TrendOut*>(out16));
    if (err != cudaSuccess && nb > 8) {  // a 16-block cluster could not be placed: fall back to the portable size
        cudaGetLastError();
        max_cluster = 8;
        attr[0].val.clusterDim.x = 8;
        cfg.gridDim = dim3(8, 1, 1);
        err = cudaLaunchKernelEx(&cfg, k_trend_prior, x, t, scratch3n, n, x_is_mean, lo, hi, outer, min_disp, trigamma_c, with_prior,
                                 reinterpret_cast<TrendOut*>(out16));
    }
    if (err != cudaSuccess) return PDQ_ERR_CUDA;
    if (int e = check_launch()) return e;
    return 1;
}

int launch_trend_eval(const LaunchCfg& c, const double* means, size_t n, const double* out16, double* fitted) {
    k_trend_eval<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(means, n, reinterpret_cast<const TrendOut*>(out16), fitted);
    if (int e = check_launch()) return e;
    return 1;
}

#endif  // PDQ_TU_P == 0

int PDQ_TUFN(launch_cooks)(const LaunchCfg& c0, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                 int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced) {
    // the per-gene staging (2 * n_in_cells doubles) bounds the genes per block: widen the lane groups until it fits
    LaunchCfg c = c0;
    const size_t plan_bytes = ((size_t)d.plan_len * 4 + 15) & ~(size_t)15;
    auto need = [&](int lgT) { return d.smem_bytes + plan_bytes + (size_t)kWarps * (32 >> lgT) * 2 * d.n_in_cells * sizeof(double); };
    while (c.lgT < 5 && need(c.lgT) > 96 * 1024) ++c.lgT;
    if (need(c.lgT) > kMaxDynSmem) return PDQ_ERR_UNSUPPORTED;
    PDQ_DISPATCH_P(d.p, {
        CooksArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, d.cell_plan, d.plan_len, d.n_cells, d.n_in_cells, counts, ld, G, c.lgT, mu, hat, ld2,
                       cutoff, cooks, ld_out, disp, outlier, replaced};
        if (int e = prep(k_cooks<P>, need(c.lgT))) return e;
        k_cooks<P><<<grid_for(G, c.lgT), kBlock, need(c.lgT), c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 1;
}


int PDQ_TUFN(launch_lfc_shrink)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* size,
                      double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian,
                      double* conv, int* status) {
    if (shrink_index < 0 || shrink_index >= d.p) return PDQ_ERR_INVALID;
    const ShrinkParams prm{1.0 / (prior_no_shrink_scale * prior_no_shrink_scale), prior_scale * prior_scale, shrink_index};
    const int force = (c.debug & PDQ_DEBUG_FORCE_SHRINK_GRID) ? 1 : 0;
    PDQ_DISPATCH_P(d.p, {
        ShrinkArgs<P> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, prm, counts, ld, G, c.lgT, size, beta, inv_hessian, conv, status, force};
        if (int e = prep(k_lfc_shrink<P>, d.smem_bytes)) return e;
        k_lfc_shrink<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
#if PDQ_TU_P == 0
    if (d.p == 2) {
        ShrinkArgs<2> a{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, prm, counts, ld, G, c.lgT, size, beta, inv_hessian, conv, status, force};
        if (int e = prep(k_lfc_shrink_grid, d.smem_bytes)) return e;
        k_lfc_shrink_grid<<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    }
#endif
    if (int e = check_launch()) return e;
    return d.p == 2 ? 2 : 1;
}

#if PDQ_TU_P == 0
int launch_gather_cols(cudaStream_t stream, const double* in, int64_t ld_in, int N, const int* idx, int R, double* out, int64_t ld_out) {
    if (R <= 0 || N <= 0) return 0;
    k_gather_cols<<<dim3((unsigned)((R + 127) / 128), (unsigned)N), 128, 0, stream>>>(in, ld_in, N, idx, R, out, ld_out);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_column_sums(cudaStream_t stream, const int64_t* counts, int64_t ld, int N, int G, double* sums) {
    k_column_sums<<<(unsigned)((G + 127) / 128), 128, 0, stream>>>(counts, ld, N, G, sums);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_scatter_rows(cudaStream_t stream, const double* in, double* out, const int* perm, int n, int nvec, int64_t stride, int width) {
    const int64_t total = (int64_t)n * width * nvec;
    if (total <= 0) return 0;
    k_scatter_rows<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(in, out, perm, n, nvec, stride, width);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_hash(cudaStream_t stream, int sm_count, const void* dptr, size_t words, uint64_t* out2) {
    k_hash<<<sm_count * 8, 256, 0, stream>>>(reinterpret_cast<const uint64_t*>(dptr), words, reinterpret_cast<unsigned long long*>(out2));
    if (int e = check_launch()) return e;
    return 1;
}

int launch_fp64_peak(const LaunchCfg& c, double* out, int iters, double* flop) {
    const int blocks = c.sm_count * 8, threads = 256;
    k_fp64_peak<<<blocks, threads, 0, c.stream>>>(out, iters, 0.999999999, 1e-9);
    *flop = 2.0 * 8.0 * (double)iters * (double)blocks * (double)threads;
    if (int e = check_launch()) return e;
    return 1;
}

int launch_size_factors(const LaunchCfg& c, const int64_t* counts, int64_t ld, int N, int G, double* logmeans,
                        double* scratch, double* sf_out) {
    k_log_means<<<grid_for(G, c.lgT), kBlock, 0, c.stream>>>(counts, ld, N, G, c.lgT, logmeans);
    k_size_factor_median<<<N, 1024, 0, c.stream>>>(counts, ld, G, logmeans, scratch, sf_out);
    if (int e = check_launch()) return e;
    return 2;
}

int launch_select_disp(const LaunchCfg& c, const double* gw, const double* mp, const double* fitted, const double* out16,
                       size_t n, double lo, double hi, double* disp, double* outlier) {
    k_select_disp<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(gw, mp, fitted, reinterpret_cast<const TrendOut*>(out16), n,
                                                                     lo, hi, disp, outlier);
    if (int e = check_launch()) return e;
    return 1;
}

#endif  // PDQ_TU_P == 0

}  // namespace pdq
