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
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

#include "pdq_gene.cuh"
#include "pdq_trend.cuh"
#include "pdq_shrink.cuh"
#include "pdq_internal.h"
#include "pdq_launch.cuh"

// This file is compiled once per RANGE OF DESIGN WIDTHS (pydeseq2_b200/build.py): the base unit (PDQ_TU_P = 0) holds the kernels
// for p = 1..8, with the p x p algebra fully unrolled in registers; one further unit per wide design width p = 9..16
// (PDQ_TU_P = p) holds that width's kernels, same source, loops over the design columns not unrolled.  The units compile in
// parallel; pdq_dispatch.cu routes a launch to the unit that owns the design's width.  The kernels that do not depend on p are
// compiled once, in pdq_common.cu.
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

// ---- MAP dispersion search -> final dispersion -> LFC fit + Wald test with a per-tile dependency (DESIGN.md §4) ----------------
// The LFC fit of a gene needs that gene's final dispersion only, and the final dispersion is an elementwise function of the
// gene's MAP estimate: the dependency between the two heavy stages is per gene tile, not per grid.  k_map_irls<.., 0> is the MAP
// search (alpha_gene as in k_alpha_mle, then select_disp per gene); it publishes every warp tile with a release store of the pass
// number into tile_done[tile].  k_map_irls<.., 1> is the LFC fit (irls_gene as in k_irls); before a tile it waits for that word.
// The second kernel is a programmatic dependent launch: its blocks become resident as soon as every block of the first has
// started and an SM has room, i.e. while the last MAP tiles are still being worked on, where two ordinary launches would drain,
// run the elementwise kernel and ramp up again.  Two kernels rather than one so that each body keeps its own register budget
// (3 resident blocks per SM for the search, 4 for the fit).
//
// Control words (device ints, LaunchCfg::tickets + kTailWords), kept consistent by the kernels themselves so that the pair
// replays inside a CUDA graph without memset nodes: the last block of each kernel zeroes its ticket counter and moves its
// flagged-gene count to the word the fallback kernel behind the pair reads; the last block of the fit bumps the pass number.
// tile_done holds (pass << 1) | deferred: words of earlier passes never match, so the array is zeroed once, when it is allocated.
constexpr int kTailWords = 16;  // offset of the control words in LaunchCfg::tickets
enum { kTailTicket = 0, kTailPass = 1, kTailBlocks = 2, kTailGridCnt = 3, kTailOptCnt = 4, kTailTicket2 = 5, kTailGridOut = 6, kTailOptOut = 7,
       kTailBlocks2 = 8 };  // ...2: ticket counter and finished blocks of the LFC kernel

template <int P>
struct TailArgs {
    AlphaArgs<P> al;  // MAP search: al.alpha = MAP estimates, al.alpha_hat = trend values
    IrlsArgs<P> ir;   // LFC fit + Wald test: ir.disp = the final dispersions written by the MAP tickets
                      // (al.ticket / ir.ticket serve k_alpha_grid / k_irls_optimizer behind the launch: ticket[1] = flagged genes)
    const double* gw;       // genewise dispersions
    const TrendOut* trend;  // device record of the trend fit (squared_logres)
    double min_disp, max_disp;
    double *disp, *outlier;
    int* words;               // control words above
    unsigned* tile_done;      // one word per warp tile
    unsigned long long* err;  // mapped host word: 1 + tile when a wait gave up
    unsigned long long timeout_ns;
};

__device__ __forceinline__ void tile_lanes(int lgT, int G, int tile, Group& grp, int& gene, bool& valid) {
    const int lane = threadIdx.x & 31;
    grp.T = 1 << lgT;
    grp.gpw = 32 >> lgT;
    grp.si = lane >> (5 - lgT);
    const int gidx = tile * grp.gpw + (lane & (grp.gpw - 1));
    valid = gidx < G;
    gene = valid ? gidx : (G - 1);
}
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long tail_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// the LFC fit of one tile and its bookkeeping, shared by k_map_irls and k_irls_deferred
template <int P>
__device__ __forceinline__ void tail_irls_tile(const TailArgs<P>& a, const Group& grp, const DesignS& d, int g, bool valid, double disp,
                                               double* lg_tab, const double* logfact, int* flagged) {
    const IrlsArgs<P>& r = a.ir;
    int st = 0;
    irls_gene<P>(grp, d, r.pinv, r.prm, r.counts + g, r.ld, disp, r.beta + (int64_t)g * P, r.mu + g, r.hat + g, r.ld_out,
                 r.conv + g, &st, valid, lg_tab, logfact, r.with_wald ? &r.wald : nullptr, r.wald_p + g, r.wald_stat + g,
                 r.wald_se + g);
    if (valid && grp.si == 0) {
        if (r.force) st = kIrlsNeedsOptimizer;
        r.status[g] = st;
        if (st != kIrlsOk) atomicAdd(flagged, 1);
    }
}

template <int P, bool STAGED, int PHASE>
__global__ void __launch_bounds__(kBlock, PHASE ? PDQ_IRLS_MINB : PDQ_ALPHA_MINB) k_map_irls(const __grid_constant__ TailArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    // both kernels read the pass number before any block of the LFC kernel exists (the MAP blocks read it before they allow the
    // dependent launch), and only the LFC kernel's last block changes it
    const unsigned pass = (unsigned)*reinterpret_cast<volatile const int*>(a.words + kTailPass) + 1u;
    if (PHASE == 0) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const DesignS d = stage_design_t<true, STAGED ? 1 : 0>(a.al.dv, P, smem);
    // scratch behind the design pack, its mbarrier and the math table: the block's log(k!) table, then one slot of 2 * kPsiK doubles
    // per gene of the warp's tile -- psi / psi' tables in the MAP kernel, the lgamma(r + k) table in the LFC kernel
    double* logfact = reinterpret_cast<double*>(smem + scratch_off(a.al.dv, true));
    if (PHASE == 1) {
        if (threadIdx.x < kPsiK) logfact[threadIdx.x] = kLogFact[threadIdx.x];
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, gpw = 32 >> a.al.lgT;
    double* slot = logfact + kPsiK + (size_t)((threadIdx.x >> 5) * gpw + (lane & (gpw - 1))) * (2 * kPsiK);
    const int G = a.al.G, ntiles = (G + gpw - 1) >> (5 - a.al.lgT);
    int* ticket = a.words + (PHASE ? kTailTicket2 : kTailTicket);
    Group grp;
    int g;
    bool valid;
    int ahead = draw_ticket(ticket);
    if (PHASE == 0) {
        // a programmatic dependent of the trend kernel (launch_map_irls): everything above is independent of the trend; the
        // fitted curve and the trend record are read only behind the trend grid's completion
        asm volatile("griddepcontrol.wait;" ::: "memory");
        AlphaParams prm = a.al.prm;
        if (a.al.prior_var_dev) prm.prior_var = *a.al.prior_var_dev;
        const double sq_logres = a.trend->squared_logres;
        for (;;) {
            const int t = __shfl_sync(0xffffffffu, ahead, 0);
            if (t >= ntiles) break;
            ahead = draw_ticket(ticket);  // the next ticket's round trip to L2 hides behind this tile
            tile_lanes(a.al.lgT, G, t, grp, g, valid);
            alpha_gene<P>(grp, d, prm, a.al.counts + g, a.al.ld, a.al.mu + g, a.al.ld_mu, a.al.alpha_hat[g], a.al.alpha + g,
                          a.al.conv + g, a.al.status + g, valid, slot, a.al.hint_in ? a.al.hint_in + 2 * (int64_t)g : nullptr,
                          nullptr);
            bool defer = false;
            if (valid && grp.si == 0) {
                if (a.al.force) {
                    a.al.status[g] = kAlphaNeedsGrid;
                    a.al.conv[g] = 0.0;
                }
                if (a.al.status[g] == kAlphaNeedsGrid) {
                    atomicAdd(a.words + kTailGridCnt, 1);
                    defer = true;
                } else {
                    bool out;
                    a.disp[g] = select_disp(a.gw[g], a.al.alpha[g], a.al.alpha_hat[g], sq_logres, a.min_disp, a.max_disp, out);
                    if (a.outlier) a.outlier[g] = out ? 1.0 : 0.0;
                }
            }
            // a tile with a gene left to the grid fallback is published as deferred: the LFC kernel skips it, and k_alpha_grid +
            // k_irls_deferred behind the pair finish it
            defer = __any_sync(0xffffffffu, defer);
            __threadfence();
            __syncwarp();  // every lane's stores of the tile are ordered before lane 0's release
            if (lane == 0) st_release_gpu(a.tile_done + t, (pass << 1) | (defer ? 1u : 0u));
        }
    } else {
        for (;;) {
            const int tile = __shfl_sync(0xffffffffu, ahead, 0);
            if (tile >= ntiles) break;
            ahead = draw_ticket(ticket);
            // Every wait ends: a block of this kernel exists only after every block of the MAP kernel has started (programmatic
            // dependent launch), so every MAP block is resident or done; MAP tiles never wait and their tickets are drawn by running
            // warps only, so every tile is published.  Both kernels walk the tiles in increasing order, so the wait is short.  The
            // time limit only turns a logic error into a reported failure (pdq_map_irls_status) instead of a hung device.
            unsigned v = 0;
            if (lane == 0) {
                v = ld_acquire_gpu(a.tile_done + tile);
                if ((v >> 1) != pass) {
                    const unsigned long long t0 = tail_timer_ns();
                    do {
                        __nanosleep(200);
                        v = ld_acquire_gpu(a.tile_done + tile);
                    } while ((v >> 1) != pass && tail_timer_ns() - t0 <= a.timeout_ns);
                    if ((v >> 1) != pass) {
                        *a.err = 1ULL + (unsigned long long)tile;
                        __threadfence_system();
                    }
                }
            }
            v = __shfl_sync(0xffffffffu, v, 0);
            __syncwarp();
            if ((v >> 1) != pass || (v & 1u)) continue;
            tile_lanes(a.al.lgT, G, tile, grp, g, valid);
            tail_irls_tile<P>(a, grp, d, g, valid, __ldcg(a.ir.disp + g), slot, logfact, a.words + kTailOptCnt);
        }
        // the MAP kernel has completed and its writes (the count of flagged genes, its control words) are visible before this
        // kernel completes: what follows in the stream is ordered behind both
        asm volatile("griddepcontrol.wait;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(a.words + (PHASE ? kTailBlocks2 : kTailBlocks), 1) == (int)gridDim.x - 1) {  // the kernel's last block
            if (PHASE == 0) {
                a.words[kTailGridOut] = atomicExch(a.words + kTailGridCnt, 0);
                a.words[kTailTicket] = 0;
                a.words[kTailBlocks] = 0;
            } else {
                a.words[kTailOptOut] = atomicExch(a.words + kTailOptCnt, 0);
                a.words[kTailTicket2] = 0;
                a.words[kTailBlocks2] = 0;
                a.words[kTailPass] = (int)pass;
            }
        }
    }
}

// The tiles the MAP kernel published as deferred, behind k_alpha_grid (which has replaced the MAP estimate of their flagged genes):
// final dispersions of the tile's genes, then the LFC fit.  Normally no tile is deferred: one wave of blocks that read the count
// of flagged genes and exit.
template <int P>
__global__ void __launch_bounds__(kBlock) k_irls_deferred(const __grid_constant__ TailArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    if (*reinterpret_cast<volatile const int*>(a.words + kTailGridOut) == 0) return;
    const DesignS d = stage_design_t<true, -1>(a.al.dv, P, smem);
    double* logfact = reinterpret_cast<double*>(smem + scratch_off(a.al.dv, true));
    if (threadIdx.x < kPsiK) logfact[threadIdx.x] = kLogFact[threadIdx.x];
    __syncthreads();
    const unsigned mark = ((unsigned)a.words[kTailPass] << 1) | 1u;  // the pass number the pair left behind is its own
    const double sq_logres = a.trend->squared_logres;
    const int lane = threadIdx.x & 31, gpw = 32 >> a.al.lgT;
    double* slot = logfact + kPsiK + (size_t)((threadIdx.x >> 5) * gpw + (lane & (gpw - 1))) * (2 * kPsiK);
    const int G = a.al.G, ntiles = (G + gpw - 1) >> (5 - a.al.lgT);
    for (int tile = blockIdx.x * kWarps + (threadIdx.x >> 5); tile < ntiles; tile += gridDim.x * kWarps) {
        if (a.tile_done[tile] != mark) continue;
        Group grp;
        int g;
        bool valid;
        tile_lanes(a.al.lgT, G, tile, grp, g, valid);
        bool out;
        const double disp = select_disp(a.gw[g], a.al.alpha[g], a.al.alpha_hat[g], sq_logres, a.min_disp, a.max_disp, out);
        if (valid && grp.si == 0) {
            a.disp[g] = disp;
            if (a.outlier) a.outlier[g] = out ? 1.0 : 0.0;
        }
        tail_irls_tile<P>(a, grp, d, g, valid, disp, slot, logfact, a.words + kTailOptOut);
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
struct WaldContrastsArgs {
    DesignView dv;
    double ridge[P * P];
    const double* tab;  // (K, P + 2): contrast, lfc_null, alt
    const double *disp, *lfc;
    int G, lgT, K;
    double *pv, *stat, *se;  // (K, ld_out)
    int64_t ld_out;
};

template <int P>
__global__ void __launch_bounds__(kBlock) k_wald_contrasts(const __grid_constant__ WaldContrastsArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    wald_contrasts_gene<P>(grp, d, a.ridge, a.disp[g], a.lfc + (int64_t)g * P, a.K, a.tab, a.pv + g, a.stat + g, a.se + g, a.ld_out,
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

// ---- method-of-moments start values folded into the genewise dispersion search (lin_reg_mu branch of the resident pass) --------
// k_mom_from_counts and k_alpha_mle are per-gene functions with the same lane layout, and the search of a gene needs only that gene's
// start value and initial means.  k_mom_alpha runs mom_fused_gene on each ticket tile and then alpha_gene on the same tile: the
// start value stays in registers, and every lane reads back the means it has just stored.  One launch instead of a grid that drains
// and a second that ramps up and reads the counts again; mom, means and mu_hat still go to HBM for the stages behind the search.
// Control words (LaunchCfg::tickets + kFoldWords) are kept consistent by the kernel itself, as in k_map_irls: the last block zeroes
// the ticket counter and moves the count of flagged genes to the word k_alpha_grid reads, so the launch needs no memset node.
constexpr int kFoldWords = 25;  // offset of the control words in LaunchCfg::tickets (behind the words of k_map_irls)
enum { kFoldTicket = 0, kFoldGridCnt = 1, kFoldBlocks = 2, kFoldGridOut = 3 };

template <int P>
struct MomAlphaArgs {
    AlphaArgs<P> al;  // genewise search: al.mu = mu_hat, al.alpha_hat unused; al.ticket + 1 = the flagged-gene word of k_alpha_grid
    SmallMat<P> pinv;
    double s_mean_inv, min_disp, max_disp, min_mu;  // start values: clip bounds of dds.py:1161, floor of lin_reg_mu
    double *mom, *means, *mu_hat;
    int* words;  // control words above
};

template <int P, bool STAGED>
__global__ void __launch_bounds__(kBlock, PDQ_ALPHA_MINB) k_mom_alpha(const __grid_constant__ MomAlphaArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design_t<true, STAGED ? 1 : 0>(a.al.dv, P, smem);
    Group grp;
    int g;
    bool valid;
    const int gpw = 32 >> a.al.lgT;
    double* psi = reinterpret_cast<double*>(smem + scratch_off(a.al.dv, true)) +
                  (size_t)((threadIdx.x >> 5) * gpw + ((threadIdx.x & 31) & (gpw - 1))) * (2 * kPsiK);
    int* ticket = a.words + kFoldTicket;
    int ahead = draw_ticket(ticket);
    while (next_tile(ticket, a.al.lgT, a.al.G, grp, g, valid, ahead, a.al.descending != 0)) {
        const double alpha_hat = mom_fused_gene<P>(grp, d, a.pinv, a.al.counts + g, a.al.ld, a.s_mean_inv, a.min_disp, a.max_disp,
                                                   a.min_mu, a.mom + g, a.means + g, a.mu_hat + g, a.al.ld_mu, valid);
        // lanes of padding genes (clamped to gene G - 1) read the means another group of this warp has just stored
        __syncwarp();
        alpha_gene<P>(grp, d, a.al.prm, a.al.counts + g, a.al.ld, a.mu_hat + g, a.al.ld_mu, alpha_hat, a.al.alpha + g, a.al.conv + g,
                      a.al.status + g, valid, psi, nullptr, a.al.hint_out ? a.al.hint_out + 2 * (int64_t)g : nullptr);
        if (valid && grp.si == 0) {
            if (a.al.force) {
                a.al.status[g] = kAlphaNeedsGrid;
                a.al.conv[g] = 0.0;
            }
            if (a.al.status[g] == kAlphaNeedsGrid) atomicAdd(a.words + kFoldGridCnt, 1);
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(a.words + kFoldBlocks, 1) == (int)gridDim.x - 1) {  // the kernel's last block
            a.words[kFoldGridOut] = atomicExch(a.words + kFoldGridCnt, 0);
            a.words[kFoldTicket] = 0;
            a.words[kFoldBlocks] = 0;
        }
    }
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
    double* ws;  // null: the cell plan and the genes' cell members in shared memory; else the members in ws, one slot per gene
};

// Cook's distances + trimmed-moments dispersions (dds.py:986-1040); the gene's cell members are staged in shared memory, or in
// the global workspace where they do not fit (cooks_in_smem)
template <int P>
__global__ void __launch_bounds__(kBlock) k_cooks(const __grid_constant__ CooksArgs<P> a) {
    extern __shared__ __align__(128) unsigned char smem[];
    const DesignS d = stage_design(a.dv, P, smem);
    int* plan_s = reinterpret_cast<int*>(smem + scratch_off(a.dv, false));
    if (!a.ws)
        for (int i = threadIdx.x; i < a.plan_len; i += blockDim.x) plan_s[i] = a.plan[i];
    __syncthreads();
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    const int* pl = a.ws ? a.plan : plan_s;
    const CellPlan plan{pl + 2 + a.n_cells + 1, pl + 2, a.n_cells, pl[1]};
    const size_t plan_bytes = ((size_t)a.plan_len * 4 + 15) & ~(size_t)15;
    const int gslot = (threadIdx.x >> 5) * grp.gpw + ((threadIdx.x & 31) & (grp.gpw - 1));
    // the slots of the lanes map_lanes marks invalid lie past G - 1's: they never share one with a valid gene
    double* vals = a.ws ? a.ws + ((size_t)blockIdx.x * kWarps * grp.gpw + gslot) * 2 * a.n_in_cells
                        : reinterpret_cast<double*>(smem + scratch_off(a.dv, false) + plan_bytes) + (size_t)gslot * 2 * a.n_in_cells;
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

// ---- launch helpers ---------------------------------------------------------------------------------
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

inline DesignView view_of(const DesignDev& d) { return DesignView{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}; }

// a kernel whose blocks take the genes map_lanes gives them, one block per kWarps warp tiles
template <class A>
int launch_genes(const LaunchCfg& c, void (*kernel)(A), const A& a, size_t smem, int G) {
    if (int e = prep(kernel, smem)) return e;
    kernel<<<grid_for(G, c.lgT), kBlock, smem, c.stream>>>(a);
    return 0;
}

// The persistent kernels are compiled for a staged pack and for one read from global memory: `kernel(std::bool_constant<STAGED>)`
// names an instantiation, and the one for d.staged is prepped and launched on its persistent grid -- every block the machine can
// hold at once, but no more blocks than warp tiles need.  `dependent`: a programmatic dependent launch (see k_map_irls).
template <class A, class F>
int launch_persistent(const LaunchCfg& c, const DesignDev& d, size_t smem, int G, const A& a, F kernel, bool dependent = false) {
    auto go = [&](auto k) -> int {
        if (int e = prep(k, smem)) return e;
        int per_sm = 1;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kBlock, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
        const int need = grid_for(G, c.lgT), fit = per_sm * c.sm_count;
        const unsigned grid = (unsigned)(need < fit ? need : fit);
        if (!dependent) {
            k<<<grid, kBlock, smem, c.stream>>>(a);
            return 0;
        }
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = 1;
        cudaLaunchConfig_t lc = {dim3(grid), dim3(kBlock), smem, c.stream, at, 1};
        return cudaLaunchKernelEx(&lc, k, a) == cudaSuccess ? 0 : PDQ_ERR_CUDA;
    };
    return d.staged ? go(kernel(std::true_type{})) : go(kernel(std::false_type{}));
}

template <int P>
SmallMat<P> pinv_of(const DesignDev& d) {
    SmallMat<P> m;
    for (int i = 0; i < P * P; ++i) m.v[i] = d.pinv[i];
    return m;
}

template <int P>
WaldParams<P> wald_params(const WaldHost& w) {
    WaldParams<P> prm;
    for (int i = 0; i < P * P; ++i) prm.ridge[i] = w.ridge[i];
    for (int i = 0; i < P; ++i) prm.contrast[i] = w.contrast[i];
    prm.lfc_null = w.lfc_null;
    prm.alt = w.alt;
    return prm;
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

// the grid fallback of two-column designs (utils.py:1125-1141) for the genes k_lfc_shrink flagged
template <int P>
__global__ void __launch_bounds__(kBlock) k_lfc_shrink_grid(const __grid_constant__ ShrinkArgs<P> a) {
    static_assert(P == 2, "apeGLM's grid fallback is for two-column designs");
    extern __shared__ __align__(128) unsigned char smem[];
    Group grp;
    int g;
    bool valid;
    map_lanes(a.lgT, a.G, grp, g, valid);
    const bool run = valid && a.status[g] == kShrinkNeedsGrid;
    if (!__syncthreads_or(run)) return;
    const DesignS d = stage_design(a.dv, P, smem);
    if (!__any_sync(0xffffffffu, run)) return;
    shrink_grid_gene(grp, d, a.prm, a.counts + g, a.ld, a.size[g], a.beta + (int64_t)g * P, a.ih + (int64_t)g * P * P, run);
}

// k_lfc_shrink_grid behind k_lfc_shrink, instantiated for two-column designs only
template <int P>
int launch_shrink_grid(const LaunchCfg& c, const DesignDev& d, const ShrinkArgs<P>& a, int G) {
    if constexpr (P == 2) return launch_genes(c, k_lfc_shrink_grid<P>, a, d.smem_bytes, G);
    return 0;
}

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

}  // namespace

int PDQ_TUFN(launch_lin_reg_mu)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_mu,
                      double* mu_out, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        LinMuArgs<P> a{view_of(d), pinv_of<P>(d), counts, ld, G, c.lgT, min_mu, mu_out, ld_out};
        if (int e = launch_genes(c, k_lin_reg_mu<P>, a, d.smem_bytes, G)) return e;
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
        a.dv = view_of(d);
        a.pinv = pinv_of<P>(d);
        a.prm = irls_params(h, d, c.debug);
        a.counts = counts; a.ld = ld; a.G = G; a.lgT = c.lgT; a.disp = disp;
        a.beta = beta; a.mu = mu; a.hat = hat; a.conv = conv; a.ld_out = ld_out;
        a.status = status; a.n_fallback = n_fallback; a.ticket = c.tickets;
        a.force = hook(c.debug, PDQ_DEBUG_FORCE_IRLS_OPTIMIZER);
        a.with_wald = w ? 1 : 0;
        a.wald_p = a.wald_stat = a.wald_se = nullptr;
        if (w) {
            a.wald = wald_params<P>(*w);
            a.wald_p = w->pv; a.wald_stat = w->stat; a.wald_se = w->se;
        }
        const size_t smem_irls = d.smem_bytes + kMathTabBytes + (size_t)(1 + kWarps * (32 >> c.lgT)) * kPsiK * sizeof(double);
        if (int e = prep(k_irls_optimizer<P>, d.smem_bytes)) return e;
        if (cudaMemsetAsync(c.tickets, 0, 2 * sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
        if (int e = launch_persistent(c, d, smem_irls, G, a, [](auto s) { return k_irls<P, decltype(s)::value>; })) return e;
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
        AlphaArgs<P> a{view_of(d), alpha_params(min_disp, max_disp, prior_var, cr_reg, prior_reg), counts, ld, G, c.lgT, mu, ld_mu,
                       alpha_hat, alpha, conv, status, prior_var_dev, c.tickets + 2, hook(c.debug, PDQ_DEBUG_FORCE_ALPHA_GRID), hint_in, hint_out,
                       alpha_descending()};
        const size_t smem_alpha = d.smem_bytes + kMathTabBytes + (size_t)kWarps * (32 >> c.lgT) * 2 * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (cudaMemsetAsync(c.tickets + 2, 0, 2 * sizeof(int), c.stream) != cudaSuccess) return PDQ_ERR_CUDA;
        if (int e = launch_persistent(c, d, smem_alpha, G, a, [](auto s) { return k_alpha_mle<P, decltype(s)::value>; })) return e;
        k_alpha_grid<P><<<fallback_grid(c.sm_count, G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
    });
    if (int e = check_launch()) return e;
    return 2;
}

int PDQ_TUFN(launch_map_irls)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const TailHost& t,
                              const IrlsHost& h, const WaldHost& w) {
    PDQ_DISPATCH_P(d.p, {
        TailArgs<P> a;
        int* words = c.tickets + kTailWords;
        // the fallback kernels read the count of flagged genes at ticket[1]: the words the last blocks of k_map_irls fill
        a.al = AlphaArgs<P>{view_of(d), alpha_params(t.min_disp, t.max_disp, t.prior_var, 1, 1), counts, ld, G, c.lgT, t.mu, t.ld_mu,
                            t.fitted, t.map, t.map_conv, t.status_map, t.prior_var_dev, words + kTailGridOut - 1,
                            hook(c.debug, PDQ_DEBUG_FORCE_ALPHA_GRID), t.hint_in, nullptr, 0};
        a.ir.dv = view_of(d);
        a.ir.pinv = pinv_of<P>(d);
        a.ir.prm = irls_params(h, d, c.debug);
        a.ir.counts = counts; a.ir.ld = ld; a.ir.G = G; a.ir.lgT = c.lgT; a.ir.disp = t.disp;
        a.ir.beta = t.beta; a.ir.mu = t.mu_out; a.ir.hat = t.hat; a.ir.conv = t.conv; a.ir.ld_out = t.ld_out;
        a.ir.status = t.status_irls; a.ir.n_fallback = nullptr; a.ir.ticket = words + kTailOptOut - 1;
        a.ir.force = hook(c.debug, PDQ_DEBUG_FORCE_IRLS_OPTIMIZER);
        a.ir.with_wald = 1;
        a.ir.wald = wald_params<P>(w);
        a.ir.wald_p = w.pv; a.ir.wald_stat = w.stat; a.ir.wald_se = w.se;
        a.gw = t.gw; a.trend = reinterpret_cast<const TrendOut*>(t.trend16);
        a.min_disp = t.min_disp; a.max_disp = t.max_disp; a.disp = t.disp; a.outlier = t.outlier;
        a.words = words; a.tile_done = t.tile_done; a.err = t.err; a.timeout_ns = 20000000000ULL;
        const size_t smem_tail = d.smem_bytes + kMathTabBytes + (size_t)(1 + 2 * kWarps * (32 >> c.lgT)) * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (int e = prep(k_irls_deferred<P>, smem_tail)) return e;
        if (int e = prep(k_irls_optimizer<P>, d.smem_bytes)) return e;
        // the MAP kernel as a programmatic dependent of what precedes it in the stream (the trend kernel in the resident pass), then
        // the LFC kernel as the MAP kernel's (see k_map_irls).  Invariant: what the MAP kernel reads before its griddepcontrol.wait --
        // the pass word, its ticket, the design pack -- is written by no kernel that triggers its dependents early.  Today the only
        // kernels that do are k_trend_prior / k_trend_prior_grid (which write none of these) and the MAP kernel itself (whose
        // dependent is the LFC kernel); any other predecessor completes, writes included, before the MAP kernel starts
        if (int e = launch_persistent(c, d, smem_tail, G, a, [](auto s) { return k_map_irls<P, decltype(s)::value, 0>; }, true)) return e;
        if (int e = launch_persistent(c, d, smem_tail, G, a, [](auto s) { return k_map_irls<P, decltype(s)::value, 1>; }, true)) return e;
        const int wave = fallback_grid(c.sm_count, G, c.lgT);
        k_alpha_grid<P><<<wave, kBlock, d.smem_bytes, c.stream>>>(a.al);
        k_irls_deferred<P><<<wave, kBlock, smem_tail, c.stream>>>(a);
        k_irls_optimizer<P><<<wave, kBlock, d.smem_bytes, c.stream>>>(a.ir);
    });
    if (int e = check_launch()) return e;
    return 5;
}

int PDQ_TUFN(launch_wald)(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, const double* mu,
                int64_t ld_mu, int G, const double* ridge, const double* contrast, double lfc_null, int alt, double* pv,
                double* stat, double* se) {
    PDQ_DISPATCH_P(d.p, {
        WaldArgs<P> a;
        a.dv = view_of(d);
        a.prm = wald_params<P>(WaldHost{ridge, contrast, lfc_null, alt, pv, stat, se});
        a.disp = disp; a.lfc = lfc; a.mu = mu; a.ld_mu = ld_mu; a.G = G; a.lgT = c.lgT;
        a.pv = pv; a.stat = stat; a.se = se;
        if (int e = launch_genes(c, k_wald<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_wald_contrasts)(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, int G,
                                    const double* ridge, int K, const double* tab, double* pv, double* stat, double* se, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        WaldContrastsArgs<P> a;
        a.dv = view_of(d);
        for (int i = 0; i < P * P; ++i) a.ridge[i] = ridge[i];
        a.tab = tab;
        a.disp = disp; a.lfc = lfc; a.G = G; a.lgT = c.lgT; a.K = K;
        a.pv = pv; a.stat = stat; a.se = se; a.ld_out = ld_out;
        if (int e = launch_genes(c, k_wald_contrasts<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_rough)(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{view_of(d), pinv_of<P>(d), normed, nullptr, ld, G, c.lgT, d.s_mean_inv, 0.0, 0.0, alpha,
                     nullptr, 0.0, nullptr, 0};
        if (int e = launch_genes(c, k_rough<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_moments)(const LaunchCfg& c, const DesignDev& d, const double* normed, int64_t ld, int G, double* alpha,
                   double* all_zero) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{view_of(d), pinv_of<P>(d), normed, nullptr, ld, G, c.lgT, d.s_mean_inv, 0.0, 0.0, alpha,
                     all_zero, 0.0, nullptr, 0};
        if (int e = launch_genes(c, k_moments<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_mom_from_counts)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G,
                           double min_disp, double max_disp, double* alpha, double* normed_mean, double min_mu, double* mu_hat,
                           int64_t ld_mu) {
    PDQ_DISPATCH_P(d.p, {
        MomArgs<P> a{view_of(d), pinv_of<P>(d), nullptr, counts, ld, G, c.lgT, d.s_mean_inv, min_disp,
                     max_disp, alpha, normed_mean, min_mu, mu_hat, ld_mu};
        if (int e = launch_genes(c, k_mom_from_counts<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_mom_alpha)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_disp,
                               double max_disp, double min_mu, double* mom, double* normed_mean, double* mu_hat, int64_t ld_mu,
                               double* alpha, double* conv, int* status, double* hint_out) {
    PDQ_DISPATCH_P(d.p, {
        MomAlphaArgs<P> a;
        int* words = c.tickets + kFoldWords;
        // genewise search (cr_reg on, no prior); k_alpha_grid behind the launch reads the flagged-gene count at ticket[1] =
        // the word the kernel's last block fills
        a.al = AlphaArgs<P>{view_of(d), alpha_params(min_disp, max_disp, 1.0, 1, 0), counts, ld, G, c.lgT, mu_hat, ld_mu, mom, alpha,
                            conv, status, nullptr, words + kFoldGridOut - 1, hook(c.debug, PDQ_DEBUG_FORCE_ALPHA_GRID), nullptr, hint_out,
                            alpha_descending()};
        a.pinv = pinv_of<P>(d);
        a.s_mean_inv = d.s_mean_inv; a.min_disp = min_disp; a.max_disp = max_disp; a.min_mu = min_mu;
        a.mom = mom; a.means = normed_mean; a.mu_hat = mu_hat; a.words = words;
        const size_t smem_alpha = d.smem_bytes + kMathTabBytes + (size_t)kWarps * (32 >> c.lgT) * 2 * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (int e = launch_persistent(c, d, smem_alpha, G, a, [](auto s) { return k_mom_alpha<P, decltype(s)::value>; })) return e;
        k_alpha_grid<P><<<fallback_grid(c.sm_count, G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a.al);
    });
    if (int e = check_launch()) return e;
    return 2;
}

int PDQ_TUFN(launch_mu_from_lfc)(const LaunchCfg& c, const DesignDev& d, const double* lfc, int G, double* mu, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        MuLfcArgs<P> a{view_of(d), lfc, G, c.lgT, mu, ld_out};
        if (int e = launch_genes(c, k_mu_from_lfc<P>, a, d.smem_bytes, G)) return e;
    });
    if (int e = check_launch()) return e;
    return 1;
}

int PDQ_TUFN(launch_cooks)(const LaunchCfg& c0, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* mu, const double* hat,
                 int64_t ld2, double cutoff, double* cooks, int64_t ld_out, double* disp, double* outlier, double* replaced, double* ws) {
    // the per-gene staging (2 * n_in_cells doubles) bounds the genes per block: widen the lane groups until it fits, and past 32
    // lanes stage in the workspace, cooks_chunk genes per launch
    LaunchCfg c = c0;
    while (c.lgT < 5 && cooks_smem(d, c.lgT) > 96 * 1024) ++c.lgT;
    const bool global = !cooks_in_smem(d);
    const int chunk = global ? cooks_chunk(d) : G;
    if (global && (!ws || chunk < 1)) return PDQ_ERR_UNSUPPORTED;
    int launches = 0;
    PDQ_DISPATCH_P(d.p, {
        for (int g0 = 0; g0 < G; g0 += chunk, ++launches) {
            const int n = G - g0 < chunk ? G - g0 : chunk;
            CooksArgs<P> a{view_of(d), d.cell_plan, d.plan_len, d.n_cells, d.n_in_cells, counts + g0, ld, n, c.lgT, mu + g0, hat + g0, ld2,
                           cutoff, cooks ? cooks + g0 : nullptr, ld_out, disp + g0, outlier + g0, replaced + g0, global ? ws : nullptr};
            if (int e = launch_genes(c, k_cooks<P>, a, global ? d.smem_bytes : cooks_smem(d, c.lgT), n)) return e;
        }
    });
    if (int e = check_launch()) return e;
    return launches;
}

int PDQ_TUFN(launch_lfc_shrink)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const double* size,
                      double prior_no_shrink_scale, double prior_scale, int shrink_index, double* beta, double* inv_hessian,
                      double* conv, int* status) {
    if (shrink_index < 0 || shrink_index >= d.p) return PDQ_ERR_INVALID;
    const ShrinkParams prm{1.0 / (prior_no_shrink_scale * prior_no_shrink_scale), prior_scale * prior_scale, shrink_index};
    const int force = hook(c.debug, PDQ_DEBUG_FORCE_SHRINK_GRID);
    PDQ_DISPATCH_P(d.p, {
        ShrinkArgs<P> a{view_of(d), prm, counts, ld, G, c.lgT, size, beta, inv_hessian, conv, status, force};
        if (int e = launch_genes(c, k_lfc_shrink<P>, a, d.smem_bytes, G)) return e;
        if (int e = launch_shrink_grid<P>(c, d, a, G)) return e;
    });
    if (int e = check_launch()) return e;
    return d.p == 2 ? 2 : 1;
}

}  // namespace pdq
