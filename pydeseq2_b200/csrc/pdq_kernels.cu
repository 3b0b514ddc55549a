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
#include "pdq_vst.cuh"
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
    unsigned* vmerged = nullptr;              // [2][kVBins] (median_bins only)
    unsigned* sel_words = nullptr;            // [2]: candidate cursors (median_bins only)
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
    // the last `kmax` of the k values are maxima, not sums (same exchange)
    __host__ __device__ void sum_many(double* v, int k, int kmax = 0) {
#if defined(__CUDA_ARCH__)
        namespace cg = cooperative_groups;
        cg::cluster_group cluster = cg::this_cluster();
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ks = k - kmax;
        for (int j = 0; j < k; ++j) {
            double w = v[j];
            if (j < ks) {
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
            } else {
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) w = fmax(w, __shfl_xor_sync(0xffffffffu, w, off));
            }
            if (lane == 0) warp_part[warp * kTrendK + j] = w;
        }
        __syncthreads();
        if ((int)threadIdx.x < ks) {
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
        if ((int)threadIdx.x >= ks && (int)threadIdx.x < k) {
            double m = warp_part[threadIdx.x];
            const int nw = blockDim.x >> 5;
            for (int w = 1; w < nw; ++w) m = fmax(m, warp_part[w * kTrendK + threadIdx.x]);
            if (nblocks > 1) {
                for (unsigned r = 0; r < nblocks; ++r)
                    cluster.map_shared_rank(slots, r)[(parity * kTrendMaxCluster + rank) * kTrendK + threadIdx.x] = m;
            } else {
                slots[parity * kTrendMaxCluster * kTrendK + threadIdx.x] = m;
            }
        }
        if (nblocks > 1) cluster.sync(); else __syncthreads();  // release the DSMEM stores / acquire the peers'
        // k threads add up the blocks' slots, everybody reads the k totals (broadcast reads).  Having EVERY thread
        // add nblocks * k slots itself would cost 160 shared-memory reads per thread and pass.
        if ((int)threadIdx.x < ks) {
            double tot = 0.0;
            for (unsigned r = 0; r < nblocks; ++r) tot += slots[(parity * kTrendMaxCluster + r) * kTrendK + threadIdx.x];
            totals[parity * kTrendK + threadIdx.x] = tot;
        } else if ((int)threadIdx.x < k) {
            double m = slots[parity * kTrendMaxCluster * kTrendK + threadIdx.x];
            for (unsigned r = 1; r < nblocks; ++r) m = fmax(m, slots[(parity * kTrendMaxCluster + r) * kTrendK + threadIdx.x]);
            totals[parity * kTrendK + threadIdx.x] = m;
        }
        __syncthreads();
        for (int j = 0; j < k; ++j) v[j] = totals[parity * kTrendK + j];
        parity ^= 1;
#else
        (void)v;
        (void)k;
        (void)kmax;
#endif
    }
#if defined(__CUDA_ARCH__)
    // median_bins hooks.  Bin j of the merged histogram lives in block j / (kVBins / nblocks) of the cluster (vmerged[slot]):
    // every block adds its non-zero bins there with DSMEM atomics, meets the others at one cluster barrier and reads the totals
    // back.  The candidate cursor lives in block 0 (sel_words[slot]).  Both are zeroed at the start of the kernel, and each slot
    // serves one selection per launch.
    __device__ void vhist_merge(unsigned* hist, int slot) {
        __syncthreads();  // local bins complete
        if (nblocks == 1) return;
        namespace cg = cooperative_groups;
        cg::cluster_group cluster = cg::this_cluster();
        const unsigned chunk = kVBins / nblocks;
        unsigned* merged = vmerged + slot * kVBins;
        for (unsigned j = threadIdx.x; j < (unsigned)kVBins; j += blockDim.x) {
            const unsigned c = hist[j];
            if (c) atomicAdd(cluster.map_shared_rank(merged, j / chunk) + j, c);
        }
        cluster.sync();
        for (unsigned j = threadIdx.x; j < (unsigned)kVBins; j += blockDim.x) hist[j] = cluster.map_shared_rank(merged, j / chunk)[j];
        __syncthreads();
    }
    __device__ unsigned cand_index(int slot) {
        return atomicAdd(cooperative_groups::this_cluster().map_shared_rank(sel_words + slot, 0), 1u);
    }
    // cluster-wide maximum of one 64-bit key per thread, as integers, through the slot exchange of max_one (the bits ride in
    // the double slots untouched).  Not a DSMEM atomicMax: a 64-bit max on shared memory has no native instruction, and the
    // compiler's fallback for a generic address (QSPC + an ATOMS compare-and-swap loop) does not reach a peer block's memory
    __device__ unsigned long long max_key(unsigned long long v) {
        namespace cg = cooperative_groups;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, off);
            v = o > v ? o : v;
        }
        if (lane == 0) warp_part[warp * kTrendK] = __longlong_as_double((long long)v);
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long m = 0ull;
            const int nw = blockDim.x >> 5;
            for (int w = 0; w < nw; ++w) {
                const unsigned long long o = (unsigned long long)__double_as_longlong(warp_part[w * kTrendK]);
                m = o > m ? o : m;
            }
            const double mb = __longlong_as_double((long long)m);
            if (nblocks > 1) {
                cg::cluster_group cluster = cg::this_cluster();
                for (unsigned r = 0; r < nblocks; ++r) cluster.map_shared_rank(slots, r)[(parity * kTrendMaxCluster + rank) * kTrendK] = mb;
            } else {
                slots[parity * kTrendMaxCluster * kTrendK] = mb;
            }
        }
        if (nblocks > 1) cg::this_cluster().sync(); else __syncthreads();
        unsigned long long m = 0ull;
        for (unsigned r = 0; r < nblocks; ++r) {
            const unsigned long long o = (unsigned long long)__double_as_longlong(slots[(parity * kTrendMaxCluster + r) * kTrendK]);
            m = o > m ? o : m;
        }
        parity ^= 1;
        return m;
    }
#endif
};

__global__ void __launch_bounds__(1024) k_trend_prior(const double* __restrict__ x, const double* __restrict__ t,
                                                      double* scratch /* 3 n doubles: xs | ts | res */, size_t n,
                                                      int x_is_mean, double lo, double hi, int outer, double min_disp,
                                                      double trigamma_c, int with_prior, TrendOut* out) {
    __shared__ double warp_part[32 * kTrendK];
    __shared__ double slots[2 * kTrendMaxCluster * kTrendK];
    __shared__ double totals[2 * kTrendK];
    __shared__ unsigned hist[514];
    __shared__ SelShared sel;
    __shared__ unsigned vmerged[2 * kVBins];
    __shared__ unsigned sel_words[2];
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    ClusterReducer red{warp_part, slots, totals, cluster.block_rank(), cluster.num_blocks(), 0, vmerged, sel_words};
    for (int j = threadIdx.x; j < 2 * kVBins; j += blockDim.x) vmerged[j] = 0;  // first used behind the fit's cluster barriers
    if (threadIdx.x < 2) sel_words[threadIdx.x] = 0;
    double *xs = scratch, *ts = scratch + n, *res = scratch + 2 * n;
    trend_prepare(red, x, t, n, x_is_mean != 0, lo, hi, xs, ts);
    TrendOut o = trend_fit_outer(red, xs, ts, n, outer != 0, false);
    // the prior's candidate buffer reuses xs, last read by the fit before the prior's first cluster barrier
    if (with_prior && o.status == 0.0)
        trend_prior_dev(red, x, t, n, lo, hi, min_disp, trigamma_c, res, reinterpret_cast<unsigned long long*>(xs), sel, hist, o);
    else
        red.sum_many(&o.n_used, 1);
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
    unsigned long long maxkey[3][2];
    unsigned hist[3][256];
    unsigned vhist[2][kVBins];        // median_bins: merged value bins and candidate cursors, one slot per selection of the launch
    unsigned cursor[2];
};
static_assert(sizeof(GridScratch) <= kGridScratchBytes, "GridScratch outgrew the context's allocation");

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
    // the last `kmax` (<= 2) of the k values are maxima, not sums: they go through the maxkey slots as order-preserving keys
    __device__ void sum_many(double* v, int k, int kmax = 0) {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, slot = p_sum % 3, mslot = p_max % 3, ks = k - kmax;
        for (int j = 0; j < k; ++j) {
            double w = v[j];
            if (j < ks) {
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) w += __shfl_xor_sync(0xffffffffu, w, off);
            } else {
#pragma unroll
                for (int off = 16; off > 0; off >>= 1) w = fmax(w, __shfl_xor_sync(0xffffffffu, w, off));
            }
            if (lane == 0) warp_part[warp * kTrendK + j] = w;
        }
        __syncthreads();
        if ((int)threadIdx.x < ks) {
            double tot = 0.0;
            const int nw = blockDim.x >> 5;
            for (int w = 0; w < nw; ++w) tot += warp_part[w * kTrendK + threadIdx.x];
            atomicAdd(&gs->acc[slot][threadIdx.x], tot);
        } else if ((int)threadIdx.x < k) {
            double m = warp_part[threadIdx.x];
            const int nw = blockDim.x >> 5;
            for (int w = 1; w < nw; ++w) m = fmax(m, warp_part[w * kTrendK + threadIdx.x]);
            atomicMax(&gs->maxkey[mslot][threadIdx.x - ks], (unsigned long long)f64_key(m));
        }
        cooperative_groups::this_grid().sync();
        if ((int)threadIdx.x < ks) totals[threadIdx.x] = *reinterpret_cast<volatile double*>(&gs->acc[slot][threadIdx.x]);
        else if ((int)threadIdx.x < k)
            totals[threadIdx.x] = f64_from_key(*reinterpret_cast<volatile unsigned long long*>(&gs->maxkey[mslot][threadIdx.x - ks]));
        if (blockIdx.x == 0 && (int)threadIdx.x < kTrendK) gs->acc[(p_sum + 2) % 3][threadIdx.x] = 0.0;
        if (kmax && blockIdx.x == 0 && threadIdx.x < 2) gs->maxkey[(p_max + 2) % 3][threadIdx.x] = 0ull;
        __syncthreads();
        for (int j = 0; j < k; ++j) v[j] = totals[j];
        __syncthreads();  // totals is overwritten by the next reduction
        ++p_sum;
        if (kmax) ++p_max;
    }
    __device__ double max_one(double v) {
        const int lane = threadIdx.x & 31, slot = p_max % 3;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, off));
        if (lane == 0) atomicMax(&gs->maxkey[slot][0], (unsigned long long)f64_key(v));
        cooperative_groups::this_grid().sync();
        const double m = f64_from_key(*reinterpret_cast<volatile unsigned long long*>(&gs->maxkey[slot][0]));
        if (blockIdx.x == 0 && threadIdx.x < 2) gs->maxkey[(p_max + 2) % 3][threadIdx.x] = 0ull;
        ++p_max;
        return m;
    }
    // median_bins hooks: the same protocol as the cluster's, through global memory (zeroed before the launch) and grid barriers
    __device__ void vhist_merge(unsigned* hist, int slot) {
        __syncthreads();  // local bins complete
        for (int j = threadIdx.x; j < kVBins; j += blockDim.x) {
            const unsigned c = hist[j];
            if (c) atomicAdd(&gs->vhist[slot][j], c);
        }
        cooperative_groups::this_grid().sync();
        for (int j = threadIdx.x; j < kVBins; j += blockDim.x) hist[j] = __ldcg(&gs->vhist[slot][j]);
        __syncthreads();
    }
    __device__ unsigned cand_index(int slot) { return atomicAdd(&gs->cursor[slot], 1u); }
    // grid-wide maximum of one 64-bit key per thread, as integers (global 64-bit atomicMax is native)
    __device__ unsigned long long max_key(unsigned long long v) {
        const int slot = p_max % 3;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const unsigned long long o = __shfl_xor_sync(0xffffffffu, v, off);
            v = o > v ? o : v;
        }
        if ((threadIdx.x & 31) == 0 && v) atomicMax(&gs->maxkey[slot][0], v);
        cooperative_groups::this_grid().sync();
        const unsigned long long m = __ldcg(&gs->maxkey[slot][0]);
        if (blockIdx.x == 0 && threadIdx.x < 2) gs->maxkey[(p_max + 2) % 3][threadIdx.x] = 0ull;
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
    __shared__ SelShared sel;
    GridReducer red{warp_part, totals, gs, 0, 0, 0};
    double *xs = scratch, *ts = scratch + n, *res = scratch + 2 * n;
    trend_prepare(red, x, t, n, x_is_mean != 0, lo, hi, xs, ts);
    TrendOut o = trend_fit_outer(red, xs, ts, n, outer != 0, false);
    if (with_prior && o.status == 0.0)  // candidate buffer: xs, as in k_trend_prior
        trend_prior_dev(red, x, t, n, lo, hi, min_disp, trigamma_c, res, reinterpret_cast<unsigned long long*>(xs), sel, hist, o);
    else
        red.sum_many(&o.n_used, 1);
    if (red.tid() == 0) *out = o;
}

// ---- size factors: median of ratios (preprocessing.py:31-102) and poscounts, over all or control genes (dds.py:628-679) --------
// SURVEY.md §8 f-2
// 1. per-gene mean over all samples of log_mean_term (ratio: -inf when the gene holds a zero, such genes are filtered out,
//    preprocessing.py:52-54).  `kept` (may be NULL): the log mean each gene enters the medians with, NaN when it is left out
//    (kept_logmean; `control` (G,) may be NULL = every gene)
__global__ void __launch_bounds__(kBlock) k_log_means(const int64_t* __restrict__ counts, int64_t ld, int N, int G, int lgT, int kind,
                                                      const uint8_t* __restrict__ control, double* __restrict__ logmeans,
                                                      double* __restrict__ kept) {
    Group grp;
    int g;
    bool valid;
    map_lanes(lgT, G, grp, g, valid);
    const int64_t* yp = counts + g + (int64_t)grp.si * ld;
    double s = 0.0;
    for (int n = grp.si; n < N; n += grp.T, yp += (int64_t)grp.T * ld) s += log_mean_term(*yp, kind);  // libdevice log: log(0) = -inf
    s = grp.sum(s);
    if (valid && grp.si == 0) {
        const double lm = s / (double)N;
        logmeans[g] = lm;
        if (kept) kept[g] = kept_logmean(lm, kind, control == nullptr || control[g] != 0);
    }
}

// 2. one block per sample: log ratios of the sample against the gene means, exact median by radix select.  `skip_zero`: zero
//    counts are left out (poscounts)
__global__ void __launch_bounds__(1024) k_size_factor_median(const int64_t* __restrict__ counts, int64_t ld, int G,
                                                             const double* __restrict__ logmeans, int skip_zero, double* scratch,
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
        bool keep;
        row[g] = log_ratio_entry(c[g], logmeans[g], keep, skip_zero != 0);
        cnt += keep;
    }
    atomicAdd(&cnt_s, cnt);
    __syncthreads();
    ClusterReducer red{warp_part, slots, totals, 0u, 1u, 0};  // one block per sample: the single-block paths of the reducer
    const double med = median_of(red, row, (size_t)G, (size_t)cnt_s, false, 0.0, hist);
    if (threadIdx.x == 0) sf_out[n] = exp(med);
}

// 3. poscounts only: sf / exp(mean(log sf)) (dds.py:674-675), one block.  A NaN size factor (a sample without a usable gene) makes
//    the mean, and so every entry, NaN, as in numpy
__global__ void __launch_bounds__(1024) k_size_factor_geomean(double* sf, int N) {
    __shared__ double part[32];
    double s = 0.0;
    for (int n = threadIdx.x; n < N; n += blockDim.x) s += log(sf[n]);
    for (int o = 16; o >= 1; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();  // every read of sf above happens before any write below
    double tot = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += part[w];
    const double gm = exp(tot / (double)N);
    for (int n = threadIdx.x; n < N; n += blockDim.x) sf[n] = sf[n] / gm;
}

// fitted = c0 + c1 / mean (dds.py:1267-1275) from the device-resident coefficients
__global__ void k_trend_eval(const double* __restrict__ means, size_t n, const TrendOut* __restrict__ c, double* fitted) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fitted[i] = c->c0 + c->c1 / means[i];
}

// final dispersions (dds.py:918-932), elementwise: select_disp (pdq_gene.cuh) per gene
__global__ void k_select_disp(const double* __restrict__ gw, const double* __restrict__ mp, const double* __restrict__ fitted,
                              const TrendOut* __restrict__ c, size_t n, double lo, double hi, double* disp, double* outlier) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool out;
    disp[i] = select_disp(gw[i], mp[i], fitted[i], c->squared_logres, lo, hi, out);
    if (outlier) outlier[i] = out ? 1.0 : 0.0;
}

// ---- variance-stabilising transform (dds.py:438-514): (N, G) int64 counts -> (N, G) float64, elementwise ----------------
// 16 bytes in and 16 bytes out per pair of genes and ~50 FP64 operations per element: bound by HBM, not by the FP64 pipe.
// With `vec` (both pitches even, both bases 16-byte aligned) a thread moves a pair of genes with one 16-byte load and one
// 16-byte store; the odd last gene of a row, and every gene without `vec`, takes the scalar path.  blockIdx.y walks the samples.
__global__ void __launch_bounds__(256) k_vst_transform(const int64_t* __restrict__ counts, int64_t ld, int N, int G,
                                                       const double* __restrict__ sf, const VstParams prm, double* __restrict__ out,
                                                       int64_t ld_out, int vec) {
    const int pairs = vec ? G >> 1 : 0;
    const int stride = gridDim.x * blockDim.x;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    for (int n = blockIdx.y; n < N; n += gridDim.y) {
        const double s = sf[n];
        const int64_t* row = counts + (int64_t)n * ld;
        double* orow = out + (int64_t)n * ld_out;
        for (int j = t; j < pairs; j += stride) {
            const longlong2 y = reinterpret_cast<const longlong2*>(row)[j];
            reinterpret_cast<double2*>(orow)[j] = make_double2(vst_value(y.x, s, prm), vst_value(y.y, s, prm));
        }
        for (int g = 2 * pairs + t; g < G; g += stride) orow[g] = vst_value(row[g], s, prm);
    }
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

// the MAP kernel, then the LFC kernel as its programmatic dependent (see k_map_irls)
template <int P, bool STAGED>
int launch_tail_pair(const LaunchCfg& c, const TailArgs<P>& a, size_t smem, int G) {
    if (int e = prep(k_map_irls<P, STAGED, 0>, smem)) return e;
    if (int e = prep(k_map_irls<P, STAGED, 1>, smem)) return e;
    k_map_irls<P, STAGED, 0><<<persistent_grid(k_map_irls<P, STAGED, 0>, smem, c.sm_count, G, c.lgT), kBlock, smem, c.stream>>>(a);
    cudaLaunchConfig_t lc = {};
    lc.gridDim = dim3((unsigned)persistent_grid(k_map_irls<P, STAGED, 1>, smem, c.sm_count, G, c.lgT));
    lc.blockDim = dim3(kBlock);
    lc.dynamicSmemBytes = smem;
    lc.stream = c.stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at;
    lc.numAttrs = 1;
    if (cudaLaunchKernelEx(&lc, k_map_irls<P, STAGED, 1>, a) != cudaSuccess) return PDQ_ERR_CUDA;
    return 0;
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

// Several (offset, rows, width) segments of one buffer in one launch, as a gather: out[off + j * width + k] = in[off + src[j] *
// width + k], or row j from row j when the segment is not permuted (a record that rides along with the per-gene vectors).  Stores
// are contiguous, so `out` may be page-locked host memory: the rows then cross the bus as full write bursts, with no copy node
// behind the launch.  The segments' element counts are laid end to end over the grid; `start` holds their running sums.
struct ScatterSegs {
    int n;
    int64_t off[kMaxScatterSegs], start[kMaxScatterSegs + 1];
    int rows[kMaxScatterSegs], width[kMaxScatterSegs], permuted[kMaxScatterSegs];
};

__global__ void k_scatter_segments(const double* __restrict__ in, double* __restrict__ out, const int* __restrict__ src,
                                   const __grid_constant__ ScatterSegs s) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= s.start[s.n]) return;
    int i = 0;
    while (t >= s.start[i + 1]) ++i;
    const int64_t r = t - s.start[i];
    const int w = s.width[i];
    const int j = (int)(r / w), k = (int)(r - (int64_t)j * w);
    out[s.off[i] + r] = in[s.off[i] + (int64_t)(s.permuted[i] ? src[j] : j) * w + k];
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

int PDQ_TUFN(launch_map_irls)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, const TailHost& t,
                              const IrlsHost& h, const WaldHost& w) {
    PDQ_DISPATCH_P(d.p, {
        TailArgs<P> a;
        const DesignView dv{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0};
        int* words = c.tickets + kTailWords;
        // the fallback kernels read the count of flagged genes at ticket[1]: the words the last blocks of k_map_irls fill
        a.al = AlphaArgs<P>{dv, AlphaParams{log(t.min_disp), log(t.max_disp), t.prior_var, 1, 1}, counts, ld, G, c.lgT, t.mu, t.ld_mu,
                            t.fitted, t.map, t.map_conv, t.status_map, t.prior_var_dev, words + kTailGridOut - 1,
                            (c.debug & PDQ_DEBUG_FORCE_ALPHA_GRID) ? 1 : 0, t.hint_in, nullptr, 0};
        a.ir.dv = dv;
        a.ir.pinv = pinv_of<P>(d);
        a.ir.prm = IrlsParams{h.min_mu, h.beta_tol, h.min_beta, h.max_beta, h.maxiter, d.full_rank, d.few_rows,
                              (c.debug & PDQ_DEBUG_FAIL_IRLS_OPTIMIZER) ? 1 : 0};
        a.ir.counts = counts; a.ir.ld = ld; a.ir.G = G; a.ir.lgT = c.lgT; a.ir.disp = t.disp;
        a.ir.beta = t.beta; a.ir.mu = t.mu_out; a.ir.hat = t.hat; a.ir.conv = t.conv; a.ir.ld_out = t.ld_out;
        a.ir.status = t.status_irls; a.ir.n_fallback = nullptr; a.ir.ticket = words + kTailOptOut - 1;
        a.ir.force = (c.debug & PDQ_DEBUG_FORCE_IRLS_OPTIMIZER) ? 1 : 0;
        a.ir.with_wald = 1;
        for (int i = 0; i < P * P; ++i) a.ir.wald.ridge[i] = w.ridge[i];
        for (int i = 0; i < P; ++i) a.ir.wald.contrast[i] = w.contrast[i];
        a.ir.wald.lfc_null = w.lfc_null;
        a.ir.wald.alt = w.alt;
        a.ir.wald_p = w.pv; a.ir.wald_stat = w.stat; a.ir.wald_se = w.se;
        a.gw = t.gw; a.trend = reinterpret_cast<const TrendOut*>(t.trend16);
        a.min_disp = t.min_disp; a.max_disp = t.max_disp; a.disp = t.disp; a.outlier = t.outlier;
        a.words = words; a.tile_done = t.tile_done; a.err = t.err; a.timeout_ns = 20000000000ULL;
        const size_t smem_tail = d.smem_bytes + kMathTabBytes + (size_t)(1 + 2 * kWarps * (32 >> c.lgT)) * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (int e = prep(k_irls_deferred<P>, smem_tail)) return e;
        if (int e = prep(k_irls_optimizer<P>, d.smem_bytes)) return e;
        if (int e = d.staged ? launch_tail_pair<P, true>(c, a, smem_tail, G) : launch_tail_pair<P, false>(c, a, smem_tail, G)) return e;
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

int PDQ_TUFN(launch_wald_contrasts)(const LaunchCfg& c, const DesignDev& d, const double* disp, const double* lfc, int G,
                                    const double* ridge, int K, const double* tab, double* pv, double* stat, double* se, int64_t ld_out) {
    PDQ_DISPATCH_P(d.p, {
        WaldContrastsArgs<P> a;
        a.dv = DesignView{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0};
        for (int i = 0; i < P * P; ++i) a.ridge[i] = ridge[i];
        a.tab = tab;
        a.disp = disp; a.lfc = lfc; a.G = G; a.lgT = c.lgT; a.K = K;
        a.pv = pv; a.stat = stat; a.se = se; a.ld_out = ld_out;
        if (int e = prep(k_wald_contrasts<P>, d.smem_bytes)) return e;
        k_wald_contrasts<P><<<grid_for(G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a);
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

int PDQ_TUFN(launch_mom_alpha)(const LaunchCfg& c, const DesignDev& d, const int64_t* counts, int64_t ld, int G, double min_disp,
                               double max_disp, double min_mu, double* mom, double* normed_mean, double* mu_hat, int64_t ld_mu,
                               double* alpha, double* conv, int* status, double* hint_out) {
    PDQ_DISPATCH_P(d.p, {
        MomAlphaArgs<P> a;
        int* words = c.tickets + kFoldWords;
        // genewise search (cr_reg on, no prior); k_alpha_grid behind the launch reads the flagged-gene count at ticket[1] =
        // the word the kernel's last block fills
        a.al = AlphaArgs<P>{{d.pack, d.N, d.staged ? (int)(d.smem_bytes - 16) : 0}, AlphaParams{log(min_disp), log(max_disp), 1.0, 1, 0},
                            counts, ld, G, c.lgT, mu_hat, ld_mu, mom, alpha, conv, status, nullptr, words + kFoldGridOut - 1,
                            (c.debug & PDQ_DEBUG_FORCE_ALPHA_GRID) ? 1 : 0, nullptr, hint_out, alpha_descending()};
        a.pinv = pinv_of<P>(d);
        a.s_mean_inv = d.s_mean_inv; a.min_disp = min_disp; a.max_disp = max_disp; a.min_mu = min_mu;
        a.mom = mom; a.means = normed_mean; a.mu_hat = mu_hat; a.words = words;
        const size_t smem_alpha = d.smem_bytes + kMathTabBytes + (size_t)kWarps * (32 >> c.lgT) * 2 * kPsiK * sizeof(double);
        if (int e = prep(k_alpha_grid<P>, d.smem_bytes)) return e;
        if (d.staged) {
            if (int e = prep(k_mom_alpha<P, true>, smem_alpha)) return e;
            k_mom_alpha<P, true><<<persistent_grid(k_mom_alpha<P, true>, smem_alpha, c.sm_count, G, c.lgT), kBlock, smem_alpha, c.stream>>>(a);
        } else {
            if (int e = prep(k_mom_alpha<P, false>, smem_alpha)) return e;
            k_mom_alpha<P, false><<<persistent_grid(k_mom_alpha<P, false>, smem_alpha, c.sm_count, G, c.lgT), kBlock, smem_alpha, c.stream>>>(a);
        }
        k_alpha_grid<P><<<fallback_grid(c.sm_count, G, c.lgT), kBlock, d.smem_bytes, c.stream>>>(a.al);
    });
    if (int e = check_launch()) return e;
    return 2;
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
    if (const char* e = getenv("PDQ_TREND_PRIOR")) {  // tuning hook: PDQ_TREND_PRIOR=0 skips the prior (times the fit alone)
        if (atoi(e) == 0) with_prior = 0;
    }
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

int launch_scatter_segments(cudaStream_t stream, const double* in, double* out, const int* src, int nseg, const int64_t* seg) {
    if (nseg < 1 || nseg > kMaxScatterSegs) return PDQ_ERR_INVALID;
    ScatterSegs s{};
    s.n = nseg;
    for (int i = 0; i < nseg; ++i) {
        s.off[i] = seg[4 * i];
        s.rows[i] = (int)seg[4 * i + 1];
        s.width[i] = (int)seg[4 * i + 2];
        s.permuted[i] = seg[4 * i + 3] != 0;
        s.start[i + 1] = s.start[i] + (int64_t)s.rows[i] * s.width[i];
    }
    if (s.start[nseg] <= 0) return 0;
    k_scatter_segments<<<(unsigned)((s.start[nseg] + 255) / 256), 256, 0, stream>>>(in, out, src, s);
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
    return launch_size_factors_ex(c, counts, ld, N, G, kSfRatio, nullptr, logmeans, nullptr, scratch, sf_out);
}

// `kept` NULL: median of ratios over every gene, whose medians read the log means directly (-inf = left out)
int launch_size_factors_ex(const LaunchCfg& c, const int64_t* counts, int64_t ld, int N, int G, int kind, const uint8_t* control,
                           double* logmeans, double* kept, double* scratch, double* sf_out) {
    k_log_means<<<grid_for(G, c.lgT), kBlock, 0, c.stream>>>(counts, ld, N, G, c.lgT, kind, control, logmeans, kept);
    k_size_factor_median<<<N, 1024, 0, c.stream>>>(counts, ld, G, kept ? kept : logmeans, kind == kSfPoscounts, scratch, sf_out);
    if (kind == kSfPoscounts) k_size_factor_geomean<<<1, 1024, 0, c.stream>>>(sf_out, N);
    if (int e = check_launch()) return e;
    return kind == kSfPoscounts ? 3 : 2;
}

// held-out samples (preprocessing.py:59-102): the medians against the caller's log means, non-finite entries = genes left out
int launch_size_factors_from_logmeans(const LaunchCfg& c, const int64_t* counts, int64_t ld, int N, int G, const double* logmeans,
                                      double* scratch, double* sf_out) {
    k_size_factor_median<<<N, 1024, 0, c.stream>>>(counts, ld, G, logmeans, 0, scratch, sf_out);
    if (int e = check_launch()) return e;
    return 1;
}

int launch_vst_transform(const LaunchCfg& c, const int64_t* counts, int64_t ld, int N, int G, const double* sf, int kind, double c0,
                         double c1, double* out, int64_t ld_out) {
    const bool vec = ld % 2 == 0 && ld_out % 2 == 0 && (reinterpret_cast<uintptr_t>(counts) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(out) & 15) == 0;
    const int units = vec ? (G + 1) / 2 : G;
    const unsigned bx = (unsigned)((units + 255) / 256);
    const unsigned by = (unsigned)(N < 65535 ? N : 65535);
    k_vst_transform<<<dim3(bx, by), 256, 0, c.stream>>>(counts, ld, N, G, sf, VstParams{kind, c0, c1}, out, ld_out, vec ? 1 : 0);
    if (int e = check_launch()) return e;
    return 1;
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
