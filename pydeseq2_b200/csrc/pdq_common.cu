// pdq_common.cu -- the kernels that do not depend on the design width, and their launchers: the dispersion trend + prior fit, the
// trend values and final dispersions, size factors, the variance-stabilising transform, the FP64 peak probe, and the resident
// pass's glue (gathers, column sums, scatters, content checksums).  Compiled once; the per-gene kernels are in pdq_kernels.cu
// (p <= 16) and pdq_wide.cu (17..128 columns).
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "pdq_gene.cuh"
#include "pdq_trend.cuh"
#include "pdq_vst.cuh"
#include "pdq_internal.h"
#include "pdq_launch.cuh"

namespace pdq {
namespace {

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

}  // namespace

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

size_t cooks_ws_bytes(const DesignDev& d, int G) {
    if (cooks_in_smem(d)) return 0;
    const size_t chunk = (size_t)cooks_chunk(d), genes = ((size_t)G + kWarps - 1) / kWarps * kWarps;
    return (genes < chunk ? genes : chunk) * cooks_gene_bytes(d);
}

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

}  // namespace pdq
