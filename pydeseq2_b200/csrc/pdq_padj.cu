// pdq_padj.cu -- DeseqStats' multiple-testing step (ds.py:486-542) for K rows of p-values at once: the rejection counts of the
// independent filter at every base-mean cutoff, and the Benjamini-Hochberg adjusted p-values of each row over its own cutoff.
//
// Each row's p-values are sorted once (cub::DeviceRadixSort on their bit patterns: non-negative doubles order as their bits; a
// gene left out of the row's set gets a key above every p in [0, 1], so the set is a prefix of the sorted row).  The rest runs
// over chunks of kChunk sorted positions:
//   rejections  k_padj_count (members of each cutoff's set per chunk) -> k_padj_scan (chunk offsets and set sizes per (row,
//               cutoff)) -> k_padj_reject (rank of every member in every set, the largest rank whose BH value is below alpha);
//               every chunk is read twice whatever the number of cutoffs: the cutoffs are bits of a per-gene mask.
//   bh          k_padj_bh_min (smallest BH value per chunk) -> k_padj_bh_suffix (minimum over the chunks to the right) ->
//               k_padj_bh_out (suffix minimum inside the chunk, clip, scatter to gene order; NaN outside the set).
// The arithmetic is pdq_padj.cuh, shared with the host emulator of the test-suite.
#include <cub/cub.cuh>

#include "pdq_internal.h"
#include "pdq_launch.cuh"
#include "pdq_padj.cuh"

namespace pdq {

namespace {

constexpr int kTPB = 256, kSlots = 4, kChunk = kTPB * kSlots, kWarps = kTPB / 32;
constexpr uint64_t kKeyOut = 0x3FF0000000000001ull;  // just above the bits of 1.0: genes outside a row's set sort after it
constexpr int kKeyBits = 62;                          // every p in [0, 1] and kKeyOut fit in bits 0..61
constexpr unsigned kFull = 0xffffffffu;

struct MinOp {
    __device__ double operator()(double a, double b) const { return b < a ? b : a; }
};

__device__ __forceinline__ double key_p(uint64_t k) { return __longlong_as_double((long long)k); }

// keys (K, G) hold the raw p-values on entry; afterwards the p-value bits of the row's set and kKeyOut elsewhere.  The set: p not
// NaN and, when `row_cutoff` is given, padj_in_set.  n_in[k] counts it; `bad` counts p-values outside [0, 1].
__global__ void k_padj_keys(uint64_t* keys, int* vals, int G, const double* bm, const double* row_cutoff, int* n_in, int* bad) {
    const int k = blockIdx.y;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    bool in = false;
    if (g < G) {
        const size_t o = (size_t)k * G + g;
        const uint64_t key = keys[o];
        const double p = key_p(key);
        if (!isnan(p) && !(p >= 0.0 && p <= 1.0)) atomicAdd(bad, 1);
        in = row_cutoff ? padj_in_set(p, bm[g], row_cutoff[k]) : !isnan(p);
        keys[o] = in ? key : kKeyOut;
        vals[o] = g;
    }
    const unsigned b = __ballot_sync(kFull, in);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(n_in + k, __popc(b));
}

__global__ void k_padj_cutoffs(const double* sorted, int G, const double* theta, int n_theta, double* cutoffs) {
    const int i = threadIdx.x;
    if (i < n_theta) cutoffs[i] = quantile_linear(sorted, G, theta[i], isnan(sorted[0]) || isnan(sorted[G - 1]));
}

__global__ void k_padj_masks(const double* bm, int G, const double* cutoffs, int n_theta, uint64_t* masks) {
    __shared__ double s_cut[kPadjMaxTheta];
    if (threadIdx.x < n_theta) s_cut[threadIdx.x] = cutoffs[threadIdx.x];
    __syncthreads();
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < G) masks[g] = padj_member_mask(bm[g], s_cut, n_theta);
}

// counts[(k, i, chunk)] = members of cutoff i's set among the chunk's sorted positions of row k
__global__ void __launch_bounds__(kTPB) k_padj_count(const int* vals, const uint64_t* masks, const int* n_in, int G, int n_theta,
                                                     int n_chunks, int* counts) {
    __shared__ int s_cnt[kPadjMaxTheta];
    const int k = blockIdx.y, c = blockIdx.x, n = n_in[k], tid = threadIdx.x;
    if (tid < n_theta) s_cnt[tid] = 0;
    __syncthreads();
    if (c * kChunk < n) {
        uint64_t m[kSlots];
#pragma unroll
        for (int j = 0; j < kSlots; ++j) {
            const int pos = c * kChunk + j * kTPB + tid;
            m[j] = pos < n ? masks[vals[(size_t)k * G + pos]] : 0;
        }
        for (int i = 0; i < n_theta; ++i) {
            int t = 0;
#pragma unroll
            for (int j = 0; j < kSlots; ++j) t += __popc(__ballot_sync(kFull, (m[j] >> i) & 1));
            if ((tid & 31) == 0 && t) atomicAdd(&s_cnt[i], t);
        }
        __syncthreads();
    }
    if (tid < n_theta) counts[((size_t)k * n_theta + tid) * n_chunks + c] = s_cnt[tid];
}

// one block per (row, cutoff): the chunk counts become exclusive offsets, the total is the set's size
__global__ void __launch_bounds__(kTPB) k_padj_scan(int* counts, int n_chunks, int* totals) {
    using Scan = cub::BlockScan<int, kTPB>;
    __shared__ typename Scan::TempStorage tmp;
    int* row = counts + (size_t)blockIdx.x * n_chunks;
    int run = 0;
    for (int base = 0; base < n_chunks; base += kTPB) {
        const int i = base + threadIdx.x;
        const int v = i < n_chunks ? row[i] : 0;
        int ex, agg;
        Scan(tmp).ExclusiveSum(v, ex, agg);
        if (i < n_chunks) row[i] = run + ex;
        run += agg;
        __syncthreads();
    }
    if (threadIdx.x == 0) totals[blockIdx.x] = run;
}

// num_rej[k, i] = max over the chunk's members of cutoff i's set of the rank r whose BH value is below alpha (atomicMax)
__global__ void __launch_bounds__(kTPB) k_padj_reject(const uint64_t* keys, const int* vals, const uint64_t* masks, const int* n_in,
                                                      const int* offsets, const int* totals, int G, int n_theta, int n_chunks,
                                                      double alpha, int* num_rej) {
    __shared__ int s_off[kPadjMaxTheta][kSlots * kWarps];
    __shared__ int s_best[kPadjMaxTheta];
    const int k = blockIdx.y, c = blockIdx.x, n = n_in[k], tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (c * kChunk >= n) return;
    uint64_t m[kSlots];
    double p[kSlots];
#pragma unroll
    for (int j = 0; j < kSlots; ++j) {
        const int pos = c * kChunk + j * kTPB + tid;
        const size_t o = (size_t)k * G + pos;
        m[j] = pos < n ? masks[vals[o]] : 0;
        p[j] = pos < n ? key_p(keys[o]) : 1.0;
    }
    for (int i = 0; i < n_theta; ++i) {
#pragma unroll
        for (int j = 0; j < kSlots; ++j) {
            const unsigned b = __ballot_sync(kFull, (m[j] >> i) & 1);
            if (lane == 0) s_off[i][j * kWarps + w] = __popc(b);
        }
    }
    if (tid < n_theta) s_best[tid] = 0;
    __syncthreads();
    if (tid < n_theta) {  // members before each (slot, warp) group: the chunk's offset plus the groups before it
        int run = offsets[((size_t)k * n_theta + tid) * n_chunks + c];
        for (int q = 0; q < kSlots * kWarps; ++q) {
            const int v = s_off[tid][q];
            s_off[tid][q] = run;
            run += v;
        }
    }
    __syncthreads();
    const unsigned le = lane == 31 ? kFull : ((2u << lane) - 1u);
    for (int i = 0; i < n_theta; ++i) {
        const int M = totals[k * n_theta + i];
        int best = 0;
#pragma unroll
        for (int j = 0; j < kSlots; ++j) {
            const bool in = (m[j] >> i) & 1;
            const unsigned b = __ballot_sync(kFull, in);
            const int base = s_off[i][j * kWarps + w];
            const bool ok = in && bh_below(p[j], base + __popc(b & le), M, alpha);
            const unsigned ob = __ballot_sync(kFull, ok);
            if (ob) {  // later slots hold later (larger) ranks
                const int h = 31 - __clz(ob);
                best = base + __popc(b & (h == 31 ? kFull : ((2u << h) - 1u)));
            }
        }
        if (lane == 0 && best) atomicMax(&s_best[i], best);
    }
    __syncthreads();
    if (tid < n_theta && s_best[tid]) atomicMax(&num_rej[k * n_theta + tid], s_best[tid]);
}

__device__ __forceinline__ double bh_at(const uint64_t* row, int pos, int n) {
    return pos < n ? bh_value(key_p(row[pos]), (int64_t)pos + 1, n) : INFINITY;
}

__global__ void __launch_bounds__(kTPB) k_padj_bh_min(const uint64_t* keys, const int* n_in, int G, int n_chunks, double* chunk_min) {
    using Reduce = cub::BlockReduce<double, kTPB>;
    __shared__ typename Reduce::TempStorage tmp;
    const int k = blockIdx.y, c = blockIdx.x, n = n_in[k];
    const uint64_t* row = keys + (size_t)k * G;
    double v = INFINITY;
#pragma unroll
    for (int j = 0; j < kSlots; ++j) v = MinOp()(v, bh_at(row, c * kChunk + j * kTPB + threadIdx.x, n));
    v = Reduce(tmp).Reduce(v, MinOp());
    if (threadIdx.x == 0) chunk_min[(size_t)k * n_chunks + c] = v;
}

// suffix[k, c] = minimum of chunk_min[k, c'] over c' > c
__global__ void __launch_bounds__(kTPB) k_padj_bh_suffix(const double* chunk_min, int n_chunks, double* suffix) {
    using Scan = cub::BlockScan<double, kTPB>;
    __shared__ typename Scan::TempStorage tmp;
    const size_t o = (size_t)blockIdx.x * n_chunks;
    double run = INFINITY;
    for (int base = 0; base < n_chunks; base += kTPB) {
        const int ri = base + threadIdx.x, c = n_chunks - 1 - ri;
        const double v = ri < n_chunks ? chunk_min[o + c] : INFINITY;
        double ex, agg;
        Scan(tmp).ExclusiveScan(v, ex, INFINITY, MinOp(), agg);
        if (ri < n_chunks) suffix[o + c] = MinOp()(run, ex);
        run = MinOp()(run, agg);
        __syncthreads();
    }
}

// the adjusted p-values of the chunk in gene order: thread t holds sorted positions chunk_end - 1 - (4 t + j), so an inclusive
// block min-scan is the suffix minimum inside the chunk
__global__ void __launch_bounds__(kTPB) k_padj_bh_out(const uint64_t* keys, const int* vals, const int* n_in, int G, int n_chunks,
                                                      const double* suffix, double* padj, int64_t ld_out) {
    using Scan = cub::BlockScan<double, kTPB>;
    __shared__ typename Scan::TempStorage tmp;
    const int k = blockIdx.y, c = blockIdx.x, n = n_in[k];
    const uint64_t* row = keys + (size_t)k * G;
    double v[kSlots];
    int pos[kSlots];
#pragma unroll
    for (int j = 0; j < kSlots; ++j) {
        pos[j] = c * kChunk + kChunk - 1 - (threadIdx.x * kSlots + j);
        v[j] = bh_at(row, pos[j], n);
    }
    Scan(tmp).InclusiveScan(v, v, MinOp());
    const double right = suffix[(size_t)k * n_chunks + c];
#pragma unroll
    for (int j = 0; j < kSlots; ++j) {
        if (pos[j] >= G) continue;
        const double a = MinOp()(v[j], right);
        padj[(size_t)k * ld_out + vals[(size_t)k * G + pos[j]]] = pos[j] < n ? (n > 1 ? clip01(a) : a) : NAN;
    }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// the sort of one row (keys, gene indices) and of the base means share the temporary storage
size_t sort_temp_bytes(int G) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (const int*)nullptr, (int*)nullptr, G, 0,
                                    kKeyBits);
    cub::DeviceRadixSort::SortKeys(nullptr, b, (const double*)nullptr, (double*)nullptr, G);
    return a > b ? a : b;
}

int sort_rows(const PadjScratch& s, int G, int K, cudaStream_t st) {
    for (int k = 0; k < K; ++k) {
        size_t tb = s.temp_bytes;
        const size_t o = (size_t)k * G;
        if (cub::DeviceRadixSort::SortPairs(s.temp, tb, s.keys_in + o, s.keys + o, s.vals_in + o, s.vals + o, G, 0, kKeyBits, st) !=
            cudaSuccess)
            return PDQ_ERR_CUDA;
    }
    return K;
}

int keys(const PadjScratch& s, int G, int K, const double* row_cutoff, cudaStream_t st) {
    if (cudaMemsetAsync(s.counters, 0, (size_t)(K + 1) * sizeof(int), st) != cudaSuccess) return PDQ_ERR_CUDA;
    k_padj_keys<<<dim3((G + kTPB - 1) / kTPB, K), kTPB, 0, st>>>(s.keys_in, s.vals_in, G, s.bm, row_cutoff, s.counters, s.counters + K);
    if (int e = check_launch()) return e;
    const int r = sort_rows(s, G, K, st);
    return r < 0 ? r : r + 1;
}

}  // namespace

static int padj_chunks(int G) { return (G + kChunk - 1) / kChunk; }

size_t padj_layout(int G, int K, int n_theta, void* base, PadjScratch* s) {
    const size_t KG = (size_t)K * G, nc = (size_t)padj_chunks(G);
    size_t off = 0;
    char* b = (char*)base;
    auto take = [&](size_t bytes) {
        void* p = b ? b + off : nullptr;
        off += align256(bytes);
        return p;
    };
    s->keys_in = (uint64_t*)take(KG * 8);
    s->keys = (uint64_t*)take(KG * 8);
    s->vals_in = (int*)take(KG * 4);
    s->vals = (int*)take(KG * 4);
    s->bm = (double*)take((size_t)G * 8);
    s->bm_sorted = (double*)take((size_t)G * 8);
    s->masks = (uint64_t*)take((size_t)G * 8);
    s->counters = (int*)take((size_t)(K + 1) * 4);
    s->theta = (double*)take(kPadjMaxTheta * 8);
    s->cutoffs = (double*)take(kPadjMaxTheta * 8);
    s->row_cutoff = (double*)take((size_t)K * 8);
    s->num_rej = (int*)take((size_t)K * n_theta * 4);
    s->totals = (int*)take((size_t)K * n_theta * 4);
    s->chunk_counts = (int*)take((size_t)K * n_theta * nc * 4);
    s->chunk_min = (double*)take((size_t)K * nc * 8);
    s->suffix = (double*)take((size_t)K * nc * 8);
    s->temp_bytes = sort_temp_bytes(G);
    s->temp = take(s->temp_bytes);
    return off;
}

int launch_padj_rejections(cudaStream_t st, const PadjScratch& s, int G, int K, int n_theta, double alpha) {
    const int nc = padj_chunks(G), gb = (G + kTPB - 1) / kTPB;
    size_t tb = s.temp_bytes;
    if (cub::DeviceRadixSort::SortKeys(s.temp, tb, s.bm, s.bm_sorted, G, 0, 64, st) != cudaSuccess) return PDQ_ERR_CUDA;
    k_padj_cutoffs<<<1, kPadjMaxTheta, 0, st>>>(s.bm_sorted, G, s.theta, n_theta, s.cutoffs);
    k_padj_masks<<<gb, kTPB, 0, st>>>(s.bm, G, s.cutoffs, n_theta, s.masks);
    if (int e = check_launch()) return e;
    const int nk = keys(s, G, K, nullptr, st);
    if (nk < 0) return nk;
    if (cudaMemsetAsync(s.num_rej, 0, (size_t)K * n_theta * 4, st) != cudaSuccess) return PDQ_ERR_CUDA;
    k_padj_count<<<dim3(nc, K), kTPB, 0, st>>>(s.vals, s.masks, s.counters, G, n_theta, nc, s.chunk_counts);
    k_padj_scan<<<K * n_theta, kTPB, 0, st>>>(s.chunk_counts, nc, s.totals);
    k_padj_reject<<<dim3(nc, K), kTPB, 0, st>>>(s.keys, s.vals, s.masks, s.counters, s.chunk_counts, s.totals, G, n_theta, nc, alpha,
                                                s.num_rej);
    if (int e = check_launch()) return e;
    return 1 + 2 + nk + 3;
}

int launch_padj_bh(cudaStream_t st, const PadjScratch& s, int G, int K, double* padj, int64_t ld_out) {
    const int nc = padj_chunks(G);
    const int nk = keys(s, G, K, s.row_cutoff, st);
    if (nk < 0) return nk;
    k_padj_bh_min<<<dim3(nc, K), kTPB, 0, st>>>(s.keys, s.counters, G, nc, s.chunk_min);
    k_padj_bh_suffix<<<K, kTPB, 0, st>>>(s.chunk_min, nc, s.suffix);
    k_padj_bh_out<<<dim3(nc, K), kTPB, 0, st>>>(s.keys, s.vals, s.counters, G, nc, s.suffix, padj, ld_out);
    if (int e = check_launch()) return e;
    return nk + 3;
}

}  // namespace pdq
