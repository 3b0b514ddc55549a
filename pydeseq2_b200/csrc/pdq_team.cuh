// pdq_team.cuh -- the cooperative building blocks of one gene's team of W warps (one block), shared by every kernel of
// pdq_wide.cu (designs of PDQ_MAX_P + 1 .. PDQ_MAX_P_LARGE columns) and by the GPU probe's team unit (tests/gpu_probe/team_probe.cu),
// which checks them directly against extended-precision references at every team width.
//   * Team<W>: the block's thread index, barrier, sum / max over the team (bit-identical in every thread) and vote;
//   * the per-gene workspace in dynamic shared memory (wide_ws_doubles, Ws, carve) and the design pack accessors;
//   * rank_chunk / vec_chunk: X^T W X and X^T W z from one staged chunk of 32 W samples;
//   * the packed Cholesky family (chol_w, chol_solve_w, chol_inverse_w, factor_ridged), matvec_w, symdot_w, quad_w, apply_pinv;
//   * wald_inverse_w / wald_se_w (the Wald test's standard error) and wdot / wmaxabs (the shrinkage optimiser's reductions).
// Every entry, row or column is owned by one thread (k = tid, tid + 32 W, ...); the team barriers between the steps are what make
// a value written by one thread visible to the others.
#pragma once

#include <cuda_runtime.h>

#include "pdq_gene.cuh"

namespace pdq {
namespace {

constexpr int kVecs = 8;  // vectors of p doubles in the workspace

// the cooperative primitives of one gene's team of W warps (the whole block)
template <int W>
struct Team {
    static constexpr int NT = 32 * W;  // threads, and samples per chunk
    static __device__ __forceinline__ int tid() { return W == 1 ? (int)(threadIdx.x & 31) : (int)threadIdx.x; }
    static __device__ __forceinline__ void sync() {
        if constexpr (W == 1) __syncwarp();
        else __syncthreads();
    }
    // total over the team, bit-identical in every thread
    static __device__ __forceinline__ double sum(double v) {
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if constexpr (W > 1) {
            __shared__ double slot[W];
            if ((threadIdx.x & 31) == 0) slot[threadIdx.x >> 5] = v;
            __syncthreads();
            v = slot[0];
            for (int w = 1; w < W; ++w) v += slot[w];
            __syncthreads();  // the slots are free again
        }
        return v;
    }
    // maximum over the team, bit-identical in every thread
    static __device__ __forceinline__ double max(double v) {
        for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
        if constexpr (W > 1) {
            __shared__ double slot[W];
            if ((threadIdx.x & 31) == 0) slot[threadIdx.x >> 5] = v;
            __syncthreads();
            v = slot[0];
            for (int w = 1; w < W; ++w) v = fmax(v, slot[w]);
            __syncthreads();
        }
        return v;
    }
    static __device__ __forceinline__ bool any(bool b) {
        if constexpr (W == 1) return __any_sync(0xffffffffu, b) != 0;
        else return __syncthreads_or(b) != 0;
    }
};

__host__ __device__ constexpr int tri_count(int p) { return (p * (p + 1) / 2 + 1) & ~1; }
// workspace of one gene: three packed p x p matrices, kVecs vectors of p, two chunk buffers of 32 W
__host__ __device__ constexpr size_t wide_ws_doubles(int p, int W = 1) { return 3 * (size_t)tri_count(p) + (size_t)kVecs * p + 64 * W; }

struct Ws {
    double *A, *L, *Li;  // packed lower triangles
    double* v[kVecs];
    double *cw, *cz;     // per-chunk staging, one slot per thread
    int p, np;
};

template <int W = 1>
__device__ __forceinline__ Ws carve(double* s, int p) {
    Ws w;
    w.p = p;
    w.np = p * (p + 1) / 2;
    const int t = tri_count(p);
    w.A = s;
    w.L = s + t;
    w.Li = s + 2 * t;
    for (int k = 0; k < kVecs; ++k) w.v[k] = s + 3 * t + k * p;
    w.cw = s + 3 * t + kVecs * p;
    w.cz = w.cw + Team<W>::NT;
    return w;
}

__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ DesignS design_of(const double* pack, int N, int p) {
    DesignS d;
    d.X = pack;
    d.sf = pack + p;
    d.lsf = pack + p + 1;
    d.N = N;
    d.RS = design_row_stride(p);
    return d;
}
__device__ __forceinline__ const double* row_of(const DesignS& d, int n) { return d.X + (size_t)n * d.RS; }

template <int W = 1>
__device__ __forceinline__ void wfill(double* a, int n, double v) {
    using T = Team<W>;
    for (int k = T::tid(); k < n; k += T::NT) a[k] = v;
}
template <int W = 1>
__device__ __forceinline__ void wcopy(double* dst, const double* src, int n) {
    using T = Team<W>;
    for (int k = T::tid(); k < n; k += T::NT) dst[k] = src[k];
}

// S += sum_{s < cnt} w[s] x_{n0+s} x_{n0+s}^T over the packed lower triangle, entries k = lane, lane + 32, ...
template <int W = 1>
__device__ void rank_chunk(const DesignS& d, int p, int n0, int cnt, const double* w, double* S) {
    using T = Team<W>;
    const int np = p * (p + 1) / 2;
    int i = 0, j = T::tid();
    while (j > i) {
        j -= i + 1;
        ++i;
    }
    for (int k = T::tid(); k < np; k += T::NT) {
        double acc = S[k];
        for (int s = 0; s < cnt; ++s) {
            const double* x = row_of(d, n0 + s);
            acc = fma(w[s] * x[i], x[j], acc);
        }
        S[k] = acc;
        j += T::NT;
        while (j > i) {
            j -= i + 1;
            ++i;
        }
    }
}

// v += sum_{s < cnt} z[s] x_{n0+s}, components split over the lanes
template <int W = 1>
__device__ void vec_chunk(const DesignS& d, int p, int n0, int cnt, const double* z, double* v) {
    using T = Team<W>;
    for (int j = T::tid(); j < p; j += T::NT) {
        double acc = v[j];
        for (int s = 0; s < cnt; ++s) acc = fma(z[s], row_of(d, n0 + s)[j], acc);
        v[j] = acc;
    }
}

__device__ __forceinline__ double xdot(const double* x, const double* b, int p) {
    double e = 0.0;
    for (int j = 0; j < p; ++j) e = fma(x[j], b[j], e);
    return e;
}

// in-place L L^T = L (packed); a non-positive pivot gives NaN through sqrt, as chol<P>
template <int W = 1>
__device__ void chol_w(double* L, int p) {
    using T = Team<W>;
    const int lane = T::tid();
    for (int j = 0; j < p; ++j) {
        T::sync();
        const double dj = sqrt(L[tri(j, j)]);
        const double inv = 1.0 / dj;
        T::sync();
        for (int i = j + 1 + lane; i < p; i += T::NT) L[tri(i, j)] *= inv;
        if (lane == 0) L[tri(j, j)] = dj;
        T::sync();
        for (int i = j + 1 + lane; i < p; i += T::NT) {
            const double lij = L[tri(i, j)];
            for (int k = j + 1; k <= i; ++k) L[tri(i, k)] = fma(-lij, L[tri(k, j)], L[tri(i, k)]);
        }
    }
    T::sync();
}

// solve (L L^T) x = v in place
template <int W = 1>
__device__ void chol_solve_w(const double* L, double* v, int p) {
    using T = Team<W>;
    const int lane = T::tid();
    for (int i = 0; i < p; ++i) {
        T::sync();
        const double xi = v[i] / L[tri(i, i)];
        T::sync();
        if (lane == 0) v[i] = xi;
        for (int r = i + 1 + lane; r < p; r += T::NT) v[r] = fma(-L[tri(r, i)], xi, v[r]);
    }
    for (int i = p - 1; i >= 0; --i) {
        T::sync();
        const double xi = v[i] / L[tri(i, i)];
        T::sync();
        if (lane == 0) v[i] = xi;
        for (int r = lane; r < i; r += T::NT) v[r] = fma(-L[tri(i, r)], xi, v[r]);
    }
    T::sync();
}

// H = (L L^T)^-1; Li = L^-1 (scratch).  H may be L itself: the second phase reads Li only
template <int W = 1>
__device__ void chol_inverse_w(const double* L, double* Li, double* H, int p) {
    using T = Team<W>;
    T::sync();
    for (int j = T::tid(); j < p; j += T::NT) {
        Li[tri(j, j)] = 1.0 / L[tri(j, j)];
        for (int i = j + 1; i < p; ++i) {
            double s = 0.0;
            for (int k = j; k < i; ++k) s = fma(-L[tri(i, k)], Li[tri(k, j)], s);
            Li[tri(i, j)] = s / L[tri(i, i)];
        }
    }
    T::sync();
    for (int i = T::tid(); i < p; i += T::NT)
        for (int j = 0; j <= i; ++j) {
            double s = 0.0;
            for (int k = i; k < p; ++k) s = fma(Li[tri(k, i)], Li[tri(k, j)], s);
            H[tri(i, j)] = s;
        }
    T::sync();
}

// x^T S x (one lane, x a design row)
__device__ __forceinline__ double quad_w(const double* S, const double* x, int p) {
    double q = 0.0;
    for (int i = 0; i < p; ++i) {
        double r = 0.0;
        for (int j = 0; j < i; ++j) r = fma(S[tri(i, j)], x[j], r);
        q = fma(x[i], fma(2.0, r, S[tri(i, i)] * x[i]), q);
    }
    return q;
}

// y = S x, rows split over the lanes
template <int W = 1>
__device__ void matvec_w(const double* S, const double* x, double* y, int p) {
    using T = Team<W>;
    T::sync();
    for (int i = T::tid(); i < p; i += T::NT) {
        double r = 0.0;
        for (int j = 0; j < p; ++j) r = fma(S[j <= i ? tri(i, j) : tri(j, i)], x[j], r);
        y[i] = r;
    }
    T::sync();
}

// sum_ij S_ij T_ij
template <int W = 1>
__device__ double symdot_w(const double* S, const double* U, int p) {
    using T = Team<W>;
    double dg = 0.0, o = 0.0;
    int i = 0, j = T::tid();
    while (j > i) {
        j -= i + 1;
        ++i;
    }
    for (int k = T::tid(); k < p * (p + 1) / 2; k += T::NT) {
        if (i == j) dg = fma(S[k], U[k], dg);
        else o = fma(S[k], U[k], o);
        j += T::NT;
        while (j > i) {
            j -= i + 1;
            ++i;
        }
    }
    return fma(2.0, T::sum(o), T::sum(dg));
}

// L = S + diag(ridge) / + the packed lower triangle `ridge_tri`, then factor
template <int W = 1>
__device__ void factor_ridged(const double* S, double* L, int p, double ridge, const double* ridge_tri) {
    using T = Team<W>;
    T::sync();
    for (int k = T::tid(); k < p * (p + 1) / 2; k += T::NT) L[k] = S[k] + (ridge_tri ? ridge_tri[k] : 0.0);
    T::sync();
    if (!ridge_tri)
        for (int i = T::tid(); i < p; i += T::NT) L[tri(i, i)] += ridge;
    chol_w<W>(L, p);
}

// beta = (X^T X)^+ v (rows of pinv split over the lanes)
template <int W = 1>
__device__ void apply_pinv(const double* pinv, const double* v, double* beta, int p) {
    using T = Team<W>;
    T::sync();
    for (int i = T::tid(); i < p; i += T::NT) {
        double s = 0.0;
        for (int j = 0; j < p; ++j) s = fma(pinv[(size_t)i * p + j], v[j], s);
        beta[i] = s;
    }
    T::sync();
}

// H = (M + ridge)^-1 into ws.L (ws.Li scratch); M in `M`
template <int W = 1>
__device__ void wald_inverse_w(const double* M, const double* ridge_tri, Ws& ws) {
    factor_ridged<W>(M, ws.L, ws.p, 0.0, ridge_tri);
    chol_inverse_w<W>(ws.L, ws.Li, ws.L, ws.p);
}

// SE of contrast c (shared memory or parameter space) against M and H = ws.L; ws.v[6], ws.v[7] scratch
template <int W = 1>
__device__ double wald_se_w(const double* M, const double* c, Ws& ws) {
    using T = Team<W>;
    matvec_w<W>(ws.L, c, ws.v[6], ws.p);
    matvec_w<W>(M, ws.v[6], ws.v[7], ws.p);
    double q = 0.0;
    for (int j = T::tid(); j < ws.p; j += T::NT) q = fma(ws.v[6][j], ws.v[7][j], q);
    return sqrt(T::sum(q));
}

// sum_j a[j] b[j], threads over the components, team total (bit-identical in every thread)
template <int W>
__device__ __forceinline__ double wdot(const double* a, const double* b, int p) {
    using T = Team<W>;
    double s = 0.0;
    for (int j = T::tid(); j < p; j += T::NT) s = fma(a[j], b[j], s);
    return T::sum(s);
}
template <int W>
__device__ __forceinline__ double wmaxabs(const double* a, int p) {
    using T = Team<W>;
    double m = 0.0;
    for (int j = T::tid(); j < p; j += T::NT) m = fmax(m, fabs(a[j]));
    return T::max(m);
}
}  // namespace
}  // namespace pdq
