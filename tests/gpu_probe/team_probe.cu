// team_probe.cu -- GPU PROBE of the team building blocks of pdq_team.cuh.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the header the wide-design kernels (pdq_wide.cu) are built from, with the library's flags, so that the cooperative
// code the kernels run -- Team<W>::sum / max / any, rank_chunk / vec_chunk, the packed Cholesky family, matvec_w, symdot_w,
// quad_w, apply_pinv, wald_inverse_w / wald_se_w, wdot / wmaxabs -- can be compared with extended-precision references at every
// team width W = 1, 2, 4, 8 and p = 1..128 (tests/test_gpu_team.py, tests/team_checks.py).  Each kernel runs one block of 32 W
// threads per problem on the workspace the kernels use: wide_ws_doubles(p, W) doubles of dynamic shared memory, carved by carve<W>.
//
// The host wrappers follow pdq_probe.cu: host pointers in; allocate, copy, launch, synchronise, copy back; the CUDA error code
// is returned (cudaErrorInvalidValue for p outside 1..128 or W outside {1, 2, 4, 8}) instead of aborting.  In-bounds work only.
#include <cuda_runtime.h>

#include <stddef.h>

#include <type_traits>
#include <vector>

#include "../../pydeseq2_b200/csrc/pdq_team.cuh"

// a named namespace: the header's kernels-side code sits in pdq's anonymous namespace, and a second anonymous namespace
// brought in next to it by `using namespace pdq` makes nvcc's launch stubs ambiguous
namespace team_probe {

using namespace pdq;

constexpr int kMaxP = 128;
constexpr int kSpdScalars = 4;  // per thread: logdet, symdot, quad, Wald SE
constexpr int kCollOut = 8;     // per thread: sum, max, sum, any, max, sum, wdot, wmaxabs

__host__ __device__ constexpr int packed(int p) { return p * (p + 1) / 2; }
// per problem: [L | x | H | Li | A b | P b]
__host__ __device__ constexpr int spd_width(int p) { return 3 * packed(p) + 3 * p; }

// One SPD problem per block.  A, S, ridge_tri packed (np each); b, c (p); P dense p x p row-major.  `ridge_tri` null: the
// scalar ridge[g] is added to the diagonal (factor_ridged's first mode) and the Wald inverse is of A alone; otherwise both the
// factor and the Wald inverse add the packed triangle, as the Wald step of the kernels does.
template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1)
    k_team_spd(const double* A, const double* b, const double* S, const double* P, const double* c, const double* ridge,
               const double* ridge_tri, int p, double* out, double* scal) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, p);
    const int g = blockIdx.x, np = packed(p), t = T::tid();
    const double* rt = ridge_tri ? ridge_tri + (size_t)g * np : nullptr;
    wcopy<W>(ws.A, A + (size_t)g * np, np);
    wcopy<W>(ws.v[0], b + (size_t)g * p, p);
    wcopy<W>(ws.v[2], b + (size_t)g * p, p);
    wcopy<W>(ws.v[5], c + (size_t)g * p, p);
    T::sync();
    double* o = out + (size_t)g * spd_width(p);
    double* sc = scal + (size_t)g * kSpdScalars * T::NT;

    matvec_w<W>(ws.A, ws.v[0], ws.v[3], p);
    apply_pinv<W>(P + (size_t)g * p * p, ws.v[0], ws.v[4], p);
    sc[T::NT + t] = symdot_w<W>(ws.A, S + (size_t)g * np, p);

    factor_ridged<W>(ws.A, ws.L, p, ridge[g], rt);
    wcopy<W>(o, ws.L, np);
    double ld2 = 0.0;  // as loss_w sums log L_ii
    for (int i = 0; i < p; ++i) ld2 += log(ws.L[tri(i, i)]);
    sc[t] = 2.0 * ld2;
    chol_solve_w<W>(ws.L, ws.v[2], p);
    chol_inverse_w<W>(ws.L, ws.Li, ws.L, p);  // H into L, as the kernels call it
    sc[2 * T::NT + t] = quad_w(ws.L, ws.v[0], p);
    wcopy<W>(o + np, ws.v[2], p);
    wcopy<W>(o + np + p, ws.L, np);
    wcopy<W>(o + 2 * np + p, ws.Li, np);
    wcopy<W>(o + 3 * np + p, ws.v[3], p);
    wcopy<W>(o + 3 * np + 2 * p, ws.v[4], p);

    wald_inverse_w<W>(ws.A, rt, ws);
    sc[3 * T::NT + t] = wald_se_w<W>(ws.A, ws.v[5], ws);
}

// X^T W X (packed) and X^T W z of one weight / response set per block, staged chunk by chunk as irls_sweep_w stages them
template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1)
    k_team_acc(const double* pack, int N, int p, const double* w, const double* z, double* out) {
    using T = Team<W>;
    extern __shared__ __align__(16) double wsm[];
    Ws ws = carve<W>(wsm, p);
    const int g = blockIdx.x, np = packed(p);
    const DesignS d = design_of(pack, N, p);
    w += (size_t)g * N;
    z += (size_t)g * N;
    wfill<W>(ws.A, np, 0.0);
    wfill<W>(ws.v[0], p, 0.0);
    for (int n0 = 0; n0 < N; n0 += T::NT) {
        const int n = n0 + T::tid();
        const double wt = n < N ? w[n] : 0.0, wz = n < N ? z[n] : 0.0;
        T::sync();
        ws.cw[T::tid()] = wt;
        ws.cz[T::tid()] = wz;
        T::sync();
        const int cnt = min(T::NT, N - n0);
        rank_chunk<W>(d, p, n0, cnt, ws.cw, ws.A);
        vec_chunk<W>(d, p, n0, cnt, ws.cz, ws.v[0]);
    }
    T::sync();
    wcopy<W>(out + (size_t)g * (np + p), ws.A, np);
    wcopy<W>(out + (size_t)g * (np + p) + np, ws.v[0], p);
}

// Every thread's result of sum(v0), max(v1), sum(v2), any(f), max(v3), sum(v4) -- back to back, so that each call reuses the
// shared slots the previous one released -- then wdot(a, b) and wmaxabs(a) over this block's len[g] components (staged in
// shared memory, as the shrinkage kernels hold their vectors).  v: 5 NT per block, f: NT, a / b: maxn per block.
template <int W>
__global__ void __launch_bounds__(32 * W, W == 1 ? 0 : 1)
    k_team_coll(const double* v, const int* f, const double* a, const double* b, const int* len, int maxn, double* out) {
    using T = Team<W>;
    extern __shared__ __align__(16) double sv[];
    const int g = blockIdx.x, t = T::tid(), n = len[g];
    const double* x = v + (size_t)g * 5 * T::NT;
    double* o = out + (size_t)g * kCollOut * T::NT;
    wcopy<W>(sv, a + (size_t)g * maxn, n);
    wcopy<W>(sv + maxn, b + (size_t)g * maxn, n);
    T::sync();
    o[t] = T::sum(x[t]);
    o[T::NT + t] = T::max(x[T::NT + t]);
    o[2 * T::NT + t] = T::sum(x[2 * T::NT + t]);
    o[3 * T::NT + t] = T::any(f[(size_t)g * T::NT + t] != 0) ? 1.0 : 0.0;
    o[4 * T::NT + t] = T::max(x[3 * T::NT + t]);
    o[5 * T::NT + t] = T::sum(x[4 * T::NT + t]);
    o[6 * T::NT + t] = wdot<W>(sv, sv + maxn, n);
    o[7 * T::NT + t] = wmaxabs<W>(sv, n);
}

// ---- host side -------------------------------------------------------------------------------------------------------
struct DevBuf {
    void* p = nullptr;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
};

#define PROBE_TRY(expr)                        \
    do {                                       \
        const cudaError_t e_ = (expr);         \
        if (e_ != cudaSuccess) return (int)e_; \
    } while (0)

cudaError_t upload(DevBuf& d, const void* h, size_t bytes) {
    cudaError_t e = cudaMalloc(&d.p, bytes);
    if (e != cudaSuccess) return e;
    return cudaMemcpy(d.p, h, bytes, cudaMemcpyHostToDevice);
}

cudaError_t finish(void* h_out, const DevBuf& d_out, size_t bytes) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return e;
    return cudaMemcpy(h_out, d_out.p, bytes, cudaMemcpyDeviceToHost);
}

// the dynamic shared memory of a launch; above the default 48 KB the kernel has to opt in, as launch_team does
template <class K>
cudaError_t allow_smem(K kernel, size_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

bool valid_pw(int p, int W) { return p >= 1 && p <= kMaxP && (W == 1 || W == 2 || W == 4 || W == 8); }

template <int W>
int run_spd(int p, const double* A, const double* b, const double* S, const double* P, const double* c, const double* ridge,
            const double* ridge_tri, int count, double* out, double* scal) {
    const size_t np = packed(p), smem = wide_ws_doubles(p, W) * sizeof(double);
    DevBuf dA, db, dS, dP, dc, dr, drt, dout, dscal;
    PROBE_TRY(upload(dA, A, sizeof(double) * np * count));
    PROBE_TRY(upload(db, b, sizeof(double) * p * count));
    PROBE_TRY(upload(dS, S, sizeof(double) * np * count));
    PROBE_TRY(upload(dP, P, sizeof(double) * p * p * count));
    PROBE_TRY(upload(dc, c, sizeof(double) * p * count));
    PROBE_TRY(upload(dr, ridge, sizeof(double) * count));
    if (ridge_tri) PROBE_TRY(upload(drt, ridge_tri, sizeof(double) * np * count));
    const size_t bytes = sizeof(double) * spd_width(p) * count, sbytes = sizeof(double) * kSpdScalars * 32 * W * count;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    PROBE_TRY(cudaMalloc(&dscal.p, sbytes));
    PROBE_TRY(allow_smem(k_team_spd<W>, smem));
    k_team_spd<W><<<count, 32 * W, smem>>>((const double*)dA.p, (const double*)db.p, (const double*)dS.p, (const double*)dP.p,
                                          (const double*)dc.p, (const double*)dr.p, (const double*)drt.p, p, (double*)dout.p,
                                          (double*)dscal.p);
    PROBE_TRY(finish(out, dout, bytes));
    PROBE_TRY(cudaMemcpy(scal, dscal.p, sbytes, cudaMemcpyDeviceToHost));
    return 0;
}

template <int W>
int run_acc(int p, int N, const double* X, const double* w, const double* z, int count, double* out) {
    std::vector<double> pack;
    design_pack(X, nullptr, false, N, p, pack);
    const size_t smem = wide_ws_doubles(p, W) * sizeof(double);
    DevBuf dpack, dw, dz, dout;
    PROBE_TRY(upload(dpack, pack.data(), sizeof(double) * pack.size()));
    PROBE_TRY(upload(dw, w, sizeof(double) * N * count));
    PROBE_TRY(upload(dz, z, sizeof(double) * N * count));
    const size_t bytes = sizeof(double) * (packed(p) + p) * count;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    PROBE_TRY(allow_smem(k_team_acc<W>, smem));
    k_team_acc<W><<<count, 32 * W, smem>>>((const double*)dpack.p, N, p, (const double*)dw.p, (const double*)dz.p, (double*)dout.p);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

template <int W>
int run_coll(const double* v, const int* f, const double* a, const double* b, const int* len, int maxn, int count, double* out) {
    constexpr int NT = 32 * W;
    const size_t smem = 2 * (size_t)maxn * sizeof(double);
    DevBuf dv, df, da, db, dl, dout;
    PROBE_TRY(upload(dv, v, sizeof(double) * 5 * NT * count));
    PROBE_TRY(upload(df, f, sizeof(int) * NT * count));
    PROBE_TRY(upload(da, a, sizeof(double) * maxn * count));
    PROBE_TRY(upload(db, b, sizeof(double) * maxn * count));
    PROBE_TRY(upload(dl, len, sizeof(int) * count));
    const size_t bytes = sizeof(double) * kCollOut * NT * count;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    PROBE_TRY(allow_smem(k_team_coll<W>, smem));
    k_team_coll<W><<<count, NT, smem>>>((const double*)dv.p, (const int*)df.p, (const double*)da.p, (const double*)db.p,
                                        (const int*)dl.p, maxn, (double*)dout.p);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

template <class F>
int with_team(int W, F&& f) {
    switch (W) {
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 4: return f(std::integral_constant<int, 4>{});
        case 8: return f(std::integral_constant<int, 8>{});
        default: return (int)cudaErrorInvalidValue;
    }
}

}  // namespace team_probe

using namespace team_probe;

extern "C" {

int team_max_p() { return kMaxP; }

// bytes of dynamic shared memory of one problem (wide_ws_doubles)
size_t team_ws_bytes(int p, int W) { return valid_pw(p, W) ? wide_ws_doubles(p, W) * sizeof(double) : 0; }

// `count` problems: out rows of spd_width(p) = [L | x | H | Li | A b | P b], scal rows of 4 x 32 W = [logdet | symdot | quad |
// Wald SE] of every thread.  ridge: one scalar per problem; ridge_tri: null, or one packed triangle per problem (see k_team_spd)
int team_spd(int p, int W, const double* A, const double* b, const double* S, const double* P, const double* c,
             const double* ridge, const double* ridge_tri, int count, double* out, double* scal) {
    if (!valid_pw(p, W) || count < 0) return (int)cudaErrorInvalidValue;
    if (count == 0) return 0;
    return with_team(W, [&](auto w) { return run_spd<decltype(w)::value>(p, A, b, S, P, c, ridge, ridge_tri, count, out, scal); });
}

// X (N x p, row-major) packed by design_pack; `count` weight / response sets w, z (N each): out rows [X^T W X packed | X^T W z]
int team_acc(int p, int W, int N, const double* X, const double* w, const double* z, int count, double* out) {
    if (!valid_pw(p, W) || N < 1 || count < 0) return (int)cudaErrorInvalidValue;
    if (count == 0) return 0;
    return with_team(W, [&](auto t) { return run_acc<decltype(t)::value>(p, N, X, w, z, count, out); });
}

// `count` blocks of 32 W threads: out rows of 8 x 32 W (see k_team_coll); len[g] in 0..maxn
int team_coll(int W, const double* v, const int* f, const double* a, const double* b, const int* len, int maxn, int count,
              double* out) {
    if (!valid_pw(1, W) || maxn < 1 || maxn > 4096 || count < 0) return (int)cudaErrorInvalidValue;
    for (int g = 0; g < count; ++g)
        if (len[g] < 0 || len[g] > maxn) return (int)cudaErrorInvalidValue;
    if (count == 0) return 0;
    return with_team(W, [&](auto t) { return run_coll<decltype(t)::value>(v, f, a, b, len, maxn, count, out); });
}

}  // extern "C"
