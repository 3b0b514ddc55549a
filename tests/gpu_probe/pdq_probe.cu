// pdq_probe.cu -- GPU PROBE of the device building blocks.  TEST INFRASTRUCTURE ONLY.
//
// Compiles the real headers (pdq_gene.cuh, which pulls in pdq_fast.cuh and pdq_math.cuh) for sm_90a, so that the DEVICE
// branches of the FP64 primitives, the per-gene recurrence tables, the lane collectives of Group and the packed Cholesky
// family can be compared with high-precision references (tests/test_gpu_math.py).  Nothing from pdq_kernels.cu is used.
// Built by tests/gpu_probe/build.py twice, mirroring the library's units: the default unit (PDQ_UNROLL_P fully unrolled,
// designs p = 1..8) and one with -DPDQ_TU_P=16 -Xptxas -O1 (the loop-and-local-memory code of the wide units, p = 1..16).
//
// The host wrappers take host pointers, allocate, copy, launch and synchronise, and return the CUDA error code (0 on
// success, cudaErrorInvalidValue for arguments they do not accept) instead of aborting.  Every launch does in-bounds work only.
#include <cuda_runtime.h>

#include <stddef.h>

#include "math_ops.h"

using namespace pdq;
using pdq_probe::kTabOut;

#if defined(PDQ_TU_P)
#define PROBE_MAX_P PDQ_TU_P
#else
#define PROBE_MAX_P 8
#endif

namespace {

__device__ double d_mtab[kMathTabLen] = {PDQ_MATH_TABLE_VALUES};

// staged like the kernels stage kMathTab: 16-byte aligned shared memory, because tlog_nb reads its (c, l) pairs as double2
__device__ __forceinline__ const double* stage_math_table(double* s) {
    for (int i = threadIdx.x; i < kMathTabLen; i += blockDim.x) s[i] = d_mtab[i];
    __syncthreads();
    return s;
}

__global__ void k_elem(int op, const double* x, const double* y, double* out, int n) {
    __shared__ __align__(16) double s_tab[kMathTabLen];
    const double* tab = stage_math_table(s_tab);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        out[i] = pdq_probe::apply(op, x[i], y[i], tab);
}

// one warp per block; the lanes are laid out as in the kernels (map_lanes / next_tile): si = lane / gpw, gene slot = lane % gpw
__global__ void k_tables(const double* r, int G, int T, double* out) {
    __shared__ __align__(16) double s_tab[kMathTabLen];
    __shared__ double s_gene[32 * kTabOut];
    const double* tab = stage_math_table(s_tab);
    const int lane = threadIdx.x & 31, gpw = 32 / T;
    const Group grp{lane / gpw, T, gpw};
    const int slot = lane % gpw;
    const int g = blockIdx.x * gpw + slot;
    const bool valid = g < G;
    double* t = s_gene + slot * kTabOut;
    pdq_probe::build_tables(grp, t, valid ? r[g] : 1.0, tab);
    // strided over the lanes of the gene: each lane also reads entries other lanes wrote, as the sweeps do
    if (valid)
        for (int k = grp.si; k < kTabOut; k += T) out[(size_t)g * kTabOut + k] = t[k];
}

// every lane's result of each collective: [sum | excl_scan | argext min | argext max | any] x n
__global__ void k_group(int T, const double* v, const int* flag, double* out, int n) {
    const int lane = threadIdx.x & 31, gpw = 32 / T;
    const Group grp{lane / gpw, T, gpw};
    const int i = blockIdx.x * 32 + lane;
    const double x = v[i];
    const double s = grp.sum(x);
    const double e = grp.excl_scan(x);
    const int amin = grp.argext(x, false);
    const int amax = grp.argext(x, true);
    const bool a = grp.any(flag[i] != 0);
    out[i] = s;
    out[n + i] = e;
    out[2 * n + i] = (double)amin;
    out[3 * n + i] = (double)amax;
    out[4 * n + i] = a ? 1.0 : 0.0;
}

template <int P>
constexpr int spd_width() {
    return 2 * P + P * (P + 1) / 2 + 3;
}

// per packed SPD matrix A, vector b, packed symmetric S: [solve A x = b (P) | A^-1 (packed) | logdet A | b'Ab | A b (P) | sum A_ij S_ij]
template <int P>
__global__ void k_spd(const double* A, const double* b, const double* S, double* out, int count) {
    constexpr int NT = P * (P + 1) / 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    Sym<P> a, s, L, inv;
    double x[P], sol[P], y[P];
PDQ_UNROLL_P
    for (int k = 0; k < NT; ++k) {
        a.a[k] = A[(size_t)i * NT + k];
        s.a[k] = S[(size_t)i * NT + k];
    }
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) x[j] = sol[j] = b[(size_t)i * P + j];
    L = a;
    chol<P>(L);
    chol_solve<P>(L, sol);
    chol_inverse<P>(L, inv);
    const double logdet = chol_logdet<P>(L);
    const double quad = sym_quad<P>(a, x);
    sym_matvec<P>(a, x, y);
    const double dot = sym_dot<P>(a, s);
    double* o = out + (size_t)i * spd_width<P>();
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) o[j] = sol[j];
PDQ_UNROLL_P
    for (int k = 0; k < NT; ++k) o[P + k] = inv.a[k];
    o[P + NT] = logdet;
    o[P + NT + 1] = quad;
PDQ_UNROLL_P
    for (int j = 0; j < P; ++j) o[P + NT + 2 + j] = y[j];
    o[2 * P + NT + 2] = dot;
}

// ---- host side -------------------------------------------------------------------------------------------------------
struct DevBuf {
    void* p = nullptr;
    ~DevBuf() {
        if (p) cudaFree(p);
    }
};

#define PROBE_TRY(expr)                          \
    do {                                         \
        const cudaError_t e_ = (expr);           \
        if (e_ != cudaSuccess) return (int)e_;   \
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

bool valid_lanes(int T) { return T == 1 || T == 2 || T == 4 || T == 8 || T == 16 || T == 32; }

template <int P>
int run_spd(const double* A, const double* b, const double* S, double* out, int count) {
    constexpr int NT = P * (P + 1) / 2;
    DevBuf dA, db, dS, dout;
    PROBE_TRY(upload(dA, A, sizeof(double) * NT * (size_t)count));
    PROBE_TRY(upload(db, b, sizeof(double) * P * (size_t)count));
    PROBE_TRY(upload(dS, S, sizeof(double) * NT * (size_t)count));
    const size_t bytes = sizeof(double) * spd_width<P>() * (size_t)count;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    k_spd<P><<<(count + 63) / 64, 64>>>((const double*)dA.p, (const double*)db.p, (const double*)dS.p, (double*)dout.p, count);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

}  // namespace

extern "C" {

// largest design width this unit instantiates k_spd for
int probe_max_p() { return PROBE_MAX_P; }

int probe_num_ops() { return pdq_probe::kNumOps; }

// out[i] = op(x[i], y[i])  (see math_ops.h; y is ignored by the one-argument ops)
int probe_elem(int op, const double* x, const double* y, double* out, int n) {
    if (op < 0 || op >= pdq_probe::kNumOps || n < 0) return (int)cudaErrorInvalidValue;
    if (n == 0) return 0;
    const size_t bytes = sizeof(double) * (size_t)n;
    DevBuf dx, dy, dout;
    PROBE_TRY(upload(dx, x, bytes));
    PROBE_TRY(upload(dy, y, bytes));
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    const int blocks = (n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024;
    k_elem<<<blocks, 256>>>(op, (const double*)dx.p, (const double*)dy.p, (double*)dout.p, n);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

// out[g * 4 kPsiK + k]: the tables of gene g at r[g] built by T lanes (math_ops.h: build_tables)
int probe_tables(const double* r, int G, int T, double* out) {
    if (!valid_lanes(T) || G < 0) return (int)cudaErrorInvalidValue;
    if (G == 0) return 0;
    const int gpw = 32 / T;
    DevBuf dr, dout;
    PROBE_TRY(upload(dr, r, sizeof(double) * (size_t)G));
    const size_t bytes = sizeof(double) * kTabOut * (size_t)G;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    k_tables<<<(G + gpw - 1) / gpw, 32>>>((const double*)dr.p, G, T, (double*)dout.p);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

// n (a multiple of 32) lanes, groups of T lanes as in the kernels; out = [sum | excl_scan | argmin | argmax | any] x n
int probe_group(int T, const double* v, const int* flag, double* out, int n) {
    if (!valid_lanes(T) || n <= 0 || n % 32 != 0) return (int)cudaErrorInvalidValue;
    DevBuf dv, df, dout;
    PROBE_TRY(upload(dv, v, sizeof(double) * (size_t)n));
    PROBE_TRY(upload(df, flag, sizeof(int) * (size_t)n));
    const size_t bytes = sizeof(double) * 5 * (size_t)n;
    PROBE_TRY(cudaMalloc(&dout.p, bytes));
    k_group<<<n / 32, 32>>>(T, (const double*)dv.p, (const int*)df.p, (double*)dout.p, n);
    PROBE_TRY(finish(out, dout, bytes));
    return 0;
}

// `count` packed P x P SPD matrices: out rows of 2 P + P (P + 1) / 2 + 3 doubles, see k_spd
int probe_spd(int P, const double* A, const double* b, const double* S, double* out, int count) {
    if (count < 0) return (int)cudaErrorInvalidValue;
    if (count == 0) return 0;
    switch (P) {
#define PROBE_SPD_CASE(p) \
    case p:               \
        return (p) <= PROBE_MAX_P ? run_spd<((p) <= PROBE_MAX_P ? (p) : 1)>(A, b, S, out, count) : (int)cudaErrorInvalidValue;
        PROBE_SPD_CASE(1) PROBE_SPD_CASE(2) PROBE_SPD_CASE(3) PROBE_SPD_CASE(4) PROBE_SPD_CASE(5) PROBE_SPD_CASE(6)
        PROBE_SPD_CASE(7) PROBE_SPD_CASE(8) PROBE_SPD_CASE(9) PROBE_SPD_CASE(10) PROBE_SPD_CASE(11) PROBE_SPD_CASE(12)
        PROBE_SPD_CASE(13) PROBE_SPD_CASE(14) PROBE_SPD_CASE(15) PROBE_SPD_CASE(16)
#undef PROBE_SPD_CASE
        default: return (int)cudaErrorInvalidValue;
    }
}

}  // extern "C"
