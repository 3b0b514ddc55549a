// pdq_launch.cuh -- what the kernel units (pdq_kernels.cu, pdq_common.cu, pdq_wide.cu, pdq_padj.cu) share around a launch: the
// block and gene tiles of the narrow per-gene kernels, the dynamic shared-memory opt-in, the launch check, and the one mapping
// of host parameters and PDQ_DEBUG_* test hooks to the kernels' parameters.
#pragma once

#include <cuda_runtime.h>
#include <math.h>

#include "pdq_gene.cuh"
#include "pdq_internal.h"

namespace pdq {

// the narrow per-gene kernels (p <= 16, pdq_kernels.cu) and the size-factor means (pdq_common.cu): kWarps warps per block, each
// owning 32 / T adjacent genes of T lanes
constexpr int kBlock = 128;
constexpr int kWarps = kBlock / 32;

// gene of a lane when block `block` (default: this block) takes the block's genes in order; grid_for blocks cover G genes
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

inline int grid_for(int G, int lgT) {
    const int genes_per_block = kWarps * (32 >> lgT);
    return (G + genes_per_block - 1) / genes_per_block;
}

// a kernel that takes more than 48 KB of dynamic shared memory has to opt in first
template <class K>
int prep(K kernel, size_t smem) {
    if (smem > kMaxDynSmem) return PDQ_ERR_UNSUPPORTED;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
        return PDQ_ERR_CUDA;
    return 0;
}

inline int check_launch() { return cudaGetLastError() == cudaSuccess ? 0 : PDQ_ERR_CUDA; }

// a test hook of the launch (LaunchCfg::debug, PDQ_DEBUG_*) as the 0 / 1 switch the kernels take
inline int hook(int debug, int flag) { return (debug & flag) ? 1 : 0; }

inline IrlsParams irls_params(const IrlsHost& h, const DesignDev& d, int debug) {
    return IrlsParams{h.min_mu, h.beta_tol, h.min_beta, h.max_beta, h.maxiter, d.full_rank, d.few_rows, hook(debug, PDQ_DEBUG_FAIL_IRLS_OPTIMIZER)};
}

inline AlphaParams alpha_params(double min_disp, double max_disp, double prior_var, int cr_reg, int prior_reg) {
    return AlphaParams{log(min_disp), log(max_disp), prior_var, cr_reg, prior_reg};
}

}  // namespace pdq
