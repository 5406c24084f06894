// Internal to the library: the pieces ICP's reductions share between icp.cu (point-to-point and L2 point-to-plane)
// and gicp.cu (generalized ICP and robust point-to-plane).  They live in a named namespace so that the per-pair state
// can cross between the two translation units.
#pragma once

#include "common.cuh"

namespace icp_shared {

constexpr int CHUNK = 1024;            // source points per CTA of the reduction
constexpr int RED_THREADS = 256;
constexpr int RED_WARPS = RED_THREADS / 32;
constexpr int PART_PLANE = 29;         // k, sum d2, J^T J[21] (upper triangle, row-major), J^T r[6] per chunk

// Per-pair state between rounds (written by k_icp_update only).
struct IcpPair {
    double upd[12];                    // the update of the last round, applied to P by the next k_icp_nn
    double fit, rmse;                  // the current correspondences' fitness and inlier RMSE
    int k, iters, done, pad;
};

// Sum over the CTA in a fixed order: the xor butterfly inside each warp, then the warp totals in warp order.  Every
// thread returns the total.
__device__ __forceinline__ double block_sum(double v, double* s_warp) {
    v = warp_sum(v);
    __syncthreads();                   // s_warp may still be read by the previous call
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < RED_WARPS; ++w) t += s_warp[w];
    return t;
}

// One round's per-chunk reduction of generalized ICP (gicp != 0) or of point-to-plane ICP under a robust loss, into
// the PART_PLANE records that k_icp_update<true> consumes (gicp.cu).  `blocks` CTAs, one per chunk as in
// k_icp_reduce.  snrm (n_cap,3) is the workspace copy of the moved source normals: round 0 fills it from
// src_normals rotated by init, later rounds rotate it in place by the update k_icp_nn applied to P.
int icp_robust_reduce(int gicp, int blocks, cudaStream_t st, const double* xyz, const int32_t* offs, int B,
                      const int32_t* cpre, const double* P, const int32_t* nn, const double* d2, const IcpPair* pst,
                      double* part, const double* tgt_normals, const double* src_normals, double* snrm,
                      const double* init, int round, int loss, double loss_k, double epsilon);

}  // namespace icp_shared
