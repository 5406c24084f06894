// The per-chunk reduction of generalized ICP (Open3D's registration_generalized_icp with
// TransformationEstimationForGeneralizedICP(epsilon, kernel)) and of point-to-plane ICP under a robust kernel
// (TransformationEstimationPointToPlane(kernel)), restated with the library's determinism rules (DESIGN.md section 8,
// "ICP").  Both write the PART_PLANE records of icp.cu's L2 point-to-plane reduction, so the per-pair update, the
// correspondences and the launch sequence are icp.cu's; regtr_icp calls icp_robust_reduce in place of
// k_icp_reduce<true> when the caller passes source normals or a loss other than L2.
#include <cfloat>

#include "icp.cuh"
#include "rigid.cuh"

namespace {

using namespace icp_shared;

// Open3D's RobustKernel::Weight(r) for loss code `loss` (REGTR_ICP_LOSS_*) with parameter k > 0.
__device__ __forceinline__ double robust_weight(int loss, double k, double r) {
    switch (loss) {
    case REGTR_ICP_LOSS_HUBER: { const double a = fabs(r); return a <= k ? 1.0 : k / a; }
    case REGTR_ICP_LOSS_CAUCHY: { const double e = r / k; return 1.0 / (1.0 + e * e); }
    case REGTR_ICP_LOSS_GM: { const double s = k + r * r; return k / (s * s); }
    case REGTR_ICP_LOSS_TUKEY: {
        if (!(fabs(r) <= k)) return 0.0;
        const double e = r / k, u = 1.0 - e * e;
        return u * u;
    }
    default: return 1.0;
    }
}

// One residual row: J = [p x n ; n] with weight w, J^T J (upper triangle, row-major) += w J J^T, J^T r += w J r.
// With w = 1 this is k_icp_reduce<true>'s accumulation operation for operation.
__device__ __forceinline__ void add_row(double px, double py, double pz, double nx, double ny, double nz, double r,
                                        double w, double H[21], double v[6]) {
    const double J[6] = {py * nz - pz * ny, pz * nx - px * nz, px * ny - py * nx, nx, ny, nz};
    int e = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a) {
        const double Jw = w * J[a];
#pragma unroll
        for (int c = a; c < 6; ++c) H[e++] += Jw * J[c];
        v[a] += Jw * r;
    }
}

// R n in float64, no contraction: the rotation part of rt_row.
__device__ __forceinline__ double rot_row(const double* m, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z));
}

// One CTA per chunk of CHUNK consecutive source points of one pair, RED_THREADS threads with a fixed per-thread
// stride and block_sum's fixed tree: deterministic, no atomics, independent of the batch.  part[g] = (k, sum d2,
// J^T J upper triangle row-major, J^T r), the record of k_icp_reduce<true>.
//
// Robust point-to-plane (GICP false): per correspondence (p moved source, q target, n its normal) r = (p - q) . n,
// J = [p x n ; n], weight robust_weight(r).
//
// Generalized ICP (GICP true): every point of the chunk first gets its moved source normal a (round 0: R_init times
// the caller's normal; later rounds: the stored one times the rotation of the update k_icp_nn applied to P this
// round), stored back in snrm.  Per correspondence, with b the target normal and c = 1 - epsilon,
// M = (I - c a a^T) + (I - c b b^T), (S, V) from svd3_jacobi's sweeps, W = V diag(1 / sqrt(S)) V^T; the three rows i of
// W (p - q) give r_i = w_i . (p - q) and J_i = [p x w_i ; w_i] (W [-[p]x | I]), each weighted by robust_weight(r_i).
// A correspondence whose M has an eigenvalue (v_j^T M v_j) or singular value that is not > 0 or not finite stays in
// k and sum d2 but leaves the update.
template <bool GICP>
__global__ void __launch_bounds__(RED_THREADS)
k_icp_robust_reduce(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                    const int32_t* __restrict__ cpre, const double* __restrict__ P, const int32_t* __restrict__ nn,
                    const double* __restrict__ d2, const IcpPair* __restrict__ pst, double* __restrict__ part,
                    const double* __restrict__ tnrm, const double* snrm_in, double* snrm,
                    const double* __restrict__ init, int round, int loss, double loss_k, double c) {
    __shared__ double s_warp[RED_WARPS];
    const int g = blockIdx.x, t = threadIdx.x;
    if (g >= cpre[B]) return;
    const int b = regtr_cloud_of(cpre, B, g);
    if (pst[b].done) return;
    const int i0 = offs[b] + (g - cpre[b]) * CHUNK, i1 = min(i0 + CHUNK, offs[b + 1]);
    const int t0 = offs[B];
    const double* rot = round == 0 ? init + 12 * b : pst[b].upd;
    const double* nsrc = round == 0 ? snrm_in : snrm;
    double k = 0.0, sd = 0.0, H[21], v[6];
    for (int e = 0; e < 21; ++e) H[e] = 0.0;
    for (int e = 0; e < 6; ++e) v[e] = 0.0;
    for (int i = i0 + t; i < i1; i += RED_THREADS) {
        double a[3];
        if constexpr (GICP) {
            const double x = nsrc[3 * i + 0], y = nsrc[3 * i + 1], z = nsrc[3 * i + 2];
            for (int r = 0; r < 3; ++r) {
                a[r] = rot_row(rot + 4 * r, x, y, z);
                snrm[3 * i + r] = a[r];
            }
        }
        const int j = nn[i];
        if (j < 0) continue;
        k += 1.0;
        sd += d2[i];
        const double px = P[3 * i + 0], py = P[3 * i + 1], pz = P[3 * i + 2];
        const double nx = tnrm[3 * (j - t0) + 0], ny = tnrm[3 * (j - t0) + 1], nz = tnrm[3 * (j - t0) + 2];
        if constexpr (!GICP) {
            const double r = (px - xyz[3 * j + 0]) * nx + (py - xyz[3 * j + 1]) * ny + (pz - xyz[3 * j + 2]) * nz;
            add_row(px, py, pz, nx, ny, nz, r, robust_weight(loss, loss_k, r), H, v);
        } else {
            const double bn[3] = {nx, ny, nz};
            double M[3][3], A[3][3], V[3][3];
            for (int r = 0; r < 3; ++r)
                for (int q = 0; q < 3; ++q) {
                    const double id = r == q ? 1.0 : 0.0;
                    M[r][q] = (id - c * a[r] * a[q]) + (id - c * bn[r] * bn[q]);
                    A[r][q] = M[r][q];
                    V[r][q] = id;
                }
            jacobi3_sweeps(A, V);              // svd3_jacobi's S and V, unsorted: W does not depend on the order
            bool ok = true;
            double is[3];
            for (int q = 0; q < 3; ++q) {
                const double S = sqrt(A[0][q] * A[0][q] + A[1][q] * A[1][q] + A[2][q] * A[2][q]);
                double lam = 0.0;
                for (int r = 0; r < 3; ++r)
                    lam += V[r][q] * (M[r][0] * V[0][q] + M[r][1] * V[1][q] + M[r][2] * V[2][q]);
                ok = ok && S > 0.0 && S <= DBL_MAX && lam > 0.0 && lam <= DBL_MAX;
                is[q] = 1.0 / sqrt(S);
            }
            if (!ok) continue;
            const double dx = px - xyz[3 * j + 0], dy = py - xyz[3 * j + 1], dz = pz - xyz[3 * j + 2];
            for (int r = 0; r < 3; ++r) {
                double w[3];
                for (int q = 0; q < 3; ++q)
                    w[q] = (V[r][0] * V[q][0] * is[0] + V[r][1] * V[q][1] * is[1]) + V[r][2] * V[q][2] * is[2];
                const double res = dx * w[0] + dy * w[1] + dz * w[2];
                add_row(px, py, pz, w[0], w[1], w[2], res, robust_weight(loss, loss_k, res), H, v);
            }
        }
    }
    double out[PART_PLANE];
    out[0] = block_sum(k, s_warp);
    out[1] = block_sum(sd, s_warp);
    for (int e = 0; e < 21; ++e) out[2 + e] = block_sum(H[e], s_warp);
    for (int e = 0; e < 6; ++e) out[23 + e] = block_sum(v[e], s_warp);
    if (t != 0) return;
    double* o = part + (size_t)PART_PLANE * g;
    for (int e = 0; e < PART_PLANE; ++e) o[e] = out[e];
}

}  // namespace

namespace icp_shared {

int icp_robust_reduce(int gicp, int blocks, cudaStream_t st, const double* xyz, const int32_t* offs, int B,
                      const int32_t* cpre, const double* P, const int32_t* nn, const double* d2, const IcpPair* pst,
                      double* part, const double* tgt_normals, const double* src_normals, double* snrm,
                      const double* init, int round, int loss, double loss_k, double epsilon) {
    const double c = 1.0 - epsilon;
    if (gicp)
        k_icp_robust_reduce<true><<<blocks, RED_THREADS, 0, st>>>(xyz, offs, B, cpre, P, nn, d2, pst, part,
                                                                  tgt_normals, src_normals, snrm, init, round, loss,
                                                                  loss_k, c);
    else
        k_icp_robust_reduce<false><<<blocks, RED_THREADS, 0, st>>>(xyz, offs, B, cpre, P, nn, d2, pst, part,
                                                                   tgt_normals, nullptr, nullptr, init, round, loss,
                                                                   loss_k, c);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // namespace icp_shared
