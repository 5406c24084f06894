// Internal to the library: the point-to-plane family's per-chunk reduction of ICP, shared by icp.cu (L2, robust and
// generalized modes) and color.cu (the colored mode).  Each translation unit instantiates only its own modes, so
// adding a mode leaves the code of the others as it was.
#pragma once

#include <cfloat>

#include "cellgrid.cuh"
#include "rigid.cuh"

namespace {

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

// The point-to-plane family's loss modes: L2 point-to-plane, point-to-plane under a robust kernel, generalized ICP
// (under the robust kernel `loss`, L2 included), colored ICP (likewise).
enum PlaneMode { PLANE_L2, PLANE_ROBUST, PLANE_GICP, PLANE_COLOR };

// Colored ICP's inputs: source and target rgb (stacked like their clouds), the targets' intensity gradients, and
// sqrt(lambda_geometric), sqrt(1 - lambda_geometric).  Unused by the other modes.
struct IcpColor {
    const double *src, *tgt, *grad;
    double sl, sp;
};

// ((r + g) + b) / 3: Open3D's intensity of an rgb colour
__device__ __forceinline__ double intensity(const double* c) { return ((c[0] + c[1]) + c[2]) / 3.0; }

// One CTA per chunk as in k_icp_reduce_point, one pass: part[g] = (k, sum d2, J^T J upper triangle row-major, J^T r).
//
// L2 and robust point-to-plane: per correspondence (p moved source, q target, n = tnrm[j - offs[B]] its normal)
// r = (p - q) . n, J = [p x n ; n], weight 1 (L2, decided at compile time) or robust_weight(r).
//
// Generalized ICP: every point of the chunk first gets its moved source normal a (round 0: R_init times the caller's
// normal snrm_in; later rounds: the stored one times the rotation of the update k_icp_nn applied to P this round),
// stored back in snrm.  Per correspondence, with b the target normal and c = 1 - epsilon,
// M = (I - c a a^T) + (I - c b b^T), (S, V) from svd3_jacobi's sweeps, W = V diag(1 / sqrt(S)) V^T; the three rows i of
// W (p - q) give r_i = w_i . (p - q) and J_i = [p x w_i ; w_i] (W [-[p]x | I]), each weighted by robust_weight(r_i).
// A correspondence whose M has an eigenvalue (v_j^T M v_j) or singular value that is not > 0 or not finite stays in
// k and sum d2 but leaves the update.
//
// Colored ICP (Open3D's TransformationEstimationForColoredICP): a correspondence with a zero target normal n stays in
// k and sum d2 and leaves the update.  Otherwise, with g = (p - q) . n, two rows: the geometric one r = sl g,
// J = [p x sl n ; sl n]; and the photometric one, with d the target's gradient, p' = p - g n,
// is0 = d . (p' - q) + it_q and m = (d . n) n - d: r = sp (is_p - is0), J = [p x sp m ; sp m].  Each row is weighted
// by robust_weight of its own r.
template <PlaneMode MODE>
__global__ void __launch_bounds__(RED_THREADS)
k_icp_reduce_plane(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                   const int32_t* __restrict__ cpre, const double* __restrict__ P, const int32_t* __restrict__ nn,
                   const double* __restrict__ d2, const IcpPair* __restrict__ pst, double* __restrict__ part,
                   const double* __restrict__ tnrm, const double* snrm_in, double* snrm,
                   const double* __restrict__ init, int round, int loss, double loss_k, double c, IcpColor col) {
    constexpr bool GICP = MODE == PLANE_GICP;
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
        if constexpr (MODE == PLANE_COLOR) {
            if (nx == 0.0 && ny == 0.0 && nz == 0.0) continue;
            const double qx = xyz[3 * j + 0], qy = xyz[3 * j + 1], qz = xyz[3 * j + 2];
            const double r = (px - qx) * nx + (py - qy) * ny + (pz - qz) * nz;
            const double rg = col.sl * r;
            add_row(px, py, pz, col.sl * nx, col.sl * ny, col.sl * nz, rg, robust_weight(loss, loss_k, rg), H, v);
            const double* d = col.grad + 3 * (j - t0);
            const double ux = (px - r * nx) - qx, uy = (py - r * ny) - qy, uz = (pz - r * nz) - qz;
            const double is0 = ((d[0] * ux + d[1] * uy) + d[2] * uz) + intensity(col.tgt + 3 * (j - t0));
            const double dn = (d[0] * nx + d[1] * ny) + d[2] * nz;
            const double ri = col.sp * (intensity(col.src + 3 * i) - is0);
            add_row(px, py, pz, col.sp * (dn * nx - d[0]), col.sp * (dn * ny - d[1]), col.sp * (dn * nz - d[2]), ri,
                    robust_weight(loss, loss_k, ri), H, v);
        } else if constexpr (!GICP) {
            const double r = (px - xyz[3 * j + 0]) * nx + (py - xyz[3 * j + 1]) * ny + (pz - xyz[3 * j + 2]) * nz;
            add_row(px, py, pz, nx, ny, nz, r, MODE == PLANE_L2 ? 1.0 : robust_weight(loss, loss_k, r), H, v);
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

// The colored mode's launch (color.cu): k_icp_reduce_plane<PLANE_COLOR> with regtr_icp's arguments.  pst is the
// IcpPair array.
void regtr_icp_reduce_colored(int blocks, cudaStream_t st, const double* xyz, const int32_t* offs, int B,
                              const int32_t* cpre, const double* P, const int32_t* nn, const double* d2,
                              const void* pst, double* part, const double* tnrm, int loss, double loss_k,
                              const double* src_rgb, const double* tgt_rgb, const double* grad, double sl, double sp);
