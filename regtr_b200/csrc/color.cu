// Colored ICP (Park et al.; Open3D's registration_colored_icp): the targets' intensity gradients
// (InitializePointCloudForColoredICP) and the colored mode of the point-to-plane family's reduction (icp.cuh), which
// regtr_icp launches in place of the other modes' (DESIGN.md section 8, "ICP").
//
// Gradients: one cell list over the fp32 copy of every cloud is built once, then one warp per point selects its
// neighbours with normal estimation's search (neighbours.cuh) and solves a 3x3 least-squares system: 1 + 4 + 1
// launches whatever C, no host synchronisation, no value atomics.
#include "icp.cuh"
#include "neighbours.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int GRD_WARPS = 8;
constexpr int GRD_MAX_NN = 64;         // two selected indices per lane, as the normals

// The fp32 copy of the clouds for their cell list, and the range check: |coordinate| beyond `bound`, or not finite,
// raises REGTR_STATUS_RANGE.
__global__ void k_color_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
                             double bound, float* __restrict__ x32, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    x32[3 * i + 0] = (float)x; x32[3 * i + 1] = (float)y; x32[3 * i + 2] = (float)z;
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One warp per point, in index order: the neighbours of warp_select_neighbours, then A^T A (upper triangle) and A^T b
// summed over the rows in order by every lane (the header's regtr_color_gradients), and lane 0 solves.
__global__ void __launch_bounds__(GRD_WARPS * 32)
k_color_gradients(const double* __restrict__ xyz, const double* __restrict__ nrm, const double* __restrict__ rgb,
                  const int32_t* __restrict__ offs, int C, int n_cap, const CellSlot* __restrict__ table, int log2t,
                  const float4* __restrict__ sxyzi, float cell, double r2, int max_nn, double* __restrict__ grad) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[C];
    for (int qi = blockIdx.x * GRD_WARPS + warp; qi < n_cap && qi < n; qi += gridDim.x * GRD_WARPS) {
        const int c = regtr_cloud_of(offs, C, qi);
        const double px = xyz[3 * qi + 0], py = xyz[3 * qi + 1], pz = xyz[3 * qi + 2];
        const double nx = nrm[3 * qi + 0], ny = nrm[3 * qi + 1], nz = nrm[3 * qi + 2];
        int sel[GRD_MAX_NN / 32];
        const int cnt = warp_select_neighbours(xyz, table, log2t, sxyzi, cell, c, px, py, pz, r2, max_nn, lane, sel);
        double g[3] = {0.0, 0.0, 0.0};
        if (cnt >= 4 && !(nx == 0.0 && ny == 0.0 && nz == 0.0)) {
            const double it = intensity(rgb + 3 * qi);
            double H[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, v[3] = {0.0, 0.0, 0.0};
            for (int s = 1; s < cnt; ++s) {
                const int j = sel_at(sel, s);
                const double qx = xyz[3 * j + 0], qy = xyz[3 * j + 1], qz = xyz[3 * j + 2];
                const double d = ((qx - px) * nx + (qy - py) * ny) + (qz - pz) * nz;
                const double a[3] = {(qx - d * nx) - px, (qy - d * ny) - py, (qz - d * nz) - pz};
                const double bi = intensity(rgb + 3 * j) - it;
                for (int r = 0, e = 0; r < 3; ++r) {
                    for (int q = r; q < 3; ++q, ++e) H[e] += a[r] * a[q];
                    v[r] -= a[r] * bi;                  // solve_ldlt solves for -v
                }
            }
            const double w = (double)(cnt - 1), a[3] = {w * nx, w * ny, w * nz};
            for (int r = 0, e = 0; r < 3; ++r)
                for (int q = r; q < 3; ++q, ++e) H[e] += a[r] * a[q];
            double x[3];
            if (lane == 0 && solve_ldlt<3>(H, v, x))
                for (int r = 0; r < 3; ++r) g[r] = x[r];
        }
        if (lane == 0)
            for (int r = 0; r < 3; ++r) grad[3 * qi + r] = g[r];
    }
}

struct GrdWs {
    float* x32;
    void *grid, *gws;
    size_t gws_bytes, total;
};

GrdWs carve_gradients(void* ws, int n_cap) {
    GrdWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    w.x32 = (float*)take(sizeof(float) * 3 * (size_t)n_cap);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.total = off;
    return w;
}

}  // namespace

void regtr_icp_reduce_colored(int blocks, cudaStream_t st, const double* xyz, const int32_t* offs, int B,
                              const int32_t* cpre, const double* P, const int32_t* nn, const double* d2,
                              const void* pst, double* part, const double* tnrm, int loss, double loss_k,
                              const double* src_rgb, const double* tgt_rgb, const double* grad, double sl, double sp) {
    k_icp_reduce_plane<PLANE_COLOR><<<blocks, RED_THREADS, 0, st>>>(
        xyz, offs, B, cpre, P, nn, d2, (const IcpPair*)pst, part, tnrm, nullptr, nullptr, nullptr, 0, loss, loss_k, 0.0,
        IcpColor{src_rgb, tgt_rgb, grad, sl, sp});
}

extern "C" {

size_t regtr_color_gradients_ws_bytes(int n_cap) { return carve_gradients(nullptr, n_cap > 0 ? n_cap : 1).total; }
size_t regtr_color_gradients_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap > 0 ? n_cap : 1); }

int regtr_color_gradients(const double* xyz, const double* normals, const double* colors, const int32_t* offs, int C,
                          int n_cap, double radius, float cell, int max_nn, double* grad, uint32_t* status, void* ws,
                          size_t ws_bytes, void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !status || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || !(radius > 0.0) ||
        !((double)cell > radius) || max_nn < 1 || max_nn > GRD_MAX_NN ||
        (n_cap > 0 && (!xyz || !normals || !colors || !grad)))
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1;      // offs[C] = 0 without points: every kernel then reads no xyz
    GrdWs w = carve_gradients(ws, nc);
    if (ws_bytes < w.total || state_bytes < regtr_color_gradients_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const double bound = regtr_overlap_coord_bound(radius, cell);
    const int T = 256;
    k_color_init<<<regtr_cdiv(nc, T), T, 0, st>>>(xyz, offs, C, nc, bound, w.x32, status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, C, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes, state,
                                        state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const int blocks = regtr_cdiv(nc, GRD_WARPS) < 4 * REGTR_NUM_SMS ? regtr_cdiv(nc, GRD_WARPS) : 4 * REGTR_NUM_SMS;
    k_color_gradients<<<blocks, GRD_WARPS * 32, 0, st>>>(xyz, normals, colors, offs, C, nc, grid_table(w.grid, (size_t)nc),
                                                         cell_table_log2(nc), grid_sxyzi(w.grid), cell, radius * radius,
                                                         max_nn, grad);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
