// Normal estimation for C stacked clouds: Open3D's estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) followed
// by orient_normals_towards_camera_location() at the origin, restated with this library's tie and boundary rules
// (DESIGN.md section 8, "Normals").  Its output feeds point-to-plane ICP (regtr_icp with tgt_normals).
//
// One cell list over the fp32 copy of every cloud is built once, then one warp per point selects its neighbours and
// solves the 3x3 eigenproblem: 1 + 4 + 1 launches whatever C, no host synchronisation, no value atomics.
#include "neighbours.cuh"
#include "rigid.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int NRM_WARPS = 8;
constexpr int NRM_MAX_NN = 64;         // two selected indices per lane

// The fp32 copy of the clouds for their cell list, and the range check: |coordinate| beyond `bound`, or not finite,
// raises REGTR_STATUS_RANGE.
__global__ void k_normals_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
                               double bound, float* __restrict__ x32, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    x32[3 * i + 0] = (float)x; x32[3 * i + 1] = (float)y; x32[3 * i + 2] = (float)z;
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One warp per point, in index order: the neighbours of warp_select_neighbours (neighbours.cuh).  Then, in that order,
// the mean and the centred covariance (float64, sequential sums, / count), its smallest eigenvector (the right singular
// vector of the smallest singular value of svd3_jacobi), normalised and flipped when n . p > 0.  Fewer than 3
// neighbours: 0.
__global__ void __launch_bounds__(NRM_WARPS * 32)
k_normals(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
          const CellSlot* __restrict__ table, int log2t, const float4* __restrict__ sxyzi, float cell, double r2,
          int max_nn, double* __restrict__ normals, int32_t* __restrict__ counts) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[C];
    for (int qi = blockIdx.x * NRM_WARPS + warp; qi < n_cap && qi < n; qi += gridDim.x * NRM_WARPS) {
        const int c = regtr_cloud_of(offs, C, qi);
        const double qx = xyz[3 * qi + 0], qy = xyz[3 * qi + 1], qz = xyz[3 * qi + 2];
        int sel[NRM_MAX_NN / 32];
        const int cnt = warp_select_neighbours(xyz, table, log2t, sxyzi, cell, c, qx, qy, qz, r2, max_nn, lane, sel);
        double nx = 0.0, ny = 0.0, nz = 0.0;
        if (cnt >= 3) {
            double m[3] = {0.0, 0.0, 0.0};
            for (int s = 0; s < cnt; ++s) {
                const int j = sel_at(sel, s);
                for (int a = 0; a < 3; ++a) m[a] += xyz[3 * j + a];
            }
            const double inv = 1.0 / (double)cnt;
            for (int a = 0; a < 3; ++a) m[a] *= inv;
            double cxx = 0.0, cxy = 0.0, cxz = 0.0, cyy = 0.0, cyz = 0.0, czz = 0.0;
            for (int s = 0; s < cnt; ++s) {
                const int j = sel_at(sel, s);
                const double dx = xyz[3 * j + 0] - m[0], dy = xyz[3 * j + 1] - m[1], dz = xyz[3 * j + 2] - m[2];
                cxx += dx * dx; cxy += dx * dy; cxz += dx * dz;
                cyy += dy * dy; cyz += dy * dz; czz += dz * dz;
            }
            if (lane == 0) {
                const double A[3][3] = {{cxx * inv, cxy * inv, cxz * inv},
                                        {cxy * inv, cyy * inv, cyz * inv},
                                        {cxz * inv, cyz * inv, czz * inv}};
                double U[3][3], S[3], V[3][3];
                svd3_jacobi(A, U, S, V);
                const double len = sqrt(V[0][2] * V[0][2] + V[1][2] * V[1][2] + V[2][2] * V[2][2]);
                nx = V[0][2] / len; ny = V[1][2] / len; nz = V[2][2] / len;
                const double d = __dadd_rn(__dadd_rn(__dmul_rn(nx, qx), __dmul_rn(ny, qy)), __dmul_rn(nz, qz));
                if (d > 0.0) { nx = -nx; ny = -ny; nz = -nz; }
            }
        }
        if (lane == 0) {
            normals[3 * qi + 0] = nx; normals[3 * qi + 1] = ny; normals[3 * qi + 2] = nz;
            if (counts) counts[qi] = cnt;
        }
    }
}

struct NrmWs {
    float* x32;
    void *grid, *gws;
    size_t gws_bytes, total;
};

NrmWs carve_normals(void* ws, int n_cap) {
    NrmWs w;
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

extern "C" {

size_t regtr_estimate_normals_ws_bytes(int n_cap) { return carve_normals(nullptr, n_cap > 0 ? n_cap : 1).total; }
size_t regtr_estimate_normals_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap > 0 ? n_cap : 1); }

int regtr_estimate_normals(const double* xyz, const int32_t* offs, int C, int n_cap, double radius, float cell,
                           int max_nn, double* normals, int32_t* counts, uint32_t* status, void* ws, size_t ws_bytes,
                           void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !status || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || !(radius > 0.0) ||
        !((double)cell > radius) || max_nn < 1 || max_nn > NRM_MAX_NN || (n_cap > 0 && (!xyz || !normals)))
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1;      // offs[C] = 0 without points: every kernel then reads no xyz
    NrmWs w = carve_normals(ws, nc);
    if (ws_bytes < w.total || state_bytes < regtr_estimate_normals_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const double bound = regtr_overlap_coord_bound(radius, cell);
    const int T = 256;
    k_normals_init<<<regtr_cdiv(nc, T), T, 0, st>>>(xyz, offs, C, nc, bound, w.x32, status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, C, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes, state,
                                        state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const int blocks = regtr_cdiv(nc, NRM_WARPS) < 4 * REGTR_NUM_SMS ? regtr_cdiv(nc, NRM_WARPS) : 4 * REGTR_NUM_SMS;
    k_normals<<<blocks, NRM_WARPS * 32, 0, st>>>(xyz, offs, C, nc, grid_table(w.grid, (size_t)nc), cell_table_log2(nc),
                                                 grid_sxyzi(w.grid), cell, radius * radius, max_nn, normals, counts);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
