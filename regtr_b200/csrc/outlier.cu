// Outlier removal for C stacked clouds: Open3D's PointCloud::RemoveStatisticalOutliers over the exact k-nearest-
// neighbour search of knn.cuh, RemoveRadiusOutliers over the library's radius rule, and the stable compaction that
// both share (regtr_select_points).  The contracts, and the summation order of the per-cloud statistics, are in
// include/regtr_b200.h.  No value atomics and no host synchronisation: a cloud's results are the same bits alone or
// in a stack, and the launch count depends on neither the data nor C.
#include "knn.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int OUT_WARPS = 8;
constexpr int STAT_CHUNK = 256;         // points per partial sum of the per-cloud statistics (a fixed tree each)
constexpr double KNN_COORD_MAX = 1e30;  // the cell list holds fp32 copies

// The fp32 copy of the clouds for their cell list, and the range check: |coordinate| beyond `bound`, or not finite,
// raises REGTR_STATUS_RANGE.
__global__ void k_outlier_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
                               double bound, float* __restrict__ x32, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    x32[3 * i + 0] = (float)x; x32[3 * i + 1] = (float)y; x32[3 * i + 2] = (float)z;
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One warp per point: its k nearest neighbours (knn_warp), then avg = (sum of sqrt(d2) in ascending key order) / m.
__global__ void __launch_bounds__(OUT_WARPS * 32)
k_knn_avg(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
          const CellSlot* __restrict__ table, int log2t, const float4* __restrict__ sxyzi, float cell, int k,
          double* __restrict__ avg) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[C];
    for (int qi = blockIdx.x * OUT_WARPS + warp; qi < n_cap && qi < n; qi += gridDim.x * OUT_WARPS) {
        const int c = regtr_cloud_of(offs, C, qi);
        double ld[KNN_SLOTS];
        int lj[KNN_SLOTS];
        const int m = knn_warp(xyz, table, log2t, sxyzi, cell, c, offs[c], offs[c + 1], xyz[3 * qi + 0],
                               xyz[3 * qi + 1], xyz[3 * qi + 2], k, lane, ld, lj);
        double s = 0.0;
        for (int e = 0; e < m; ++e) {
            double d;
            int j;
            knn_at(ld, lj, e, d, j);
            s = __dadd_rn(s, __dsqrt_rn(d));
        }
        if (lane == 0) avg[qi] = __ddiv_rn(s, (double)m);
    }
}

// coffs[c] = the first chunk of cloud c: sum over c' < c of ceil(n_c' / STAT_CHUNK).  One CTA.
__global__ void __launch_bounds__(1024)
k_chunk_offsets(const int32_t* __restrict__ offs, int C, int32_t* __restrict__ coffs) {
    __shared__ int s_sum[1024];
    int carry = 0;
    for (int base = 0; base < C; base += 1024) {
        const int c = base + threadIdx.x;
        const int v = c < C ? (offs[c + 1] - offs[c] + STAT_CHUNK - 1) / STAT_CHUNK : 0;
        s_sum[threadIdx.x] = v;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            const int t = threadIdx.x >= o ? s_sum[threadIdx.x - o] : 0;
            __syncthreads();
            s_sum[threadIdx.x] += t;
            __syncthreads();
        }
        if (c < C) coffs[c + 1] = carry + s_sum[threadIdx.x];
        carry += s_sum[1023];
        __syncthreads();
    }
    if (threadIdx.x == 0) coffs[0] = 0;
}

// One warp per chunk g of STAT_CHUNK points of one cloud, anchored at the cloud's first point: part[g] = the sum of
// f(avg) over the chunk by the fixed tree e[i] += e[i + h], h = 128, 64, ..., 1, past-the-end entries 0.
// PASS 0: f = avg where avg > 0, else 0.  PASS 1: f = (avg - mean)^2 where avg > 0, else 0 (mean = stats[3c]).
template <int PASS>
__global__ void __launch_bounds__(OUT_WARPS * 32)
k_chunk_sum(const double* __restrict__ avg, const int32_t* __restrict__ offs, int C, const int32_t* __restrict__ coffs,
            int g_cap, const double* __restrict__ stats, double* __restrict__ part) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int G = coffs[C];
    for (int g = blockIdx.x * OUT_WARPS + warp; g < g_cap && g < G; g += gridDim.x * OUT_WARPS) {
        const int c = regtr_cloud_of(coffs, C, g);
        const int a = offs[c] + (g - coffs[c]) * STAT_CHUNK, b = offs[c + 1];
        const double mean = PASS == 1 ? stats[3 * c] : 0.0;
        double e[STAT_CHUNK / 32];
#pragma unroll
        for (int m = 0; m < STAT_CHUNK / 32; ++m) {
            const int i = a + 32 * m + lane;
            const double v = i < b ? avg[i] : 0.0;
            if (PASS == 0) e[m] = v > 0.0 ? v : 0.0;
            else e[m] = v > 0.0 ? __dmul_rn(__dsub_rn(v, mean), __dsub_rn(v, mean)) : 0.0;
        }
#pragma unroll
        for (int h = STAT_CHUNK / 64; h > 0; h >>= 1) {
#pragma unroll
            for (int m = 0; m < h; ++m) e[m] = __dadd_rn(e[m], e[m + h]);
        }
        double s = e[0];
#pragma unroll
        for (int h = 16; h > 0; h >>= 1) s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, h));
        if (lane == 0) part[g] = s;
    }
}

// One thread per cloud: its chunk partials added in ascending chunk order.  PASS 0: stats[3c] = cloud_mean = sum /
// n_c.  PASS 1: std_dev = sqrt(sq_sum / (n_c - 1)) and threshold = cloud_mean + std_ratio * std_dev.
template <int PASS>
__global__ void k_cloud_stats(const int32_t* __restrict__ offs, int C, const int32_t* __restrict__ coffs,
                              const double* __restrict__ part, double std_ratio, double* __restrict__ stats) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    double s = 0.0;
    for (int g = coffs[c]; g < coffs[c + 1]; ++g) s = __dadd_rn(s, part[g]);
    const double valid = (double)(offs[c + 1] - offs[c]);
    if (PASS == 0) {
        stats[3 * c] = __ddiv_rn(s, valid);
    } else {
        const double sd = __dsqrt_rn(__ddiv_rn(s, __dsub_rn(valid, 1.0)));
        stats[3 * c + 1] = sd;
        stats[3 * c + 2] = __dadd_rn(stats[3 * c], __dmul_rn(std_ratio, sd));
    }
}

// keep[i] = avg > 0 and avg < threshold of its cloud.
__global__ void k_stat_keep(const double* __restrict__ avg, const int32_t* __restrict__ offs, int C, int n_cap,
                            const double* __restrict__ stats, int32_t* __restrict__ keep) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double v = avg[i], thr = stats[3 * regtr_cloud_of(offs, C, i) + 2];
    keep[i] = v > 0.0 && v < thr ? 1 : 0;
}

// One warp per point: the points of its own cloud with d2 strictly below r2, itself included, over the 27 cells around
// it (lanes 0..26 look one up each, candidates flattened 32 wide as in warp_select_neighbours).  The full count.
__global__ void __launch_bounds__(OUT_WARPS * 32)
k_radius_count(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
               const CellSlot* __restrict__ table, int log2t, const float4* __restrict__ sxyzi, float cell, double r2,
               int nb_points, int32_t* __restrict__ counts, int32_t* __restrict__ keep) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[C];
    for (int qi = blockIdx.x * OUT_WARPS + warp; qi < n_cap && qi < n; qi += gridDim.x * OUT_WARPS) {
        const int c = regtr_cloud_of(offs, C, qi);
        const double qx = xyz[3 * qi + 0], qy = xyz[3 * qi + 1], qz = xyz[3 * qi + 2];
        const int cx = regtr_cell_of((float)qx, cell), cy = regtr_cell_of((float)qy, cell),
                  cz = regtr_cell_of((float)qz, cell);
        int c_start = 0, c_cnt = 0;
        if (lane < 27) {
            const int x = cx + lane / 9 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane % 3 - 1;
            if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767)
                cell_lookup(table, log2t, regtr_pack_key(c, x, y, z), c_start, c_cnt);
        }
        int pre = c_cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
        }
        const int total = __shfl_sync(0xffffffffu, pre, 31);
        int cnt = 0;
        for (int base = 0; base < total; base += 32) {
            const int t = base + lane;
            int cellid = 0;
#pragma unroll
            for (int step = 16; step > 0; step >>= 1) {
                const int pv = __shfl_sync(0xffffffffu, pre, cellid + step - 1);
                if (pv <= t) cellid += step;
            }
            const int cell_pre = __shfl_sync(0xffffffffu, pre, cellid);
            const int cell_cnt = __shfl_sync(0xffffffffu, c_cnt, cellid);
            const int cell_start = __shfl_sync(0xffffffffu, c_start, cellid);
            if (t < total) {
                const int j = __float_as_int(sxyzi[cell_start + (t - (cell_pre - cell_cnt))].w);
                if (knn_d2(xyz, j, qx, qy, qz) < r2) ++cnt;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0) {
            counts[qi] = cnt;
            keep[qi] = cnt >= nb_points ? 1 : 0;
        }
    }
}

// flag[i] = 1 where point i < offs[C] is kept, 0 elsewhere (n_cap + 1 entries: the scan's last one is the total).
__global__ void k_select_flags(const int32_t* __restrict__ keep, const int32_t* __restrict__ offs, int C, int n_cap,
                               int32_t* __restrict__ flag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_cap) return;
    flag[i] = i < n_cap && i < offs[C] && keep[i] != 0 ? 1 : 0;
}

// Kept point i goes to row pre[i], with its attribute row and its index inside its cloud; out_offs[c] = pre[offs[c]].
__global__ void k_select_scatter(const double* __restrict__ xyz, const double* __restrict__ attr,
                                 const int32_t* __restrict__ flag, const int32_t* __restrict__ pre,
                                 const int32_t* __restrict__ offs, int C, int n_cap, double* __restrict__ out_xyz,
                                 double* __restrict__ out_attr, int32_t* __restrict__ out_index,
                                 int32_t* __restrict__ out_offs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= C) out_offs[i] = pre[offs[i]];
    if (i >= n_cap || !flag[i]) return;
    const size_t r = (size_t)pre[i];
#pragma unroll
    for (int d = 0; d < 3; ++d) out_xyz[3 * r + d] = xyz[3 * (size_t)i + d];
    if (attr) {
#pragma unroll
        for (int d = 0; d < 3; ++d) out_attr[3 * r + d] = attr[3 * (size_t)i + d];
    }
    if (out_index) out_index[r] = i - offs[regtr_cloud_of(offs, C, i)];
}

struct OutWs {
    float* x32;
    void *grid, *gws;
    int32_t* coffs;
    double* part;
    size_t gws_bytes, total;
};

// chunks of the statistics: at most one partial per STAT_CHUNK points plus one per cloud
int chunk_cap(int n_cap, int C) { return regtr_cdiv(n_cap, STAT_CHUNK) + C; }

OutWs carve_outlier(void* ws, int n_cap, int C) {
    OutWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    w.x32 = (float*)take(sizeof(float) * 3 * (size_t)n_cap);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.coffs = (int32_t*)take(sizeof(int32_t) * ((size_t)C + 1));
    w.part = (double*)take(sizeof(double) * (size_t)chunk_cap(n_cap, C));
    w.total = off;
    return w;
}

int warp_blocks(int n) {
    const int b = regtr_cdiv(n, OUT_WARPS);
    return b < 4 * REGTR_NUM_SMS ? b : 4 * REGTR_NUM_SMS;
}

}  // namespace

extern "C" {

size_t regtr_outlier_ws_bytes(int n_cap, int C) {
    return carve_outlier(nullptr, n_cap > 0 ? n_cap : 1, C > 0 ? C : 1).total;
}
size_t regtr_outlier_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap > 0 ? n_cap : 1); }

int regtr_statistical_outlier(const double* xyz, const int32_t* offs, int C, int n_cap, int nb_neighbors,
                              double std_ratio, float cell, double* avg, int32_t* keep, double* stats,
                              uint32_t* status, void* ws, size_t ws_bytes, void* state, size_t state_bytes,
                              void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !stats || !status || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || nb_neighbors < 1 ||
        nb_neighbors > KNN_MAX_K || !(std_ratio > 0.0) || !isfinite(std_ratio) || !(cell > 0.f) || !isfinite(cell) ||
        (n_cap > 0 && (!xyz || !avg || !keep)))
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1;      // offs[C] = 0 without points: every kernel then reads no xyz
    OutWs w = carve_outlier(ws, nc, C);
    if (ws_bytes < w.total || state_bytes < regtr_outlier_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const int T = 256, G = chunk_cap(nc, C);
    k_outlier_init<<<regtr_cdiv(nc, T), T, 0, st>>>(xyz, offs, C, nc, KNN_COORD_MAX, w.x32, status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, C, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes, state,
                                        state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    k_knn_avg<<<warp_blocks(nc), OUT_WARPS * 32, 0, st>>>(xyz, offs, C, nc, grid_table(w.grid, (size_t)nc),
                                                          cell_table_log2(nc), grid_sxyzi(w.grid), cell, nb_neighbors,
                                                          avg);
    REGTR_CHECK_LAUNCH();
    k_chunk_offsets<<<1, 1024, 0, st>>>(offs, C, w.coffs);
    REGTR_CHECK_LAUNCH();
    k_chunk_sum<0><<<warp_blocks(G), OUT_WARPS * 32, 0, st>>>(avg, offs, C, w.coffs, G, stats, w.part);
    REGTR_CHECK_LAUNCH();
    k_cloud_stats<0><<<regtr_cdiv(C, 128), 128, 0, st>>>(offs, C, w.coffs, w.part, std_ratio, stats);
    REGTR_CHECK_LAUNCH();
    k_chunk_sum<1><<<warp_blocks(G), OUT_WARPS * 32, 0, st>>>(avg, offs, C, w.coffs, G, stats, w.part);
    REGTR_CHECK_LAUNCH();
    k_cloud_stats<1><<<regtr_cdiv(C, 128), 128, 0, st>>>(offs, C, w.coffs, w.part, std_ratio, stats);
    REGTR_CHECK_LAUNCH();
    k_stat_keep<<<regtr_cdiv(nc, T), T, 0, st>>>(avg, offs, C, nc, stats, keep);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_radius_outlier(const double* xyz, const int32_t* offs, int C, int n_cap, int nb_points, double radius,
                         float cell, int32_t* counts, int32_t* keep, uint32_t* status, void* ws, size_t ws_bytes,
                         void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !status || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || nb_points < 1 || !(radius > 0.0) ||
        !isfinite(radius) || !((double)cell > radius) || !isfinite(cell) || (n_cap > 0 && (!xyz || !counts || !keep)))
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1;
    OutWs w = carve_outlier(ws, nc, C);
    if (ws_bytes < w.total || state_bytes < regtr_outlier_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const int T = 256;
    k_outlier_init<<<regtr_cdiv(nc, T), T, 0, st>>>(xyz, offs, C, nc, regtr_overlap_coord_bound(radius, cell), w.x32,
                                                    status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, C, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes, state,
                                        state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    k_radius_count<<<warp_blocks(nc), OUT_WARPS * 32, 0, st>>>(xyz, offs, C, nc, grid_table(w.grid, (size_t)nc),
                                                               cell_table_log2(nc), grid_sxyzi(w.grid), cell,
                                                               radius * radius, nb_points, counts, keep);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_select_points_ws_bytes(int n_cap) { return 2 * regtr_align(sizeof(int32_t) * ((size_t)n_cap + 1)); }
size_t regtr_select_points_state_bytes(int n_cap) { return scan_state_bytes((long long)n_cap + 1); }

int regtr_select_points(const double* xyz, const double* attr, const int32_t* keep, const int32_t* offs, int C,
                        int n_cap, double* out_xyz, double* out_attr, int32_t* out_index, int32_t* out_offs, void* ws,
                        size_t ws_bytes, void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !out_offs || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || (attr && !out_attr) ||
        (n_cap > 0 && (!xyz || !keep || !out_xyz)))
        return REGTR_ERR_ARG;
    if (ws_bytes < regtr_select_points_ws_bytes(n_cap) || state_bytes < regtr_select_points_state_bytes(n_cap))
        return REGTR_ERR_WORKSPACE;
    int32_t* flag = (int32_t*)ws;
    int32_t* pre = (int32_t*)((char*)ws + regtr_align(sizeof(int32_t) * ((size_t)n_cap + 1)));
    const int T = 256;
    k_select_flags<<<regtr_cdiv(n_cap + 1, T), T, 0, st>>>(keep, offs, C, n_cap, flag);
    REGTR_CHECK_LAUNCH();
    const int rc = launch_scan<0>(flag, pre, n_cap + 1, nullptr, state, st);
    if (rc != REGTR_OK) return rc;
    k_select_scatter<<<regtr_cdiv((n_cap > C ? n_cap : C) + 1, T), T, 0, st>>>(xyz, attr, flag, pre, offs, C, n_cap,
                                                                              out_xyz, out_attr, out_index, out_offs);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
