// Internal to the library: exact k-nearest-neighbour search over a cell list (Open3D's SearchKNN restated with this
// library's rules), used by the statistical outlier filter (outlier.cu).
//
// The neighbours of a query q of cloud c are the k points of c with the smallest (d2, index) keys, q itself included,
// d2 = (dx dx + dy dy) + dz dz in float64 with every operation rounded on its own; all of c's points when it has fewer
// than k.  There is no radius.  The result is defined by that rule alone: the search below provably finds those keys,
// so neither the cell size nor the other clouds of the call change a bit of it.
//
// One warp per query.  The warp holds the keys found so far as a sorted list, entry s in lane s % 32, slot s / 32
// (k <= 64: two slots).  It visits the cells of the query's cloud in rings of growing Chebyshev radius r around the
// query's cell, and stops after ring r when the list is full and its k-th d2 lies strictly below the squared lower
// bound on the distance of any point outside the searched (2r+1)^3 box, or when it has seen every point of the cloud.
// After KNN_MAX_RING rings without stopping it sweeps the whole cloud instead, which bounds the work on sparse or
// clustered geometry.
#pragma once

#include "cellgrid.cuh"

namespace {

constexpr int KNN_MAX_K = 64;
constexpr int KNN_SLOTS = KNN_MAX_K / 32;
constexpr int KNN_MAX_RING = 4;
constexpr int KNN_NO_INDEX = 0x7fffffff;

// The cells of rings 0..KNN_MAX_RING as packed offsets (dx + 8) | (dy + 8) << 4 | (dz + 8) << 8, ring by ring; ring r
// starts at entry (2r - 1)^3 (0 for r = 0) and ends at (2r + 1)^3.
constexpr int KNN_RING_CELLS = (2 * KNN_MAX_RING + 1) * (2 * KNN_MAX_RING + 1) * (2 * KNN_MAX_RING + 1);
struct KnnRingTable {
    unsigned short off[KNN_RING_CELLS];
};
constexpr KnnRingTable knn_ring_table() {
    KnnRingTable t{};
    int n = 0;
    for (int r = 0; r <= KNN_MAX_RING; ++r)
        for (int x = -r; x <= r; ++x)
            for (int y = -r; y <= r; ++y)
                for (int z = -r; z <= r; ++z)
                    if (x == -r || x == r || y == -r || y == r || z == -r || z == r)
                        t.off[n++] = (unsigned short)((x + 8) | (y + 8) << 4 | (z + 8) << 8);
    return t;
}
__device__ const KnnRingTable g_knn_rings = knn_ring_table();

__device__ __forceinline__ bool knn_less(double da, int ja, double db, int jb) {
    return da < db || (da == db && ja < jb);
}

__device__ __forceinline__ double knn_d2(const double* __restrict__ xyz, int j, double qx, double qy, double qz) {
    const double dx = __dsub_rn(qx, xyz[3 * (size_t)j + 0]), dy = __dsub_rn(qy, xyz[3 * (size_t)j + 1]),
                 dz = __dsub_rn(qz, xyz[3 * (size_t)j + 2]);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Entry s of the warp's list (every lane gets it).  Every slot is shuffled and the result selected, so that the list
// stays in registers (a selection among the slots before the shuffle compiles to an indexed local-memory load).
__device__ __forceinline__ void knn_at(const double (&ld)[KNN_SLOTS], const int (&lj)[KNN_SLOTS], int s, double& d,
                                       int& j) {
#pragma unroll
    for (int t = 0; t < KNN_SLOTS; ++t) {
        const double v = __shfl_sync(0xffffffffu, ld[t], s & 31);
        const int w = __shfl_sync(0xffffffffu, lj[t], s & 31);
        if (t == 0 || (s >> 5) == t) { d = v; j = w; }
    }
}

__device__ __forceinline__ void knn_clear(double (&ld)[KNN_SLOTS], int (&lj)[KNN_SLOTS], double& kd, int& kj) {
#pragma unroll
    for (int t = 0; t < KNN_SLOTS; ++t) { ld[t] = INFINITY; lj[t] = KNN_NO_INDEX; }
    kd = INFINITY; kj = KNN_NO_INDEX;
}

// Merge the lanes' candidates (has: lane holds one) into the sorted list of the k smallest keys, one at a time in lane
// order; (kd, kj) is the list's k-th key, (inf, KNN_NO_INDEX) while it holds fewer than k.  Warp-uniform control.
__device__ __forceinline__ void knn_merge(double (&ld)[KNN_SLOTS], int (&lj)[KNN_SLOTS], int k, double& kd, int& kj,
                                          double d2, int j, bool has, int lane) {
    unsigned m = __ballot_sync(0xffffffffu, has && knn_less(d2, j, kd, kj));
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const double cd = __shfl_sync(0xffffffffu, d2, src);
        const int cj = __shfl_sync(0xffffffffu, j, src);
        if (!knn_less(cd, cj, kd, kj)) continue;         // an earlier insertion lowered the k-th key
        int pos = 0;
#pragma unroll
        for (int t = 0; t < KNN_SLOTS; ++t) pos += __popc(__ballot_sync(0xffffffffu, knn_less(ld[t], lj[t], cd, cj)));
        double prev_d = 0.0;
        int prev_j = 0;
#pragma unroll
        for (int t = 0; t < KNN_SLOTS; ++t) {
            // entry s - 1 of the old list for entry s = 32 t + lane
            double ud = __shfl_up_sync(0xffffffffu, ld[t], 1);
            int uj = __shfl_up_sync(0xffffffffu, lj[t], 1);
            const double wd = __shfl_sync(0xffffffffu, ld[t], 31);
            const int wj = __shfl_sync(0xffffffffu, lj[t], 31);
            if (lane == 0) { ud = prev_d; uj = prev_j; }
            prev_d = wd; prev_j = wj;
            const int s = 32 * t + lane;
            if (s >= k) { ld[t] = INFINITY; lj[t] = KNN_NO_INDEX; }
            else if (s == pos) { ld[t] = cd; lj[t] = cj; }
            else if (s > pos) { ld[t] = ud; lj[t] = uj; }
        }
        knn_at(ld, lj, k - 1, kd, kj);
    }
}

// Candidates j of the 32 cells held by the lanes ((start, count) in the cell-ordered sxyzi), flattened 32 at a time
// as in warp_select_neighbours (neighbours.cuh).  -> the number of candidates.
__device__ __forceinline__ int knn_merge_cells(const double* __restrict__ xyz, const float4* __restrict__ sxyzi,
                                               int c_start, int c_cnt, double qx, double qy, double qz,
                                               double (&ld)[KNN_SLOTS], int (&lj)[KNN_SLOTS], int k, double& kd,
                                               int& kj, int lane) {
    int pre = c_cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, pre, o);
        if (lane >= o) pre += v;
    }
    const int total = __shfl_sync(0xffffffffu, pre, 31);
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
        double d2 = 0.0;
        int j = 0;
        if (t < total) {
            j = __float_as_int(sxyzi[cell_start + (t - (cell_pre - cell_cnt))].w);
            d2 = knn_d2(xyz, j, qx, qy, qz);
        }
        knn_merge(ld, lj, k, kd, kj, d2, j, t < total, lane);
    }
    return total;
}

// The k nearest neighbours of (qx, qy, qz) among points a..b-1 (cloud c) into the warp's list, ascending (d2, index).
// -> min(k, b - a), the number of entries.  The cell list holds the fp32 copies of the points with cells
// floor(fp32(p) / cell) (regtr_cellgrid_build), every cell index inside +-32766.
__device__ __forceinline__ int knn_warp(const double* __restrict__ xyz, const CellSlot* __restrict__ table, int log2t,
                                        const float4* __restrict__ sxyzi, float cell, int c, int a, int b, double qx,
                                        double qy, double qz, int k, int lane, double (&ld)[KNN_SLOTS],
                                        int (&lj)[KNN_SLOTS]) {
    double kd;
    int kj;
    knn_clear(ld, lj, kd, kj);
    const int n_c = b - a;
    const int cx = regtr_cell_of((float)qx, cell), cy = regtr_cell_of((float)qy, cell),
              cz = regtr_cell_of((float)qz, cell);
    // A point p lands in cell floor(t), t = fp32(fp32(p) / cell), |t - p / cell| <= (2u + u^2) |p| / cell.  A point
    // outside the box of rings 0..r lies in a cell below c - r or above c + r on some axis (c, t the query's), so on
    // that axis |q - p| (1 + 2u + u^2) > (r + w) cell - (4u + 2u^2) |q|, w = min(t - c, c + 1 - t) the query's margin
    // inside its own cell: `edge`, `slack` and `shrink` below, with room for the rounding of the bound and of d2.
    const double u = 5.9604644775390625e-08;
    const double mq = fmax(fabs(qx), fmax(fabs(qy), fabs(qz)));
    const double slack = (4.0 * u + 2.0 * u * u) * mq + 1e-40, shrink = 1.0 / (1.0 + 2.0 * u + u * u);
    double edge = 1.0;
    {
        const float t[3] = {__fdiv_rn((float)qx, cell), __fdiv_rn((float)qy, cell), __fdiv_rn((float)qz, cell)};
        const int cq[3] = {cx, cy, cz};
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const double f = (double)t[d] - (double)cq[d];               // exact: t and its floor are floats
            edge = fmin(edge, fmin(f, 1.0 - f));
        }
        edge = fmax(edge, 0.0);
    }
    int seen = 0;
    bool done = false;
    for (int r = 0; r <= KNN_MAX_RING && !done; ++r) {
        const int lo = r == 0 ? 0 : (2 * r - 1) * (2 * r - 1) * (2 * r - 1), hi = (2 * r + 1) * (2 * r + 1) * (2 * r + 1);
        for (int base = lo; base < hi; base += 32) {
            const int t = base + lane;
            int c_start = 0, c_cnt = 0;
            if (t < hi) {
                const int o = g_knn_rings.off[t];
                const int x = cx + (o & 15) - 8, y = cy + ((o >> 4) & 15) - 8, z = cz + (o >> 8) - 8;
                if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767)
                    cell_lookup(table, log2t, regtr_pack_key(c, x, y, z), c_start, c_cnt);
            }
            seen += knn_merge_cells(xyz, sxyzi, c_start, c_cnt, qx, qy, qz, ld, lj, k, kd, kj, lane);
        }
        if (seen >= n_c) {
            done = true;
        } else {
            const double lb = __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)r, edge), (double)cell), slack), shrink);
            if (lb > 0.0 && kd < __dmul_rn(__dmul_rn(lb, lb), 1.0 - 1e-12)) done = true;
        }
    }
    if (!done) {                                         // bounded fallback: every point of the cloud
        knn_clear(ld, lj, kd, kj);
        for (int base = a; base < b; base += 32) {
            const int j = base + lane;
            const double d2 = j < b ? knn_d2(xyz, j, qx, qy, qz) : 0.0;
            knn_merge(ld, lj, k, kd, kj, d2, j, j < b, lane);
        }
    }
    return min(k, n_c);
}

}  // namespace
