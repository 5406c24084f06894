// Internal to the library: the warp-wide hybrid neighbour selection (the max_nn nearest points of a point's own cloud
// strictly within a radius, ties to the lower index) shared by normal estimation (normals.cu) and FPFH (fpfh.cu).
#pragma once

#include "cellgrid.cuh"

namespace {

// Entry s of a selection lives in lane s % 32, slot s / 32.
template <int SLOTS>
__device__ __forceinline__ int sel_at(const int (&sel)[SLOTS], int s) {
    int v = sel[0];
#pragma unroll
    for (int k = 1; k < SLOTS; ++k)
        if ((s >> 5) == k) v = sel[k];
    return __shfl_sync(0xffffffffu, v, s & 31);
}

// One warp, one query point (qx, qy, qz) of cloud c.  Lanes 0..26 look up one stencil cell each and the candidates are
// flattened 32 wide, as in k_icp_nn.  The neighbours are the candidates with d2 = (dx dx + dy dy) + dz dz (float64, no
// contraction) strictly below r2, the point itself included; the warp extracts the next-smallest (d2, index) key
// max_nn (<= 32 SLOTS) times, so nothing depends on how many candidates lie within the radius.  -> the neighbour
// count; entry s (ascending (d2, index)) is sel_at(sel, s).
template <int SLOTS>
__device__ __forceinline__ int warp_select_neighbours(const double* __restrict__ xyz, const CellSlot* __restrict__ table,
                                                      int log2t, const float4* __restrict__ sxyzi, float cell, int c,
                                                      double qx, double qy, double qz, double r2, int max_nn, int lane,
                                                      int (&sel)[SLOTS]) {
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
    // selection: key s is the smallest (d2, index) above key s - 1; lane s % 32 keeps its index
    double pd = -1.0;
    int pj = -1, cnt = 0;
#pragma unroll
    for (int k = 0; k < SLOTS; ++k) sel[k] = -1;
    for (int s = 0; s < max_nn; ++s) {
        double best = r2;
        int bi = -1;
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
                const double dx = __dsub_rn(qx, xyz[3 * j + 0]), dy = __dsub_rn(qy, xyz[3 * j + 1]),
                             dz = __dsub_rn(qz, xyz[3 * j + 2]);
                const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                const bool above = d2 > pd || (d2 == pd && j > pj);
                if (d2 < r2 && above && (bi < 0 || d2 < best || (d2 == best && j < bi))) { best = d2; bi = j; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
        }
        if (bi < 0) break;                               // warp-uniform: every lane holds the same key
#pragma unroll
        for (int k = 0; k < SLOTS; ++k) sel[k] = lane == (s & 31) && (s >> 5) == k ? bi : sel[k];
        pd = best; pj = bi; cnt = s + 1;
    }
    return cnt;
}

}  // namespace
