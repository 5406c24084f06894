// Shared helpers for the regtr_b200 CUDA kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/regtr_b200.h"

#define REGTR_NUM_SMS 132

#define REGTR_CHECK_LAUNCH()                                         \
    do {                                                             \
        cudaError_t e__ = cudaGetLastError();                        \
        if (e__ != cudaSuccess) return -(1000 + (int)e__);           \
    } while (0)

static inline int regtr_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }
static inline size_t regtr_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// 64-bit spatial key: [cloud:16][x:16][y:16][z:16], coordinates biased by 32768.
__device__ __forceinline__ unsigned long long regtr_pack_key(int cloud, int x, int y, int z) {
    return ((unsigned long long)(unsigned)cloud << 48) | ((unsigned long long)(unsigned)(x + 32768) << 32) |
           ((unsigned long long)(unsigned)(y + 32768) << 16) | (unsigned long long)(unsigned)(z + 32768);
}

// floor(p / cell) with IEEE division -- the pinned voxel rule (DESIGN.md H1-ii).
__device__ __forceinline__ int regtr_cell_of(float p, float cell) { return (int)floorf(__fdiv_rn(p, cell)); }

// Index of the cloud that owns packed row i: largest c with offs[c] <= i.
__device__ __forceinline__ int regtr_cloud_of(const int32_t* __restrict__ offs, int n_clouds, int i) {
    int lo = 0, hi = n_clouds;  // invariant: offs[lo] <= i < offs[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (offs[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// (row, column group) of flat work item t for a row of `w` items: 32-bit arithmetic, a shift when w is a power of two
// (a 64-bit divide costs ~100 issue slots -- more than the rest of an elementwise kernel).  Callers bound the grid
// so that t < 2^31.
__device__ __forceinline__ void regtr_row_col(unsigned t, unsigned w, int& row, int& col) {
    if ((w & (w - 1u)) == 0u) { const int sh = 31 - __clz((int)w); row = (int)(t >> sh); col = (int)(t & (w - 1u)); }
    else { row = (int)(t / w); col = (int)(t - (unsigned)row * w); }
}

// round-to-nearest-even to TF32 precision (10 mantissa bits): the hi half of regtr_split_tf32 (x = hi + lo with
// lo = regtr_tf32_rne(x - hi)); unbiased, so split errors do not accumulate linearly along K as truncation does
__device__ __forceinline__ float regtr_tf32_rne(float x) {
    uint32_t u = __float_as_uint(x);
    u += 0x0FFFu + ((u >> 13) & 1u);
    return __uint_as_float(u & 0xFFFFE000u);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
