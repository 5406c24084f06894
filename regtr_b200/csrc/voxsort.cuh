// Internal to the library: the sort-based voxel grouping shared by regtr_grid_subsample_sorted (preprocess.cu) and
// regtr_voxel_down_sample (voxel.cu).  Both sort 64-bit keys [cloud:16][x:16][y:16][z:16] with their point indices by
// a stable library radix sort, flag the first position of every voxel, scan the flags into output rows and find each
// cloud's first row by binary search; only the key and the averaging kernels differ.
#pragma once

#include <cub/cub.cuh>

#include "cellgrid.cuh"

namespace {

// flag[j] = 1 where sorted position j starts a new voxel (j < n), else 0; flag[n_cap] = 0.
__global__ void k_head_flags(const unsigned long long* __restrict__ skeys, int n_cap, int32_t* __restrict__ flag) {
    int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j > n_cap) return;
    int f = 0;
    if (j < n_cap) {
        const unsigned long long k = skeys[j];
        f = (k != KEY_PAD) && (j == 0 || skeys[j - 1] != k);
    }
    flag[j] = f;
}

__device__ __forceinline__ int lower_bound_u64(const unsigned long long* __restrict__ a, int lo, int hi,
                                               unsigned long long v) {
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (a[mid] < v) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// out_offs[c] = number of voxels whose key is below cloud c's first key.
__global__ void k_cloud_offsets(const unsigned long long* __restrict__ skeys, const int32_t* __restrict__ rank,
                                int n_cap, int n_clouds, int out_cap, int32_t* __restrict__ out_offs) {
    int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c > n_clouds) return;
    if (c == n_clouds) { out_offs[c] = min(rank[n_cap], out_cap); return; }
    const int pos = lower_bound_u64(skeys, 0, n_cap, (unsigned long long)c << 48);
    out_offs[c] = min(rank[pos], out_cap);      // clamped on overflow (status flag set by the averaging kernel)
}

struct SubWs {
    unsigned long long *keys_in, *keys_out;
    int32_t *vals_in, *vals_out, *rank;
    void* cub_tmp;
    size_t cub_bytes;
    size_t total;
};

size_t cub_tmp_bytes(int n_cap) {
    size_t a = 0, b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, a, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (int32_t*)nullptr, (int32_t*)nullptr, n_cap, 0, 64, (cudaStream_t)0);
    cub::DeviceScan::ExclusiveSum(nullptr, b, (int32_t*)nullptr, (int32_t*)nullptr, n_cap + 1, (cudaStream_t)0);
    return a > b ? a : b;
}

SubWs carve(void* ws, int n_cap) {
    SubWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    w.keys_in = (unsigned long long*)take(sizeof(unsigned long long) * (size_t)n_cap);
    w.keys_out = (unsigned long long*)take(sizeof(unsigned long long) * (size_t)n_cap);
    w.vals_in = (int32_t*)take(sizeof(int32_t) * ((size_t)n_cap + 1));   // also holds the n_cap+1 head flags
    w.vals_out = (int32_t*)take(sizeof(int32_t) * (size_t)n_cap);
    w.rank = (int32_t*)take(sizeof(int32_t) * ((size_t)n_cap + 1));
    w.cub_bytes = cub_tmp_bytes(n_cap);
    w.cub_tmp = take(w.cub_bytes);
    w.total = off;
    return w;
}

int key_bits(int n_clouds) {
    int b = 1;
    while ((1 << b) <= n_clouds) ++b;  // 2^b > n_clouds, so the all-ones pad field sorts last
    return 48 + b;
}

// Sort keys_in / vals_in (n_cap pairs) into keys_out / vals_out, flag the voxel heads and scan them into w.rank
// (rank[j] = output row of the voxel that starts at sorted position j; rank[n_cap] = the number of voxels).
int sort_and_rank(const SubWs& w, int n_cap, int n_clouds, cudaStream_t st) {
    size_t tb = w.cub_bytes;
    cub::DeviceRadixSort::SortPairs(w.cub_tmp, tb, w.keys_in, w.keys_out, w.vals_in, w.vals_out, n_cap, 0,
                                    key_bits(n_clouds), st);
    REGTR_CHECK_LAUNCH();
    k_head_flags<<<regtr_cdiv(n_cap + 1, 256), 256, 0, st>>>(w.keys_out, n_cap, w.vals_in);
    REGTR_CHECK_LAUNCH();
    tb = w.cub_bytes;
    cub::DeviceScan::ExclusiveSum(w.cub_tmp, tb, w.vals_in, w.rank, n_cap + 1, st);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // namespace
