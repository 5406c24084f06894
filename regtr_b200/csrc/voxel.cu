// Float64 voxel down-sampling with attributes (Open3D's PointCloud::VoxelDownSample): one output row per occupied
// voxel of a grid anchored at each cloud's bounding-box minimum, the mean of its member points and of their
// attributes.  The multi-scale ICP pyramid (eval.icp_refine with voxels=) down-samples every level with it.
//
// The grouping is regtr_grid_subsample_sorted's (voxsort.cuh): stable radix sort of [cloud][vx][vy][vz] keys with
// the point indices, head flags, their scan into output rows.  What differs from that fp32 KPConv path: float64
// input, the grid origin at lo - V / 2 per cloud (lo the exact per-axis minimum), unsigned 16-bit voxel indices,
// float64 means and the optional attribute array.  No value atomics: reruns, and a cloud alone or in a stack, give
// the same bits.
#include "voxsort.cuh"

namespace {

constexpr int MIN_THREADS = 512;

// lo[3c + d] = the minimum of axis d over cloud c (+inf for an empty cloud).  One CTA per cloud; a minimum is exact,
// so the reduction order does not matter.
__global__ void __launch_bounds__(MIN_THREADS)
k_cloud_min(const double* __restrict__ xyz, const int32_t* __restrict__ offs, double* __restrict__ lo) {
    __shared__ double s_min[3][MIN_THREADS / 32];
    const int c = blockIdx.x;
    const int a = offs[c], b = offs[c + 1];
    double m[3] = {INFINITY, INFINITY, INFINITY};
    for (int i = a + threadIdx.x; i < b; i += MIN_THREADS) {
#pragma unroll
        for (int d = 0; d < 3; ++d) m[d] = fmin(m[d], xyz[3 * (size_t)i + d]);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        double v = m[d];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (lane == 0) s_min[d][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < 3) {
        double v = INFINITY;
        for (int w = 0; w < MIN_THREADS / 32; ++w) v = fmin(v, s_min[threadIdx.x][w]);
        lo[3 * c + threadIdx.x] = v;
    }
}

// key[i] = [cloud][vx][vy][vz] with v = floor((p - (lo - V/2)) / V) per axis, each operation rounded on its own
// (no contraction), for i < offs[C]; KEY_PAD beyond.  val[i] = i.  An index outside 0..65535 or a non-finite
// coordinate raises REGTR_STATUS_KEY_RANGE and is clamped into the range (the output is then not meaningful).
__global__ void k_voxel_keys(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int n_clouds, int n_cap,
                             double voxel, const double* __restrict__ lo, unsigned long long* __restrict__ keys,
                             int32_t* __restrict__ vals, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap) return;
    unsigned long long key = KEY_PAD;
    if (i < offs[n_clouds]) {
        const int c = regtr_cloud_of(offs, n_clouds, i);
        const double half = __dmul_rn(0.5, voxel);
        bool bad = false;
        unsigned v[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const double p = xyz[3 * (size_t)i + d];
            const double t = floor(__ddiv_rn(__dsub_rn(p, __dsub_rn(lo[3 * c + d], half)), voxel));
            if (!(t >= 0.0 && t <= 65535.0) || !isfinite(p)) bad = true;
            v[d] = t >= 0.0 ? (t <= 65535.0 ? (unsigned)t : 65535u) : 0u;   // NaN -> 0
        }
        if (bad) atomicOr(status, REGTR_STATUS_KEY_RANGE);
        key = ((unsigned long long)(unsigned)c << 48) | ((unsigned long long)v[0] << 32) |
              ((unsigned long long)v[1] << 16) | (unsigned long long)v[2];
    }
    keys[i] = key;
    vals[i] = i;
}

// One thread per voxel head: float64 running sums over the members in ascending point index (the radix sort is
// stable), each divided by the count.
__global__ void k_voxel_mean64(const double* __restrict__ xyz, const double* __restrict__ attr,
                               const unsigned long long* __restrict__ skeys, const int32_t* __restrict__ sidx,
                               const int32_t* __restrict__ rank, int n_cap, double* __restrict__ out_xyz,
                               double* __restrict__ out_attr) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_cap) return;
    const unsigned long long k = skeys[j];
    if (k == KEY_PAD || (j > 0 && skeys[j - 1] == k)) return;
    double s[3] = {0.0, 0.0, 0.0}, a[3] = {0.0, 0.0, 0.0};
    int cnt = 0;
    for (int t = j; t < n_cap && skeys[t] == k; ++t) {
        const size_t i = (size_t)sidx[t];
#pragma unroll
        for (int d = 0; d < 3; ++d) s[d] = __dadd_rn(s[d], xyz[3 * i + d]);
        if (attr) {
#pragma unroll
            for (int d = 0; d < 3; ++d) a[d] = __dadd_rn(a[d], attr[3 * i + d]);
        }
        ++cnt;
    }
    const double c = (double)cnt;
    const size_t m = (size_t)rank[j];
#pragma unroll
    for (int d = 0; d < 3; ++d) out_xyz[3 * m + d] = __ddiv_rn(s[d], c);
    if (attr) {
#pragma unroll
        for (int d = 0; d < 3; ++d) out_attr[3 * m + d] = __ddiv_rn(a[d], c);
    }
}

size_t lo_offset(int n_cap) { return carve(nullptr, n_cap).total; }

}  // namespace

extern "C" {

size_t regtr_voxel_down_sample_ws_bytes(int n_cap, int C) {
    if (n_cap <= 0) return 256;
    return lo_offset(n_cap) + regtr_align(sizeof(double) * 3 * (size_t)(C > 0 ? C : 1));
}

int regtr_voxel_down_sample(const double* xyz, const double* attr, const int32_t* offs, int C, int n_cap,
                            double voxel, double* out_xyz, double* out_attr, int32_t* out_offs, uint32_t* status,
                            void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !out_offs || !status || C <= 0 || C > 32767 || n_cap < 0 || !(voxel > 0.0) || !isfinite(voxel) ||
        (attr && !out_attr))
        return REGTR_ERR_ARG;
    if (n_cap == 0) {
        cudaMemsetAsync(out_offs, 0, sizeof(int32_t) * (C + 1), st);
        return REGTR_OK;
    }
    if (!xyz || !out_xyz || !ws) return REGTR_ERR_ARG;
    if (ws_bytes < regtr_voxel_down_sample_ws_bytes(n_cap, C)) return REGTR_ERR_WORKSPACE;
    const SubWs w = carve(ws, n_cap);
    double* lo = (double*)((char*)ws + lo_offset(n_cap));
    const int T = 256;
    k_cloud_min<<<C, MIN_THREADS, 0, st>>>(xyz, offs, lo);
    REGTR_CHECK_LAUNCH();
    k_voxel_keys<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, C, n_cap, voxel, lo, w.keys_in, w.vals_in, status);
    REGTR_CHECK_LAUNCH();
    const int rc = sort_and_rank(w, n_cap, C, st);
    if (rc != REGTR_OK) return rc;
    k_voxel_mean64<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, attr, w.keys_out, w.vals_out, w.rank, n_cap, out_xyz,
                                                       out_attr);
    REGTR_CHECK_LAUNCH();
    k_cloud_offsets<<<regtr_cdiv(C + 1, 128), 128, 0, st>>>(w.keys_out, w.rank, n_cap, C, n_cap, out_offs);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
