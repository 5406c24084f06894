// FPFH features and their nearest-neighbour matching: Open3D's ComputeFPFHFeature(KDTreeSearchParamHybrid(radius,
// max_nn)) for C stacked clouds, and the feature-space correspondences of registration_ransac_based_on_feature_matching
// (forward nearest target, reverse nearest source, the mutual filter and its fallback) for B pairs, restated with this
// library's tie and order rules (DESIGN.md section 8, "FPFH and feature matching").  Float64 throughout, no value
// atomics, no host synchronisation, launch counts fixed by the arguments.
#include "neighbours.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int FD = REGTR_FPFH_DIM;                 // 33 = 3 x 11 bins
constexpr int FP_WARPS = 8;
constexpr int FP_THREADS = 128;                    // per-thread passes (SPFH, FPFH)
constexpr int FP_SLOTS = REGTR_FPFH_MAX_NN / 32;   // four selected indices per lane

__device__ __forceinline__ double dot3(const double* a, const double* b) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
    c[0] = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
    c[1] = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
    c[2] = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
}

// Open3D's ComputePairFeatures(p1, n1, p2, n2) -> (f0, f1, f2), every product and sum rounded on its own.  The swap
// test |a1| < |a2| is Open3D's acos(|a1|) > acos(|a2|) without the acos.  false: the zero feature (|d| = 0 or |v| = 0).
__device__ __forceinline__ bool pair_feature(const double* p1, const double* n1, const double* p2, const double* n2,
                                             double& f0, double& f1, double& f2) {
    double d[3] = {__dsub_rn(p2[0], p1[0]), __dsub_rn(p2[1], p1[1]), __dsub_rn(p2[2], p1[2])};
    const double dn = sqrt(dot3(d, d));
    if (dn == 0.0) return false;
    const double a1 = dot3(n1, d) / dn, a2 = dot3(n2, d) / dn;
    const bool sw = fabs(a1) < fabs(a2);
    double m1[3], m2[3];
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        m1[e] = sw ? n2[e] : n1[e];
        m2[e] = sw ? n1[e] : n2[e];
        d[e] = sw ? -d[e] : d[e];
    }
    f2 = sw ? -a2 : a1;
    double v[3], w[3];
    cross3(d, m1, v);
    const double vn = sqrt(dot3(v, v));
    if (vn == 0.0) return false;
    v[0] = v[0] / vn; v[1] = v[1] / vn; v[2] = v[2] / vn;
    cross3(m1, v, w);
    f1 = dot3(v, m2);
    f0 = atan2(dot3(w, m2), dot3(m1, m2));
    return true;
}

__device__ __forceinline__ int fpfh_bin(double x) {          // floor(x), clamped to 0..10
    const double f = floor(x);
    return f < 0.0 ? 0 : (f >= 11.0 ? 10 : (int)f);
}

// The fp32 copy of the clouds for their cell list, and the range check (as k_normals_init).
__global__ void k_fpfh_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
                            double bound, float* __restrict__ x32, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    x32[3 * i + 0] = (float)x; x32[3 * i + 1] = (float)y; x32[3 * i + 2] = (float)z;
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One warp per point: the neighbour list of warp_select_neighbours, stored as (index, d2) entries in ascending
// (d2, index) order, max_nn slots per point, and the count.
__global__ void __launch_bounds__(FP_WARPS * 32, 1)
k_fpfh_select(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
              const CellSlot* __restrict__ table, int log2t, const float4* __restrict__ sxyzi, float cell, double r2,
              int max_nn, int32_t* __restrict__ nidx, double* __restrict__ nd2, int32_t* __restrict__ ncnt,
              int32_t* __restrict__ counts) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[C];
    for (int qi = blockIdx.x * FP_WARPS + warp; qi < n_cap && qi < n; qi += gridDim.x * FP_WARPS) {
        const int c = regtr_cloud_of(offs, C, qi);
        const double qx = xyz[3 * qi + 0], qy = xyz[3 * qi + 1], qz = xyz[3 * qi + 2];
        int sel[FP_SLOTS];
        const int cnt = warp_select_neighbours(xyz, table, log2t, sxyzi, cell, c, qx, qy, qz, r2, max_nn, lane, sel);
#pragma unroll
        for (int k = 0; k < FP_SLOTS; ++k) {
            const int s = 32 * k + lane;
            if (s < cnt) {
                const int j = sel[k];
                const double dx = __dsub_rn(qx, xyz[3 * j + 0]), dy = __dsub_rn(qy, xyz[3 * j + 1]),
                             dz = __dsub_rn(qz, xyz[3 * j + 2]);
                nidx[(size_t)qi * max_nn + s] = j;
                nd2[(size_t)qi * max_nn + s] = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)),
                                                         __dmul_rn(dz, dz));
            }
        }
        if (lane == 0) {
            ncnt[qi] = cnt;
            if (counts) counts[qi] = cnt;
        }
    }
}

// One thread per point: its SPFH (Open3D's ComputeSPFHFeature).  Entries k >= 1 of a list of count >= 2 add
// 100 / (count - 1) to the three bins of their pair feature, in entry order; fewer than 2 neighbours: zeros.
__global__ void __launch_bounds__(FP_THREADS)
k_fpfh_spfh(const double* __restrict__ xyz, const double* __restrict__ normals, const int32_t* __restrict__ offs,
            int C, int n_cap, int max_nn, const int32_t* __restrict__ nidx, const int32_t* __restrict__ ncnt,
            double* __restrict__ spfh) {
    __shared__ double hist[FD * FP_THREADS];
    const int i = blockIdx.x * FP_THREADS + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    double* h = hist + threadIdx.x;
    for (int b = 0; b < FD; ++b) h[b * FP_THREADS] = 0.0;
    const int cnt = ncnt[i];
    if (cnt > 1) {
        const double inc = 100.0 / (double)(cnt - 1);
        const double p1[3] = {xyz[3 * i + 0], xyz[3 * i + 1], xyz[3 * i + 2]};
        const double n1[3] = {normals[3 * i + 0], normals[3 * i + 1], normals[3 * i + 2]};
        const double two_pi = 2.0 * M_PI;
        for (int k = 1; k < cnt; ++k) {
            const int j = nidx[(size_t)i * max_nn + k];
            const double p2[3] = {xyz[3 * j + 0], xyz[3 * j + 1], xyz[3 * j + 2]};
            const double n2[3] = {normals[3 * j + 0], normals[3 * j + 1], normals[3 * j + 2]};
            double f0 = 0.0, f1 = 0.0, f2 = 0.0;
            if (!pair_feature(p1, n1, p2, n2, f0, f1, f2)) { f0 = 0.0; f1 = 0.0; f2 = 0.0; }
            const int b0 = fpfh_bin(__dmul_rn(11.0, __dadd_rn(f0, M_PI)) / two_pi);
            const int b1 = 11 + fpfh_bin(__dmul_rn(__dmul_rn(11.0, __dadd_rn(f1, 1.0)), 0.5));
            const int b2 = 22 + fpfh_bin(__dmul_rn(__dmul_rn(11.0, __dadd_rn(f2, 1.0)), 0.5));
            h[b0 * FP_THREADS] = __dadd_rn(h[b0 * FP_THREADS], inc);
            h[b1 * FP_THREADS] = __dadd_rn(h[b1 * FP_THREADS], inc);
            h[b2 * FP_THREADS] = __dadd_rn(h[b2 * FP_THREADS], inc);
        }
    }
    for (int b = 0; b < FD; ++b) spfh[(size_t)i * FD + b] = h[b * FP_THREADS];
}

// One thread per point: its FPFH (Open3D's ComputeFPFHFeature).  Entries k >= 1 with d2 != 0, in entry order, add
// val = spfh[j][b] / d2 to feature[b] and to sum[b / 11]; then each third is scaled by 100 / sum (sum != 0) and the
// point's own SPFH is added.  Fewer than 2 neighbours: zeros.
__global__ void __launch_bounds__(FP_THREADS)
k_fpfh_feature(const int32_t* __restrict__ offs, int C, int n_cap, int max_nn, const int32_t* __restrict__ nidx,
               const double* __restrict__ nd2, const int32_t* __restrict__ ncnt, const double* __restrict__ spfh,
               double* __restrict__ feature) {
    const int i = blockIdx.x * FP_THREADS + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const int cnt = ncnt[i];
    double f[FD];
#pragma unroll
    for (int b = 0; b < FD; ++b) f[b] = 0.0;
    if (cnt > 1) {
        double sum[3] = {0.0, 0.0, 0.0};
        for (int k = 1; k < cnt; ++k) {
            const double d2 = nd2[(size_t)i * max_nn + k];
            if (d2 == 0.0) continue;
            const double* sj = spfh + (size_t)nidx[(size_t)i * max_nn + k] * FD;
#pragma unroll
            for (int b = 0; b < FD; ++b) {
                const double val = sj[b] / d2;
                sum[b / 11] = __dadd_rn(sum[b / 11], val);
                f[b] = __dadd_rn(f[b], val);
            }
        }
#pragma unroll
        for (int t = 0; t < 3; ++t)
            if (sum[t] != 0.0) sum[t] = 100.0 / sum[t];
        const double* si = spfh + (size_t)i * FD;
#pragma unroll
        for (int b = 0; b < FD; ++b) f[b] = __dadd_rn(__dmul_rn(f[b], sum[b / 11]), si[b]);
    }
#pragma unroll
    for (int b = 0; b < FD; ++b) feature[(size_t)i * FD + b] = f[b];
}

struct FpfhWs {
    float* x32;
    void *grid, *gws;
    int32_t *nidx, *ncnt;
    double *nd2, *spfh;
    size_t gws_bytes, total;
};

FpfhWs carve_fpfh(void* ws, int n_cap, int max_nn) {
    FpfhWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    w.x32 = (float*)take(sizeof(float) * 3 * (size_t)n_cap);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.nidx = (int32_t*)take(sizeof(int32_t) * (size_t)n_cap * max_nn);
    w.nd2 = (double*)take(sizeof(double) * (size_t)n_cap * max_nn);
    w.ncnt = (int32_t*)take(sizeof(int32_t) * (size_t)n_cap);
    w.spfh = (double*)take(sizeof(double) * (size_t)n_cap * FD);
    w.total = off;
    return w;
}

// ------------------------------------------------------------------------------------------------ feature matching

constexpr int FM_ROWS = 256;                 // source rows per CTA, one per thread, held in registers
constexpr int FM_WARPS = FM_ROWS / 32;
constexpr int FM_TN = 32;                    // target columns per shared-memory tile
constexpr int FM_CS = 512;                   // target columns per CTA
constexpr int FM_LD = 34;                    // tile row pitch in doubles (16-byte aligned pairs)
constexpr int FM_ILP = 4;                    // columns in flight per thread

__host__ __device__ inline int fm_chunks(int nt_max) { return (nt_max + FM_CS - 1) / FM_CS; }
__host__ __device__ inline int fm_row_blocks(int ns_max) { return (ns_max + FM_ROWS - 1) / FM_ROWS; }

// One CTA per (pair b, block of FM_ROWS source rows, chunk of FM_CS target columns): d2(i, j) = sum over k = 0..32 of
// (a_k - b_k)^2, accumulated in that order without contraction.  Per source row, the lowest (d2, j) of the chunk goes
// to the forward partials [b][chunk][i]; per target column, the lowest (d2, i) of the row block to the reverse partials
// [b][row block][j].  The second launch reduces both in ascending order, so the result does not depend on the tiling.
__global__ void __launch_bounds__(FM_ROWS, 2)
k_fm_sweep(const double* __restrict__ fs, const int32_t* __restrict__ soffs, const double* __restrict__ ft,
           const int32_t* __restrict__ toffs, int ns_max, int nt_max, double* __restrict__ fwd_d2,
           int32_t* __restrict__ fwd_j, double* __restrict__ rev_d2, int32_t* __restrict__ rev_i) {
    __shared__ __align__(16) double tile[FM_TN * FM_LD];
    __shared__ unsigned long long wkey[FM_WARPS][FM_TN];
    __shared__ int wrow[FM_WARPS][FM_TN];
    const int b = blockIdx.y, nch = fm_chunks(nt_max), nrb = fm_row_blocks(ns_max);
    const int rb = blockIdx.x / nch, ch = blockIdx.x - rb * nch;
    const int s0 = soffs[b], t0 = toffs[b];
    const int ns = min(soffs[b + 1] - s0, ns_max), nt = min(toffs[b + 1] - t0, nt_max);
    const int r0 = rb * FM_ROWS, c0 = ch * FM_CS;
    if (r0 >= ns || c0 >= nt) return;                                      // CTA-uniform
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int i = r0 + tid;
    const bool live = i < ns;
    double a[FD];
#pragma unroll
    for (int k = 0; k < FD; ++k) a[k] = live ? fs[(size_t)(s0 + i) * FD + k] : 0.0;
    double fbest = 0.0;
    int fj = -1;
    const int c1 = min(c0 + FM_CS, nt);
    for (int tc = c0; tc < c1; tc += FM_TN) {
        const int w = min(FM_TN, c1 - tc);
        __syncthreads();                                                   // the previous tile is consumed
        for (int e = tid; e < FM_TN * FD; e += FM_ROWS) {
            const int col = e / FD, k = e - col * FD;
            tile[col * FM_LD + k] = col < w ? ft[(size_t)(t0 + tc + col) * FD + k] : 0.0;
        }
        __syncthreads();
        for (int cc = 0; cc < w; cc += FM_ILP) {
            double acc[FM_ILP];
#pragma unroll
            for (int u = 0; u < FM_ILP; ++u) acc[u] = 0.0;
#pragma unroll
            for (int k = 0; k < FD; ++k) {
#pragma unroll
                for (int u = 0; u < FM_ILP; ++u) {
                    const double t = __dsub_rn(a[k], tile[(cc + u) * FM_LD + k]);
                    acc[u] = __dadd_rn(acc[u], __dmul_rn(t, t));
                }
            }
#pragma unroll
            for (int u = 0; u < FM_ILP; ++u) {
                const int col = cc + u;
                if (col >= w) break;                                       // CTA-uniform
                if (live && (fj < 0 || acc[u] < fbest)) { fbest = acc[u]; fj = tc + col; }
                // the warp's lowest (d2, row): d2 >= 0, so its bit pattern orders as its value
                const unsigned long long key = live ? (unsigned long long)__double_as_longlong(acc[u]) : ~0ull;
                const unsigned hi = __reduce_min_sync(0xffffffffu, (unsigned)(key >> 32));
                const unsigned lo = __reduce_min_sync(0xffffffffu, (unsigned)(key >> 32) == hi ? (unsigned)key : ~0u);
                const unsigned long long kmin = ((unsigned long long)hi << 32) | lo;
                const unsigned at = __ballot_sync(0xffffffffu, key == kmin);
                if (lane == 0) { wkey[warp][col] = kmin; wrow[warp][col] = r0 + warp * 32 + __ffs(at) - 1; }
            }
        }
        __syncthreads();
        if (tid < w) {                           // the warps in row order: only a strictly lower key moves the row up
            unsigned long long bk = wkey[0][tid];
            int bi = wrow[0][tid];
#pragma unroll
            for (int v = 1; v < FM_WARPS; ++v)
                if (wkey[v][tid] < bk) { bk = wkey[v][tid]; bi = wrow[v][tid]; }
            const size_t o = ((size_t)b * nrb + rb) * nt_max + tc + tid;
            rev_d2[o] = __longlong_as_double((long long)bk);
            rev_i[o] = bi;
        }
    }
    if (live) {
        const size_t o = ((size_t)b * nch + ch) * ns_max + i;
        fwd_d2[o] = fbest;
        fwd_j[o] = fj;
    }
}

// Thread x of pair b: the nearest target of source x (chunks in ascending order) with its coordinates, and the nearest
// source of target x (row blocks in ascending order); ties stay with the lower index.
__global__ void k_fm_reduce(const double* __restrict__ tgt_xyz, const int32_t* __restrict__ soffs,
                            const int32_t* __restrict__ toffs, int ns_max, int nt_max,
                            const double* __restrict__ fwd_d2, const int32_t* __restrict__ fwd_j,
                            const double* __restrict__ rev_d2, const int32_t* __restrict__ rev_i,
                            int32_t* __restrict__ nn_st, int32_t* __restrict__ nn_ts, double* __restrict__ corr_tgt) {
    const int b = blockIdx.y, x = blockIdx.x * blockDim.x + threadIdx.x;
    const int nch = fm_chunks(nt_max), nrb = fm_row_blocks(ns_max);
    const int s0 = soffs[b], t0 = toffs[b];
    const int ns = min(soffs[b + 1] - s0, ns_max), nt = min(toffs[b + 1] - t0, nt_max);
    if (x < ns) {
        double bd = 0.0;
        int bj = -1;
        for (int ch = 0; ch < fm_chunks(nt); ++ch) {
            const size_t o = ((size_t)b * nch + ch) * ns_max + x;
            const double d = fwd_d2[o];
            if (bj < 0 || d < bd) { bd = d; bj = fwd_j[o]; }
        }
        nn_st[s0 + x] = bj;
        for (int e = 0; e < 3; ++e) corr_tgt[3 * (s0 + x) + e] = bj >= 0 ? tgt_xyz[3 * (t0 + bj) + e] : 0.0;
    }
    if (x < nt) {
        double bd = 0.0;
        int bi = -1;
        for (int rb = 0; rb < fm_row_blocks(ns); ++rb) {
            const size_t o = ((size_t)b * nrb + rb) * nt_max + x;
            const double d = rev_d2[o];
            if (bi < 0 || d < bd) { bd = d; bi = rev_i[o]; }
        }
        nn_ts[t0 + x] = bi;
    }
}

// One CTA per pair: the mutual count (nn_ts[nn_st[i]] == i), then the mask: the mutual matches, or every match without
// the mutual filter or when fewer than min_mutual are mutual (Open3D's fallback).
__global__ void __launch_bounds__(256)
k_fm_finalize(const int32_t* __restrict__ soffs, const int32_t* __restrict__ toffs, int ns_max,
              const int32_t* __restrict__ nn_st, const int32_t* __restrict__ nn_ts, int mutual_filter, int min_mutual,
              uint8_t* __restrict__ mask, int32_t* __restrict__ n_mutual) {
    __shared__ int part[8];
    const int b = blockIdx.x, s0 = soffs[b], t0 = toffs[b], ns = min(soffs[b + 1] - s0, ns_max);
    int cnt = 0;
    for (int i = threadIdx.x; i < ns; i += blockDim.x) {
        const int j = nn_st[s0 + i];
        cnt += j >= 0 && nn_ts[t0 + j] == i;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = cnt;
    __syncthreads();
    int total = 0;
    for (int v = 0; v < 8; ++v) total += part[v];
    const bool all = !mutual_filter || total < min_mutual;
    for (int i = threadIdx.x; i < ns; i += blockDim.x) {
        const int j = nn_st[s0 + i];
        mask[s0 + i] = all ? (j >= 0) : (j >= 0 && nn_ts[t0 + j] == i);
    }
    if (threadIdx.x == 0) n_mutual[b] = total;
}

struct FmWs {
    double *fwd_d2, *rev_d2;
    int32_t *fwd_j, *rev_i, *nn_ts;
    size_t total;
};

FmWs carve_fm(void* ws, int B, int ns_max, int nt_max, int nt_cap) {
    FmWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t nf = (size_t)B * fm_chunks(nt_max) * ns_max, nr = (size_t)B * fm_row_blocks(ns_max) * nt_max;
    w.fwd_d2 = (double*)take(sizeof(double) * nf);
    w.fwd_j = (int32_t*)take(sizeof(int32_t) * nf);
    w.rev_d2 = (double*)take(sizeof(double) * nr);
    w.rev_i = (int32_t*)take(sizeof(int32_t) * nr);
    w.nn_ts = (int32_t*)take(sizeof(int32_t) * (size_t)(nt_cap > 0 ? nt_cap : 1));
    w.total = off;
    return w;
}

}  // namespace

extern "C" {

size_t regtr_fpfh_ws_bytes(int n_cap, int max_nn) {
    return carve_fpfh(nullptr, n_cap > 0 ? n_cap : 1, max_nn > 0 ? max_nn : 1).total;
}
size_t regtr_fpfh_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap > 0 ? n_cap : 1); }

int regtr_fpfh(const double* xyz, const double* normals, const int32_t* offs, int C, int n_cap, double radius,
               float cell, int max_nn, double* feature, int32_t* counts, uint32_t* status, void* ws, size_t ws_bytes,
               void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !status || !ws || !state || C <= 0 || C > 32767 || n_cap < 0 || !(radius > 0.0) ||
        !((double)cell > radius) || max_nn < 1 || max_nn > REGTR_FPFH_MAX_NN ||
        (n_cap > 0 && (!xyz || !normals || !feature)))
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1;      // offs[C] = 0 without points: every kernel then reads no xyz
    FpfhWs w = carve_fpfh(ws, nc, max_nn);
    if (ws_bytes < w.total || state_bytes < regtr_fpfh_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const double bound = regtr_overlap_coord_bound(radius, cell);
    k_fpfh_init<<<regtr_cdiv(nc, 256), 256, 0, st>>>(xyz, offs, C, nc, bound, w.x32, status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, C, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes, state,
                                        state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const int blocks = regtr_cdiv(nc, FP_WARPS) < 4 * REGTR_NUM_SMS ? regtr_cdiv(nc, FP_WARPS) : 4 * REGTR_NUM_SMS;
    k_fpfh_select<<<blocks, FP_WARPS * 32, 0, st>>>(xyz, offs, C, nc, grid_table(w.grid, (size_t)nc),
                                                    cell_table_log2(nc), grid_sxyzi(w.grid), cell, radius * radius,
                                                    max_nn, w.nidx, w.nd2, w.ncnt, counts);
    REGTR_CHECK_LAUNCH();
    k_fpfh_spfh<<<regtr_cdiv(nc, FP_THREADS), FP_THREADS, 0, st>>>(xyz, normals, offs, C, nc, max_nn, w.nidx, w.ncnt,
                                                                   w.spfh);
    REGTR_CHECK_LAUNCH();
    k_fpfh_feature<<<regtr_cdiv(nc, FP_THREADS), FP_THREADS, 0, st>>>(offs, C, nc, max_nn, w.nidx, w.nd2, w.ncnt,
                                                                      w.spfh, feature);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_feature_match_ws_bytes(int B, int ns_max, int nt_max, int nt_cap) {
    return carve_fm(nullptr, B > 0 ? B : 1, ns_max > 0 ? ns_max : 1, nt_max > 0 ? nt_max : 1, nt_cap).total;
}

int regtr_feature_match(const double* src_feat, const int32_t* soffs, const double* tgt_feat, const double* tgt_xyz,
                        const int32_t* toffs, int B, int ns_max, int nt_max, int nt_cap, int mutual_filter,
                        int min_mutual, int32_t* nn, double* corr_tgt, uint8_t* mask, int32_t* n_mutual, void* ws,
                        size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!soffs || !toffs || !n_mutual || !ws || B <= 0 || B > 65535 || ns_max < 0 || nt_max < 0 ||
        nt_cap < nt_max || (ns_max > 0 && (!src_feat || !nn || !corr_tgt || !mask)) ||
        (nt_max > 0 && (!tgt_feat || !tgt_xyz)))
        return REGTR_ERR_ARG;
    const int nsm = ns_max > 0 ? ns_max : 1, ntm = nt_max > 0 ? nt_max : 1;
    FmWs w = carve_fm(ws, B, nsm, ntm, nt_cap);
    if (ws_bytes < w.total) return REGTR_ERR_WORKSPACE;
    k_fm_sweep<<<dim3(fm_row_blocks(nsm) * fm_chunks(ntm), B), FM_ROWS, 0, st>>>(
        src_feat, soffs, tgt_feat, toffs, nsm, ntm, w.fwd_d2, w.fwd_j, w.rev_d2, w.rev_i);
    REGTR_CHECK_LAUNCH();
    k_fm_reduce<<<dim3(regtr_cdiv(nsm > ntm ? nsm : ntm, 256), B), 256, 0, st>>>(
        tgt_xyz, soffs, toffs, nsm, ntm, w.fwd_d2, w.fwd_j, w.rev_d2, w.rev_i, nn, w.nn_ts, corr_tgt);
    REGTR_CHECK_LAUNCH();
    k_fm_finalize<<<B, 256, 0, st>>>(soffs, toffs, nsm, nn, w.nn_ts, mutual_filter, min_mutual, mask, n_mutual);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
