// Training-data preparation for 3DMatch pairs: overlap ground truth and the reference's four augmentations.
//
// Reference behaviour replaced (paths relative to /root/reference/src):
//   utils/pointcloud.py:8-65            compute_overlap (Open3D radius search, nearest first, mutual correspondences)
//   data_loaders/threedmatch.py:79-86   the overlap of the ALIGNED clouds, computed before any augmentation
//   data_loaders/transforms.py:15-149   RigidPerturb -> Jitter -> ShufflePoints -> RandomSwap
// Parity rules: DESIGN.md section 8, "Training data".
//
// Stacked clouds as in the forward: src_0..src_{B-1}, tgt_0..tgt_{B-1} with int32 device offsets; every launch covers
// the whole batch, and nothing synchronises with the host.
#include "cellgrid.cuh"
#include "philox.cuh"
#include "rigid.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);

namespace {

constexpr int NN_WARPS = 8;

// ------------------------------------------------------------------------------------------------- overlap
// Source clouds moved by the ground-truth pose in float64 (the reference's se3_transform(pose, src_xyz) on the
// float64 arrays), targets copied; an fp32 copy of both for the cell list; |coordinate| beyond `bound` raises
// REGTR_STATUS_RANGE (the cell list's rounding could then hide a neighbour from the 27-cell stencil).
__global__ void k_align(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, int n_cap,
                        const double* __restrict__ pose, double bound, double* __restrict__ xa,
                        float* __restrict__ x32, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[2 * B]) return;
    const int c = regtr_cloud_of(offs, 2 * B, i);
    double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (c < B) {
        const double* m = pose + 12 * c;
        const double ax = rt_row(m, x, y, z), ay = rt_row(m + 4, x, y, z), az = rt_row(m + 8, x, y, z);
        x = ax; y = ay; z = az;
    }
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
    xa[3 * i + 0] = x; xa[3 * i + 1] = y; xa[3 * i + 2] = z;
    x32[3 * i + 0] = (float)x; x32[3 * i + 1] = (float)y; x32[3 * i + 2] = (float)z;
}

// Every point of cloud c moved by pose c in float64 (rt_row, as k_align), rounded once to fp32.
__global__ void k_transform_clouds(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int C, int n_cap,
                                   const double* __restrict__ pose, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_cap || i >= offs[C]) return;
    const double* m = pose + 12 * regtr_cloud_of(offs, C, i);
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    out[3 * i + 0] = (float)rt_row(m, x, y, z);
    out[3 * i + 1] = (float)rt_row(m + 4, x, y, z);
    out[3 * i + 2] = (float)rt_row(m + 8, x, y, z);
}

// One warp per query, in the cell-sorted order of the stacked set: lanes 0..26 look up one stencil cell each in the
// PARTNER cloud (src_b <-> tgt_b), candidates are flattened 32 wide, the squared distance is evaluated in float64 on
// the aligned coordinates ((dx dx + dy dy) + dz dz, no contraction); the nearest support with d2 < r2 wins, equal
// distances go to the lowest index.  nn[i] = that support's index inside its cloud, or -1.
__global__ void __launch_bounds__(NN_WARPS * 32)
k_overlap_nn(const double* __restrict__ xa, const float* __restrict__ x32, const int32_t* __restrict__ offs, int B,
             int n_cap, const int32_t* __restrict__ order, const CellSlot* __restrict__ table, int log2t,
             const float4* __restrict__ sxyzi, float cell, double r2, int32_t* __restrict__ nn) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n = offs[2 * B];
    for (int slot = blockIdx.x * NN_WARPS + warp; slot < n_cap; slot += gridDim.x * NN_WARPS) {
        const int qi = order[slot];
        if (qi < 0 || qi >= n) continue;
        const int c = regtr_cloud_of(offs, 2 * B, qi);
        const int pc = c < B ? c + B : c - B;
        const int cx = regtr_cell_of(x32[3 * qi + 0], cell), cy = regtr_cell_of(x32[3 * qi + 1], cell),
                  cz = regtr_cell_of(x32[3 * qi + 2], cell);
        const double qx = xa[3 * qi + 0], qy = xa[3 * qi + 1], qz = xa[3 * qi + 2];
        int c_start = 0, c_cnt = 0;
        if (lane < 27) {
            const int x = cx + lane / 9 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane % 3 - 1;
            if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767)
                cell_lookup(table, log2t, regtr_pack_key(pc, x, y, z), c_start, c_cnt);
        }
        int pre = c_cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
        }
        const int total = __shfl_sync(0xffffffffu, pre, 31);
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
                const double dx = __dsub_rn(qx, xa[3 * j + 0]), dy = __dsub_rn(qy, xa[3 * j + 1]),
                             dz = __dsub_rn(qz, xa[3 * j + 2]);
                const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                if (d2 < best || (d2 == best && bi >= 0 && j < bi)) { best = d2; bi = j; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) nn[qi] = bi >= 0 ? bi - offs[pc] : -1;
    }
}

// ------------------------------------------------------------------------------------------------- registration fit
// One CTA per (pair, direction): cloud c < B is source b = c (queries moved by pose b, partners the raw target),
// c >= B is target b = c - B (partners the moved source).  Per inlier the squared distance is k_overlap_nn's
// ((dx dx + dy dy) + dz dz) on k_align's moved source (rt_row), so it is the value that passed "< r2".  Each thread
// sums its strided points in ascending order, then a fixed shared-memory tree: deterministic, no atomics on values.
// A match outside the partner cloud or not strictly within the radius is not counted and raises
// REGTR_STATUS_INPUT (nn then did not come from regtr_overlap_nn on these inputs).
constexpr int FIT_THREADS = 256;

__global__ void __launch_bounds__(FIT_THREADS)
k_registration_fit(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                   const double* __restrict__ pose, double r2, const int32_t* __restrict__ nn,
                   double* __restrict__ out, uint32_t* status) {
    __shared__ double s_sum[FIT_THREADS];
    __shared__ int s_cnt[FIT_THREADS];
    const int c = blockIdx.x, t = threadIdx.x;
    const int b = c < B ? c : c - B, pc = c < B ? c + B : c - B;
    const double* m = pose + 12 * b;
    const int a0 = offs[c], a1 = offs[c + 1], p0 = offs[pc], np_ = offs[pc + 1] - p0;
    double sum = 0.0;
    int cnt = 0;
    bool bad = false;
    for (int i = a0 + t; i < a1; i += FIT_THREADS) {
        const int j = nn[i];
        if (j < 0) continue;
        if (j >= np_) { bad = true; continue; }
        const double* s = xyz + 3 * (size_t)(c < B ? i : p0 + j);     // the source end of the match
        const double* q = xyz + 3 * (size_t)(c < B ? p0 + j : i);     // the target end
        const double sx = s[0], sy = s[1], sz = s[2];
        const double dx = __dsub_rn(rt_row(m, sx, sy, sz), q[0]), dy = __dsub_rn(rt_row(m + 4, sx, sy, sz), q[1]),
                     dz = __dsub_rn(rt_row(m + 8, sx, sy, sz), q[2]);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (!(d2 < r2)) { bad = true; continue; }
        sum = __dadd_rn(sum, d2);
        ++cnt;
    }
    if (bad) atomicOr(status, REGTR_STATUS_INPUT);
    s_sum[t] = sum;
    s_cnt[t] = cnt;
    __syncthreads();
    for (int h = FIT_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) { s_sum[t] = __dadd_rn(s_sum[t], s_sum[t + h]); s_cnt[t] += s_cnt[t + h]; }
        __syncthreads();
    }
    if (t != 0) return;
    const int n = a1 - a0, k = s_cnt[0];
    double* o = out + 4 * b + (c < B ? 0 : 2);
    o[0] = n > 0 ? __ddiv_rn((double)k, (double)n) : 0.0;
    o[1] = k > 0 ? __dsqrt_rn(__ddiv_rn(s_sum[0], (double)k)) : 0.0;
}

// ------------------------------------------------------------------------------------------------- information
// One CTA per pair: Lambda = sum G^T G over the source points with a match, q the matched target point.  The 21 unique
// entries of G^T G are ten distinct sums (y^2 + z^2, x^2 + z^2, x^2 + y^2, xy, xz, yz, x, y, z, count); each thread
// sums its strided points in ascending order, then a fixed shared-memory tree, as in k_registration_fit.  A match
// outside the target or not strictly within the radius of the moved source point is skipped and raises
// REGTR_STATUS_INPUT.
constexpr int INFO_SUMS = 10;

__global__ void __launch_bounds__(FIT_THREADS)
k_registration_information(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                           const double* __restrict__ pose, double r2, const int32_t* __restrict__ nn,
                           double* __restrict__ out, uint32_t* status) {
    __shared__ double s_sum[INFO_SUMS][FIT_THREADS];
    const int b = blockIdx.x, t = threadIdx.x;
    const double* m = pose + 12 * b;
    const int a0 = offs[b], a1 = offs[b + 1], p0 = offs[B + b], np_ = offs[B + b + 1] - p0;
    double acc[INFO_SUMS];
#pragma unroll
    for (int k = 0; k < INFO_SUMS; ++k) acc[k] = 0.0;
    bool bad = false;
    for (int i = a0 + t; i < a1; i += FIT_THREADS) {
        const int j = nn[i];
        if (j < 0) continue;
        if (j >= np_) { bad = true; continue; }
        const double* s = xyz + 3 * (size_t)i;
        const double* q = xyz + 3 * (size_t)(p0 + j);
        const double x = q[0], y = q[1], z = q[2];
        const double dx = __dsub_rn(rt_row(m, s[0], s[1], s[2]), x), dy = __dsub_rn(rt_row(m + 4, s[0], s[1], s[2]), y),
                     dz = __dsub_rn(rt_row(m + 8, s[0], s[1], s[2]), z);
        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
        if (!(d2 < r2)) { bad = true; continue; }
        const double xx = __dmul_rn(x, x), yy = __dmul_rn(y, y), zz = __dmul_rn(z, z);
        acc[0] = __dadd_rn(acc[0], __dadd_rn(zz, yy));
        acc[1] = __dadd_rn(acc[1], __dadd_rn(zz, xx));
        acc[2] = __dadd_rn(acc[2], __dadd_rn(yy, xx));
        acc[3] = __dadd_rn(acc[3], __dmul_rn(x, y));
        acc[4] = __dadd_rn(acc[4], __dmul_rn(x, z));
        acc[5] = __dadd_rn(acc[5], __dmul_rn(y, z));
        acc[6] = __dadd_rn(acc[6], x);
        acc[7] = __dadd_rn(acc[7], y);
        acc[8] = __dadd_rn(acc[8], z);
        acc[9] = __dadd_rn(acc[9], 1.0);
    }
    if (bad) atomicOr(status, REGTR_STATUS_INPUT);
#pragma unroll
    for (int k = 0; k < INFO_SUMS; ++k) s_sum[k][t] = acc[k];
    __syncthreads();
    for (int h = FIT_THREADS / 2; h > 0; h >>= 1) {
        if (t < h)
#pragma unroll
            for (int k = 0; k < INFO_SUMS; ++k) s_sum[k][t] = __dadd_rn(s_sum[k][t], s_sum[k][t + h]);
        __syncthreads();
    }
    if (t >= 36) return;
    // G^T G: rows 0-2 the rotation block [[y2+z2, -xy, -xz], [-xy, x2+z2, -yz], [-xz, -yz, x2+y2]], the coupling
    // [[0, -z, y], [z, 0, -x], [-y, x, 0]] and its transpose, the count on the translation diagonal
    const int r = t / 6, c = t % 6, lo = r < c ? r : c, hi = r < c ? c : r;
    double v = 0.0;
    if (hi < 3) {
        const int idx[3][3] = {{0, 3, 4}, {3, 1, 5}, {4, 5, 2}};
        v = s_sum[idx[lo][hi]][0];
        if (lo != hi) v = -v;
    } else if (lo < 3) {
        const int a = lo, k = hi - 3;                // coupling entry (a, 3 + k)
        if (a != k) {
            v = s_sum[6 + (3 - a - k)][0];           // the sum of the remaining axis' coordinate
            if ((a + 1) % 3 == k) v = -v;            // (0,1): -z, (1,2): -x, (2,0): -y; the other order positive
        }
    } else if (lo == hi) {
        v = s_sum[9][0];
    }
    out[36 * (size_t)b + t] = v;
}

// ------------------------------------------------------------------------------------------------- augmentation
// One CTA per pair.  pert[b] = (R | t) of the host-drawn perturbation; flags: REGTR_PREP_*.  With CENTRE ('small'),
// the rotation turns about the centroid c of the perturbed cloud (float64 mean in a fixed order): t' = (t + c) - R c.
// Source perturbed: pose' = pose P^-1, else pose' = P pose; swapped: pose'' = pose'^-1.  mat[cloud] receives the
// transform of every input cloud (identity for the unperturbed one); out_pose the final pose in fp32.
__global__ void __launch_bounds__(256)
k_prep_pose(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, const double* __restrict__ pose,
            const double* __restrict__ pert, const int32_t* __restrict__ flags, double* __restrict__ mat,
            float* __restrict__ out_pose) {
    __shared__ double s_sum[3][256];
    const int b = blockIdx.x, t = threadIdx.x;
    const int f = flags[b];
    const int pc = (f & REGTR_PREP_PERTURB_SRC) ? b : B + b;
    double c[3] = {0.0, 0.0, 0.0};
    if (f & REGTR_PREP_CENTRE) {
        const int a0 = offs[pc], a1 = offs[pc + 1];
        double sx = 0.0, sy = 0.0, sz = 0.0;
        for (int i = a0 + t; i < a1; i += 256) {
            sx = __dadd_rn(sx, xyz[3 * i + 0]); sy = __dadd_rn(sy, xyz[3 * i + 1]); sz = __dadd_rn(sz, xyz[3 * i + 2]);
        }
        s_sum[0][t] = sx; s_sum[1][t] = sy; s_sum[2][t] = sz;
        __syncthreads();
        for (int h = 128; h > 0; h >>= 1) {
            if (t < h)
                for (int a = 0; a < 3; ++a) s_sum[a][t] = __dadd_rn(s_sum[a][t], s_sum[a][t + h]);
            __syncthreads();
        }
        if (a1 > a0)
            for (int a = 0; a < 3; ++a) c[a] = __ddiv_rn(s_sum[a][0], (double)(a1 - a0));
    }
    if (t != 0) return;
    double P[12], Q[12], O[12];
    for (int k = 0; k < 12; ++k) P[k] = pert[12 * b + k];
    if (f & REGTR_PREP_CENTRE)
        for (int a = 0; a < 3; ++a) {
            const double rc = __dadd_rn(__dadd_rn(__dmul_rn(P[4 * a], c[0]), __dmul_rn(P[4 * a + 1], c[1])),
                                        __dmul_rn(P[4 * a + 2], c[2]));
            P[4 * a + 3] = __dsub_rn(__dadd_rn(P[4 * a + 3], c[a]), rc);
        }
    auto inv = [](const double* A, double* R) {          // (A^T | -A^T t)
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 3; ++j) R[4 * i + j] = A[4 * j + i];
            R[4 * i + 3] = -__dadd_rn(__dadd_rn(__dmul_rn(A[i], A[3]), __dmul_rn(A[4 + i], A[7])), __dmul_rn(A[8 + i], A[11]));
        }
    };
    auto cat = [](const double* A, const double* Bm, double* R) {    // A Bm as rigid transforms
        for (int i = 0; i < 3; ++i) {
            for (int j = 0; j < 4; ++j) {
                double s = __dadd_rn(__dadd_rn(__dmul_rn(A[4 * i], Bm[j]), __dmul_rn(A[4 * i + 1], Bm[4 + j])),
                                     __dmul_rn(A[4 * i + 2], Bm[8 + j]));
                R[4 * i + j] = j == 3 ? __dadd_rn(s, A[4 * i + 3]) : s;
            }
        }
    };
    const double* G = pose + 12 * b;
    if (f & REGTR_PREP_PERTURB_SRC) { inv(P, Q); cat(G, Q, O); }
    else cat(P, G, O);
    if (f & REGTR_PREP_SWAP) { inv(O, Q); for (int k = 0; k < 12; ++k) O[k] = Q[k]; }
    for (int k = 0; k < 12; ++k) out_pose[12 * b + k] = (float)O[k];
    const int other = pc == b ? B + b : b;
    for (int k = 0; k < 12; ++k) {
        mat[12 * pc + k] = P[k];
        mat[12 * other + k] = (k % 5 == 0) ? 1.0 : 0.0;     // identity: entries 0, 5, 10
    }
}

// Which input cloud fills output slot s (src_0..src_{B-1}, tgt_0..tgt_{B-1} of the augmented batch): a swapped
// pair's new source is its old target.
__device__ __forceinline__ int input_cloud(int s, int B, const int32_t* __restrict__ flags) {
    const int b = s < B ? s : s - B;
    const int side = (s < B) ^ ((flags[b] & REGTR_PREP_SWAP) != 0) ? 0 : 1;
    return side * B + b;
}

// One thread per output point: out[k] of slot s = transform(in[perm(k)]) + noise, one fp32 rounding of the float64
// value; the overlap mask follows the permutation.  The noise of input point j of (pair, side) is
// sigma * Box-Muller(Philox(counter = (j, 2 pair + side, step), key = seed)), pair = pair_base + b: the position of
// the pair in the global batch, so a slice of a batch draws what the same pairs draw in the whole batch.
__global__ void k_augment_points(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                                 const int32_t* __restrict__ nn, const double* __restrict__ mat,
                                 const int32_t* __restrict__ flags, const int32_t* __restrict__ out_offs, int out_cap,
                                 unsigned long long seed, unsigned long long step, int pair_base, double noise,
                                 float* __restrict__ out_xyz, uint8_t* __restrict__ out_mask) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= out_cap || p >= out_offs[2 * B]) return;
    const int s = regtr_cloud_of(out_offs, 2 * B, p);
    const int cin = input_cloud(s, B, flags);
    const int b = cin < B ? cin : cin - B, side = cin < B ? 0 : 1;
    const Keys ks = make_keys(seed, step);
    const int a0 = offs[cin];
    const Perm pm = make_perm(offs[cin + 1] - a0, (flags[b] & REGTR_PREP_SHUFFLE) != 0, ks, pair_base + b, side);
    const unsigned j = perm_fwd(pm, (unsigned)(p - out_offs[s]));
    const int i = a0 + (int)j;
    const double* m = mat + 12 * cin;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    double v[3] = {rt_row(m, x, y, z), rt_row(m + 4, x, y, z), rt_row(m + 8, x, y, z)};
    if (noise != 0.0) {
        const U4 r = philox(U4{j, 2u * (unsigned)(pair_base + b) + (unsigned)side, ks.s0, ks.s1}, ks.k0, ks.k1);
        const double m0 = sqrt(-2.0 * log(u01(r.x))), m1 = sqrt(-2.0 * log(u01(r.z)));
        double s0, c0, s1, c1;
        sincospi(2.0 * u01(r.y), &s0, &c0);
        sincospi(2.0 * u01(r.w), &s1, &c1);
        const double g[3] = {m0 * c0, m0 * s0, m1 * c1};
        for (int a = 0; a < 3; ++a) v[a] = __dadd_rn(v[a], __dmul_rn(noise, g[a]));
    }
    out_xyz[3 * p + 0] = (float)v[0]; out_xyz[3 * p + 1] = (float)v[1]; out_xyz[3 * p + 2] = (float)v[2];
    out_mask[p] = nn[i] >= 0;
}

// flag[i] = 1 for a source point kept as a correspondence: it has a neighbour with a nonzero index (the reference's
// `src_corr > 0`), the match is mutual, and both endpoints survive the shuffle's truncation to max_pts.  pos[i] =
// (new source index, new target index) before the swap.  flag[n_src_cap] = 0 (the scan's total).
__global__ void k_corr_flags(const int32_t* __restrict__ offs, int B, int n_src_cap, const int32_t* __restrict__ nn,
                             const int32_t* __restrict__ flags, unsigned long long seed, unsigned long long step,
                             int pair_base, int max_pts, int32_t* __restrict__ flag, int2* __restrict__ pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i > n_src_cap) return;
    int keep = 0;
    if (i < offs[B]) {
        const int b = regtr_cloud_of(offs, B, i);
        const int il = i - offs[b], s = nn[i];
        const int ns = offs[b + 1] - offs[b], nt = offs[B + b + 1] - offs[B + b];
        if (s > 0 && nn[offs[B + b] + s] == il) {
            const Keys ks = make_keys(seed, step);
            const bool sh = (flags[b] & REGTR_PREP_SHUFFLE) != 0;
            const int a = (int)perm_inv(make_perm(ns, sh, ks, pair_base + b, 0), (unsigned)il);
            const int t = (int)perm_inv(make_perm(nt, sh, ks, pair_base + b, 1), (unsigned)s);
            if (a < min(ns, max_pts) && t < min(nt, max_pts)) { keep = 1; pos[i] = make_int2(a, t); }
        }
    }
    flag[i] = keep;
}

// corr (2, corr_cap): kept pairs in ascending source index, rows swapped for swapped pairs; corr_offs[b] = first
// column of pair b (corr_offs[B] = total).
__global__ void k_corr_write(const int32_t* __restrict__ offs, int B, int n_src_cap, const int32_t* __restrict__ flag,
                             const int32_t* __restrict__ pre, const int2* __restrict__ pos,
                             const int32_t* __restrict__ flags, int corr_cap, int32_t* __restrict__ corr,
                             int32_t* __restrict__ corr_offs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= B) corr_offs[i] = pre[offs[i]];
    if (i >= n_src_cap || !flag[i]) return;
    const int b = regtr_cloud_of(offs, B, i);
    const int2 q = pos[i];
    const int k = pre[i];
    const bool sw = (flags[b] & REGTR_PREP_SWAP) != 0;
    corr[k] = sw ? q.y : q.x;
    corr[corr_cap + k] = sw ? q.x : q.y;
}

struct OverlapWs {
    double* xa;
    float* x32;
    void* grid;
    int32_t* order;
    void* gws;
    size_t gws_bytes, total;
};

OverlapWs carve_overlap(void* ws, int n_cap) {
    OverlapWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t n = (size_t)(n_cap > 0 ? n_cap : 1);
    w.xa = (double*)take(sizeof(double) * 3 * n);
    w.x32 = (float*)take(sizeof(float) * 3 * n);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.order = (int32_t*)take(sizeof(int32_t) * n);
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.total = off;
    return w;
}

struct AugWs {
    double* mat;
    int32_t *flag, *pre;
    int2* pos;
    size_t total;
};

AugWs carve_aug(void* ws, int n_src_cap, int B) {
    AugWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    w.mat = (double*)take(sizeof(double) * 24 * (size_t)B);
    w.flag = (int32_t*)take(sizeof(int32_t) * ((size_t)n_src_cap + 1));
    w.pre = (int32_t*)take(sizeof(int32_t) * ((size_t)n_src_cap + 1));
    w.pos = (int2*)take(sizeof(int2) * ((size_t)n_src_cap + 1));
    w.total = off;
    return w;
}

}  // namespace

extern "C" {

double regtr_overlap_coord_bound(double radius, float cell) {
    // Per point, fp32(x) / cell rounded to fp32 is within (2u + u^2)|x| / cell of x / cell (u = 2^-24); a pair of
    // points closer than r per axis therefore lands in neighbouring cells while r + (4u + 2u^2) M <= cell.
    const double u = 5.9604644775390625e-08;
    return ((double)cell - radius * (1.0 + 2.220446049250313e-16)) / (4.0 * u + 2.0 * u * u);
}

size_t regtr_overlap_ws_bytes(int n_cap) { return carve_overlap(nullptr, n_cap).total; }
size_t regtr_overlap_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap); }

int regtr_overlap_nn(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose, double radius,
                     float cell, int32_t* nn, uint32_t* status, void* ws, size_t ws_bytes, void* state,
                     size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !pose || !status || B <= 0 || 2 * B > 32767 || n_cap < 0 || !(radius > 0.0) ||
        !((double)cell > radius))
        return REGTR_ERR_ARG;
    if (n_cap == 0) return REGTR_OK;
    if (!xyz || !nn || !ws || !state) return REGTR_ERR_ARG;
    OverlapWs w = carve_overlap(ws, n_cap);
    if (ws_bytes < w.total || state_bytes < regtr_overlap_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const int T = 256;
    k_align<<<regtr_cdiv(n_cap, T), T, 0, st>>>(xyz, offs, B, n_cap, pose, regtr_overlap_coord_bound(radius, cell),
                                               w.xa, w.x32, status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, offs, 2 * B, n_cap, cell, w.grid, w.order, status, w.gws, w.gws_bytes,
                                        state, state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const int blocks = regtr_cdiv(n_cap, NN_WARPS);
    k_overlap_nn<<<blocks < 8 * REGTR_NUM_SMS ? blocks : 8 * REGTR_NUM_SMS, NN_WARPS * 32, 0, st>>>(
        w.xa, w.x32, offs, B, n_cap, w.order, grid_table(w.grid, (size_t)n_cap), cell_table_log2(n_cap),
        grid_sxyzi(w.grid), cell, radius * radius, nn);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_registration_fit(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose,
                           double radius, const int32_t* nn, double* out, uint32_t* status, void* stream_) {
    if (!offs || !pose || !out || !status || B <= 0 || 2 * B > 32767 || n_cap < 0 || !(radius > 0.0))
        return REGTR_ERR_ARG;
    if (n_cap > 0 && (!xyz || !nn)) return REGTR_ERR_ARG;
    k_registration_fit<<<2 * B, FIT_THREADS, 0, (cudaStream_t)stream_>>>(xyz, offs, B, pose, radius * radius, nn,
                                                                        out, status);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_registration_information(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose,
                                   double radius, const int32_t* nn, double* out, uint32_t* status, void* stream_) {
    if (!offs || !pose || !out || !status || B <= 0 || 2 * B > 32767 || n_cap < 0 || !(radius > 0.0))
        return REGTR_ERR_ARG;
    if (n_cap > 0 && (!xyz || !nn)) return REGTR_ERR_ARG;
    k_registration_information<<<B, FIT_THREADS, 0, (cudaStream_t)stream_>>>(xyz, offs, B, pose, radius * radius, nn,
                                                                            out, status);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_transform_clouds(const double* xyz, const int32_t* offs, int C, int n_cap, const double* pose, float* out,
                           void* stream_) {
    if (!offs || !pose || C <= 0 || C > 32767 || n_cap < 0) return REGTR_ERR_ARG;
    if (n_cap == 0) return REGTR_OK;
    if (!xyz || !out) return REGTR_ERR_ARG;
    const int T = 256;
    k_transform_clouds<<<regtr_cdiv(n_cap, T), T, 0, (cudaStream_t)stream_>>>(xyz, offs, C, n_cap, pose, out);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_train_augment_ws_bytes(int n_src_cap, int B) { return carve_aug(nullptr, n_src_cap, B).total; }
size_t regtr_train_augment_state_bytes(int n_src_cap) { return scan_state_bytes((long long)n_src_cap + 1); }

int regtr_train_augment(const double* xyz, const int32_t* offs, int B, int n_src_cap, const double* pose,
                        const int32_t* nn, const double* pert, const int32_t* flags, unsigned long long seed,
                        unsigned long long step, int pair_base, double noise, int max_pts, const int32_t* out_offs,
                        int out_cap, float* out_xyz, uint8_t* out_mask, float* out_pose, int32_t* corr, int corr_cap,
                        int32_t* corr_offs, void* ws, size_t ws_bytes, void* state, size_t state_bytes,
                        void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (pair_base < 0 || pair_base > (1 << 30)) return REGTR_ERR_ARG;
    if (!offs || !pose || !pert || !flags || !out_offs || !out_pose || !corr_offs || B <= 0 || 2 * B > 32767 ||
        n_src_cap < 0 || n_src_cap >= (1 << 30) || out_cap < 0 || corr_cap < n_src_cap || max_pts < 0 ||
        !(noise >= 0.0) || !ws || !state)
        return REGTR_ERR_ARG;
    if ((out_cap > 0 && (!xyz || !nn || !out_xyz || !out_mask)) || (n_src_cap > 0 && !corr)) return REGTR_ERR_ARG;
    AugWs w = carve_aug(ws, n_src_cap, B);
    if (ws_bytes < w.total || state_bytes < regtr_train_augment_state_bytes(n_src_cap)) return REGTR_ERR_WORKSPACE;
    const int T = 256;
    k_prep_pose<<<B, 256, 0, st>>>(xyz, offs, B, pose, pert, flags, w.mat, out_pose);
    REGTR_CHECK_LAUNCH();
    if (out_cap > 0) {
        k_augment_points<<<regtr_cdiv(out_cap, T), T, 0, st>>>(xyz, offs, B, nn, w.mat, flags, out_offs, out_cap, seed,
                                                               step, pair_base, noise, out_xyz, out_mask);
        REGTR_CHECK_LAUNCH();
    }
    k_corr_flags<<<regtr_cdiv(n_src_cap + 1, T), T, 0, st>>>(offs, B, n_src_cap, nn, flags, seed, step, pair_base,
                                                            max_pts, w.flag, w.pos);
    REGTR_CHECK_LAUNCH();
    const int rc = launch_scan<0>(w.flag, w.pre, n_src_cap + 1, nullptr, state, st);
    if (rc != REGTR_OK) return rc;
    k_corr_write<<<regtr_cdiv((n_src_cap > B ? n_src_cap : B) + 1, T), T, 0, st>>>(offs, B, n_src_cap, w.flag, w.pre,
                                                                                  w.pos, flags, corr_cap, corr,
                                                                                  corr_offs);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
