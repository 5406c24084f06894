// RANSAC over correspondences for B pairs at once: Open3D's registration_ransac_based_on_correspondence with
// TransformationEstimationPointToPoint (no scaling), CorrespondenceCheckerBasedOnEdgeLength / ...BasedOnDistance and
// RANSACConvergenceCriteria(max_iteration, confidence), restated with one deterministic sequential rule (DESIGN.md
// section 8, "RANSAC"; include/regtr_b200.h, regtr_ransac).
//
// Set-up: the valid correspondences of every pair are compacted in their original order, and one cell list is built
// over the targets (as ICP does).  Then the hypotheses run in chunks of first_chunk * 2^c (at most
// REGTR_RANSAC_CHUNK_MAX), three launches per chunk: generate (one thread per (pair, hypothesis): sample, checkers, Umeyama), validate (one
// CTA per (flagged hypothesis, block of VB source points), regtr_overlap_nn's search) and scan (one warp per pair:
// the hypotheses of the chunk in index order, the best and stop rule).  Only the scan decides: the other two stages
// may work on hypotheses past the stop, whose results are never read, so the output does not depend on the chunking
// or the batch.  The launch count depends on the arguments alone and nothing synchronises with the host.
#include <cfloat>

#include "cellgrid.cuh"
#include "philox.cuh"
#include "rigid.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int VB = 1024;                 // source points per validation CTA
constexpr int VAL_THREADS = 256;         // = regtr_registration_fit's FIT_THREADS: the same per-thread chains
constexpr int VAL_WARPS = VAL_THREADS / 32;
constexpr int GEN_THREADS = 128;
constexpr int SCAN_WARPS = 4;
constexpr unsigned RANSAC_WORD3 = 0x52534143u;   // "RSAC": counter word 3 of every sample draw

// Per-pair state between chunks (written by k_ransac_scan only, after k_ransac_compact).
struct RansacPair {
    int est_k;                           // Open3D's est_k_global
    int k;                               // hypotheses walked
    int vals;                            // hypotheses validated
    int best;                            // index of the best hypothesis, -1 before any
    int done, n_valid;
    double fit, rmse;                    // the best result
};

// One validation CTA's sums: Sigma d^2 of the matched points of its block and their count; rng: a moved source
// coordinate of the block beyond the bound.
struct Partial {
    double sum;
    int cnt, rng;
};

__device__ __forceinline__ double norm3_rn(double dx, double dy, double dz) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// The targets' fp32 copy for their cell list and their own offsets (tofs[c] = offs[B + c] - offs[B]), the source
// blocks of the validation (pair b owns blocks [bpre[b], bpre[b+1]), ceil(n_b / VB) of them) and the work counter.
// |coordinate| of a target beyond `bound`, or not finite, raises REGTR_STATUS_RANGE.
__global__ void k_ransac_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, int n_cap,
                              double bound, float* __restrict__ x32, int32_t* __restrict__ tofs,
                              int32_t* __restrict__ bpre, int* __restrict__ work_count, uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= B) tofs[i] = offs[B + i] - offs[B];
    if (i == 0) {
        int acc = 0;
        bpre[0] = 0;
        for (int b = 0; b < B; ++b) { acc += (offs[b + 1] - offs[b] + VB - 1) / VB; bpre[b + 1] = acc; }
        *work_count = 0;
    }
    if (i >= n_cap || i < offs[B] || i >= offs[2 * B]) return;
    const double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    const int j = i - offs[B];
    x32[3 * j + 0] = (float)x; x32[3 * j + 1] = (float)y; x32[3 * j + 2] = (float)z;
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One CTA per pair: the valid correspondences (mask[i] != 0, every one without a mask) copied in their original
// order to the front of the pair's range of ka / kc, n_valid of them; the initial state and Open3D's empty result
// (identity, zeros, best -1).  A pair with n_valid < ransac_n or max_iter = 0 is done at once.
__global__ void __launch_bounds__(VAL_THREADS)
k_ransac_compact(const double* __restrict__ ca, const double* __restrict__ cc, const int32_t* __restrict__ coffs,
                 const uint8_t* __restrict__ mask, int ransac_n, int max_iter, double* __restrict__ ka,
                 double* __restrict__ kc, RansacPair* __restrict__ pst, double* __restrict__ pose_out,
                 double* __restrict__ result) {
    __shared__ int s_warp[VAL_WARPS];
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int m0 = coffs[b], m1 = coffs[b + 1];
    int base = 0;                                      // valid correspondences before this round
    for (int r = m0; r < m1; r += VAL_THREADS) {
        const int i = r + t;
        const int f = i < m1 && (!mask || mask[i] != 0);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp[warp] = __popc(bal);
        __syncthreads();
        int before = base, total = base;
        for (int w = 0; w < VAL_WARPS; ++w) {
            if (w < warp) before += s_warp[w];
            total += s_warp[w];
        }
        if (f) {
            const int o = m0 + before + __popc(bal & ((1u << lane) - 1u));
            for (int a = 0; a < 3; ++a) { ka[3 * o + a] = ca[3 * i + a]; kc[3 * o + a] = cc[3 * i + a]; }
        }
        base = total;
        __syncthreads();
    }
    if (t != 0) return;
    RansacPair s;
    s.est_k = max_iter; s.k = 0; s.vals = 0; s.best = -1;
    s.done = base < ransac_n || max_iter == 0;
    s.n_valid = base;
    s.fit = 0.0; s.rmse = 0.0;
    pst[b] = s;
    for (int e = 0; e < 12; ++e) pose_out[12 * b + e] = (e % 5 == 0) ? 1.0 : 0.0;
    double* o = result + 5 * b;
    o[0] = 0.0; o[1] = 0.0; o[2] = 0.0; o[3] = 0.0; o[4] = -1.0;
}

// One thread per hypothesis k = s0 + h of pair b = blockIdx.y (skipped when the pair is done or k >= est_k).  The
// sample: draw j < ransac_n is mulhi32(w, n_valid), w word j & 3 of Philox4x32-10 at counter
// (k, pair_base + b, j >> 2, "RSAC") with key (seed lo, seed hi).  Rejected (flag 0): a repeated index; the edge-length
// checker (edge > 0) failing on a pair; Umeyama without scaling (means, Sigma = sum (c - mc)(a - ma)^T / n, Jacobi
// SVD, reflection fix, t = mc - R ma) with S[1] <= 1e-12 S[0]; the distance checker (dist > 0) failing on a point.
// Otherwise flag 1, T stored, and the hypothesis's validation blocks appended to the work list.
__global__ void __launch_bounds__(GEN_THREADS)
k_ransac_generate(const double* __restrict__ ka, const double* __restrict__ kc, const int32_t* __restrict__ coffs,
                  const int32_t* __restrict__ offs, const int32_t* __restrict__ bpre, const RansacPair* __restrict__ pst,
                  int s0, int hc, int hcap, int ransac_n, double edge, double dist, unsigned k0, unsigned k1,
                  int pair_base, double* __restrict__ hyp, int* __restrict__ hflag, int2* __restrict__ work,
                  int* work_count) {
    const int b = blockIdx.y, h = blockIdx.x * GEN_THREADS + threadIdx.x;
    if (h >= hc) return;
    const RansacPair s = pst[b];
    const int k = s0 + h;
    if (s.done || k >= s.est_k) return;
    const int n = s.n_valid;
    const double* A = ka + 3 * (size_t)coffs[b];
    const double* C = kc + 3 * (size_t)coffs[b];
    int idx[REGTR_RANSAC_MAX_N];
    U4 v{0u, 0u, 0u, 0u};
    for (int j = 0; j < ransac_n; ++j) {
        if ((j & 3) == 0) v = philox(U4{(unsigned)k, (unsigned)(pair_base + b), (unsigned)(j >> 2), RANSAC_WORD3}, k0, k1);
        const unsigned w = (j & 3) == 0 ? v.x : (j & 3) == 1 ? v.y : (j & 3) == 2 ? v.z : v.w;
        idx[j] = (int)__umulhi(w, (unsigned)n);
    }
    bool ok = true;
    for (int i = 0; i < ransac_n && ok; ++i)
        for (int j = i + 1; j < ransac_n; ++j) ok = ok && idx[i] != idx[j];
    if (ok && edge > 0.0) {
        for (int i = 0; i < ransac_n && ok; ++i)
            for (int j = i + 1; j < ransac_n; ++j) {
                const double* ai = A + 3 * idx[i]; const double* aj = A + 3 * idx[j];
                const double* ci = C + 3 * idx[i]; const double* cj = C + 3 * idx[j];
                const double da = norm3_rn(__dsub_rn(ai[0], aj[0]), __dsub_rn(ai[1], aj[1]), __dsub_rn(ai[2], aj[2]));
                const double dc = norm3_rn(__dsub_rn(ci[0], cj[0]), __dsub_rn(ci[1], cj[1]), __dsub_rn(ci[2], cj[2]));
                ok = ok && !(da < __dmul_rn(dc, edge) || dc < __dmul_rn(da, edge));
            }
    }
    double T[12];
    if (ok) {
        double ma[3] = {0.0, 0.0, 0.0}, mc[3] = {0.0, 0.0, 0.0};
        for (int j = 0; j < ransac_n; ++j)
            for (int a = 0; a < 3; ++a) { ma[a] += A[3 * idx[j] + a]; mc[a] += C[3 * idx[j] + a]; }
        for (int a = 0; a < 3; ++a) { ma[a] /= (double)ransac_n; mc[a] /= (double)ransac_n; }
        double Sg[3][3] = {{0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0}};
        for (int j = 0; j < ransac_n; ++j) {
            double dp[3], dq[3];
            for (int a = 0; a < 3; ++a) { dp[a] = A[3 * idx[j] + a] - ma[a]; dq[a] = C[3 * idx[j] + a] - mc[a]; }
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) Sg[r][c] += dq[r] * dp[c];
        }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Sg[r][c] /= (double)ransac_n;
        double U[3][3], S[3], V[3][3];
        svd3_jacobi(Sg, U, S, V);
        ok = S[1] > 1e-12 * S[0];
        const double d = det3(U) * det3(V) < 0.0 ? -1.0 : 1.0;
        double R[3][3];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) R[r][c] = U[r][0] * V[c][0] + U[r][1] * V[c][1] + d * U[r][2] * V[c][2];
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) T[4 * r + c] = R[r][c];
            T[4 * r + 3] = mc[r] - (R[r][0] * ma[0] + R[r][1] * ma[1] + R[r][2] * ma[2]);
        }
    }
    if (ok && dist > 0.0) {
        for (int j = 0; j < ransac_n && ok; ++j) {
            const double* a = A + 3 * idx[j]; const double* c = C + 3 * idx[j];
            const double e = norm3_rn(__dsub_rn(rt_row(T, a[0], a[1], a[2]), c[0]),
                                      __dsub_rn(rt_row(T + 4, a[0], a[1], a[2]), c[1]),
                                      __dsub_rn(rt_row(T + 8, a[0], a[1], a[2]), c[2]));
            ok = !(e > dist);
        }
    }
    const size_t slot = (size_t)b * hcap + h;
    hflag[slot] = ok ? 1 : 0;
    if (!ok) return;
    for (int e = 0; e < 12; ++e) hyp[12 * slot + e] = T[e];
    const int nb = bpre[b + 1] - bpre[b];
    if (nb == 0) return;
    const int w0 = atomicAdd(work_count, nb);          // list order is free: every item writes its own slot
    for (int j = 0; j < nb; ++j) work[w0 + j] = make_int2(b * hcap + h, j);
}

// One CTA per work item (flagged hypothesis h of pair b, source block j), grid-strided over the list.  The block's
// points are moved by T (rt_row) and searched as in k_overlap_nn (one warp per point, lanes 0..26 one stencil cell
// each, float64 d2 = (dx dx + dy dy) + dz dz without contraction, strictly below r2, ties to the lowest index).
// Thread t = 32 warp + lane owns points i0 + t + 256 r in ascending r and sums their d2 (k_registration_fit's
// chain), then the fixed tree of k_registration_fit.  part[h][bpre[b] + j] = (sum, count, range flag).
__global__ void __launch_bounds__(VAL_THREADS)
k_ransac_validate(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, int hcap, int nbtot,
                  const int32_t* __restrict__ bpre, const double* __restrict__ hyp, const int2* __restrict__ work,
                  const int* __restrict__ work_count, const CellSlot* __restrict__ table, int log2t,
                  const float4* __restrict__ sxyzi, float cell, double r2, double bound, Partial* __restrict__ part) {
    __shared__ double s_sum[VAL_THREADS];
    __shared__ int s_cnt[VAL_THREADS];
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    const int nw = *work_count, t0 = offs[B];
    for (int it = blockIdx.x; it < nw; it += gridDim.x) {
        const int2 wi = work[it];
        const int b = wi.x / hcap, h = wi.x - b * hcap, j = wi.y;
        const double* m = hyp + 12 * (size_t)wi.x;
        const int i0 = offs[b] + j * VB, i1 = min(i0 + VB, offs[b + 1]);
        double sum = 0.0;
        int cnt = 0, rng = 0;
        for (int r = 0; r < VB / VAL_THREADS; ++r) {
            const int g = i0 + VAL_THREADS * r + 32 * warp;          // this warp's 32 points
            if (g >= i1) break;
            double px = 0.0, py = 0.0, pz = 0.0;
            if (g + lane < i1) {
                const double x = xyz[3 * (g + lane) + 0], y = xyz[3 * (g + lane) + 1], z = xyz[3 * (g + lane) + 2];
                px = rt_row(m, x, y, z); py = rt_row(m + 4, x, y, z); pz = rt_row(m + 8, x, y, z);
                if (!(fabs(px) <= bound && fabs(py) <= bound && fabs(pz) <= bound)) rng = 1;
            }
            const int np_ = min(32, i1 - g);
            for (int l = 0; l < np_; ++l) {
                const double qx = __shfl_sync(0xffffffffu, px, l), qy = __shfl_sync(0xffffffffu, py, l),
                             qz = __shfl_sync(0xffffffffu, pz, l);
                const int cx = regtr_cell_of((float)qx, cell), cy = regtr_cell_of((float)qy, cell),
                          cz = regtr_cell_of((float)qz, cell);
                int c_start = 0, c_cnt = 0;
                if (lane < 27) {
                    const int x = cx + lane / 9 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane % 3 - 1;
                    if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767)
                        cell_lookup(table, log2t, regtr_pack_key(b, x, y, z), c_start, c_cnt);
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
                    const int tt = base + lane;
                    int cellid = 0;
#pragma unroll
                    for (int step = 16; step > 0; step >>= 1) {
                        const int pv = __shfl_sync(0xffffffffu, pre, cellid + step - 1);
                        if (pv <= tt) cellid += step;
                    }
                    const int cell_pre = __shfl_sync(0xffffffffu, pre, cellid);
                    const int cell_cnt = __shfl_sync(0xffffffffu, c_cnt, cellid);
                    const int cell_start = __shfl_sync(0xffffffffu, c_start, cellid);
                    if (tt < total) {
                        const int q = t0 + __float_as_int(sxyzi[cell_start + (tt - (cell_pre - cell_cnt))].w);
                        const double dx = __dsub_rn(qx, xyz[3 * q + 0]), dy = __dsub_rn(qy, xyz[3 * q + 1]),
                                     dz = __dsub_rn(qz, xyz[3 * q + 2]);
                        const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                        if (d2 < best || (d2 == best && bi >= 0 && q < bi)) { best = d2; bi = q; }
                    }
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const double ob = __shfl_xor_sync(0xffffffffu, best, o);
                    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                    if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
                }
                if (lane == l && bi >= 0) { sum = __dadd_rn(sum, best); ++cnt; }
            }
        }
        const int any_rng = __syncthreads_or(rng);
        s_sum[t] = sum;
        s_cnt[t] = cnt;
        __syncthreads();
        for (int hh = VAL_THREADS / 2; hh > 0; hh >>= 1) {
            if (t < hh) { s_sum[t] = __dadd_rn(s_sum[t], s_sum[t + hh]); s_cnt[t] += s_cnt[t + hh]; }
            __syncthreads();
        }
        if (t == 0) {
            Partial p;
            p.sum = s_sum[0]; p.cnt = s_cnt[0]; p.rng = any_rng;
            part[(size_t)h * nbtot + bpre[b] + j] = p;
        }
        __syncthreads();                                 // s_sum / s_cnt are reused by the next item
    }
}

// One warp per pair: the chunk's hypotheses k = s0 .. s0 + hc - 1 in order while k < est_k.  A flagged one is
// validated: its blocks' sums are combined (lane l adds blocks l, l + 32, ... in order, then the xor butterfly),
// fitness = count / n_src, rmse = sqrt(sum / count); validations += 1 and its range flag goes to the status word.
// Better (higher fitness, or equal fitness and lower rmse): it becomes the best, pose_out = its T, and
// d = log(1 - confidence) / log(1 - fitness^n) (the power by n - 1 products) lowers est_k to ceil(d) when
// 0 <= d < est_k.  The pair is done once k >= est_k or k = max_iter.  The last warp of the grid resets the work list.
__global__ void __launch_bounds__(SCAN_WARPS * 32)
k_ransac_scan(const int32_t* __restrict__ offs, int B, int s0, int hc, int hcap, int nbtot, int max_iter,
              int ransac_n, double log_conf, const int32_t* __restrict__ bpre, const double* __restrict__ hyp,
              const int* __restrict__ hflag, const Partial* __restrict__ part, RansacPair* __restrict__ pst,
              double* __restrict__ pose_out, double* __restrict__ result, int* work_count, uint32_t* status) {
    const int lane = threadIdx.x & 31, b = blockIdx.x * SCAN_WARPS + (threadIdx.x >> 5);
    if (blockIdx.x == 0 && threadIdx.x == 0) *work_count = 0;   // validate has finished: stream order
    if (b >= B) return;
    RansacPair s = pst[b];
    if (s.done) return;
    const int n_src = offs[b + 1] - offs[b], p0 = bpre[b], nb = bpre[b + 1] - p0;
    const int end = s0 + hc;
    int walked = s.k, rng = 0;
    bool stop = false;
    for (int base = 0; base < hc && !stop; base += 32) {
        const int h = base + lane;
        const bool f = h < hc && s0 + h < s.est_k && hflag[(size_t)b * hcap + h] != 0;
        unsigned todo = __ballot_sync(0xffffffffu, f);
        while (todo) {
            const int l = __ffs(todo) - 1;
            todo &= todo - 1u;
            const int hh = base + l, k = s0 + hh;
            if (k >= s.est_k) { stop = true; break; }
            double sum = 0.0;
            int cnt = 0, rg = 0;
            for (int j = lane; j < nb; j += 32) {
                const Partial p = part[(size_t)hh * nbtot + p0 + j];
                sum = __dadd_rn(sum, p.sum); cnt += p.cnt; rg |= p.rng;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                sum = __dadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o));
                cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
            }
            rng |= __any_sync(0xffffffffu, rg);
            const double fit = n_src > 0 ? __ddiv_rn((double)cnt, (double)n_src) : 0.0;
            const double rmse = cnt > 0 ? __dsqrt_rn(__ddiv_rn(sum, (double)cnt)) : 0.0;
            s.vals += 1;
            walked = k + 1;
            if (fit > s.fit || (fit == s.fit && rmse < s.rmse)) {
                s.fit = fit; s.rmse = rmse; s.best = k;
                if (lane < 12) pose_out[12 * b + lane] = hyp[12 * ((size_t)b * hcap + hh) + lane];
                double pw = fit;
                for (int e = 1; e < ransac_n; ++e) pw = __dmul_rn(pw, fit);
                const double d = __ddiv_rn(log_conf, log(__dsub_rn(1.0, pw)));
                if (d >= 0.0 && d < (double)s.est_k) s.est_k = (int)ceil(d);
            }
        }
    }
    const int reach = s.est_k < end ? s.est_k : end;
    s.k = walked > reach ? walked : reach;
    s.done = s.k >= s.est_k || s.k >= max_iter;
    if (lane == 0) {
        pst[b] = s;
        double* o = result + 5 * b;
        o[0] = s.fit; o[1] = s.rmse; o[2] = (double)s.k; o[3] = (double)s.vals; o[4] = (double)s.best;
        if (rng) atomicOr(status, REGTR_STATUS_RANGE);
    }
}

struct RansacWs {
    double *ka, *kc, *hyp;
    float* x32;
    int32_t *tofs, *bpre;
    int *hflag, *work_count;
    int2* work;
    Partial* part;
    RansacPair* pst;
    void *grid, *gws;
    size_t gws_bytes, total;
};

// The chunk sizes: first_chunk * 2^c, at most REGTR_RANSAC_CHUNK_MAX, the last one cut at max_iter.
int chunk_size(long long start, int first_chunk, int c, int max_iter) {
    long long sz = (long long)first_chunk << (c < 20 ? c : 20);
    if (sz > REGTR_RANSAC_CHUNK_MAX) sz = REGTR_RANSAC_CHUNK_MAX;
    if (sz > max_iter - start) sz = max_iter - start;
    return (int)sz;
}

int largest_chunk(int max_iter, int first_chunk) {
    long long start = 0;
    int big = 0;
    for (int c = 0; start < max_iter; ++c) {
        const int sz = chunk_size(start, first_chunk, c, max_iter);
        big = sz > big ? sz : big;
        start += sz;
    }
    return big > 0 ? big : 1;
}

int n_blocks_cap(int n_cap, int B) { return regtr_cdiv(n_cap, VB) + B; }

RansacWs carve_ransac(void* ws, int n_cap, int m_cap, int B, int hcap) {
    RansacWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t n = (size_t)n_cap, m = (size_t)m_cap, H = (size_t)hcap, nbt = (size_t)n_blocks_cap(n_cap, B);
    w.ka = (double*)take(sizeof(double) * 3 * m);
    w.kc = (double*)take(sizeof(double) * 3 * m);
    w.x32 = (float*)take(sizeof(float) * 3 * n);
    w.tofs = (int32_t*)take(sizeof(int32_t) * ((size_t)B + 1));
    w.bpre = (int32_t*)take(sizeof(int32_t) * ((size_t)B + 1));
    w.work_count = (int*)take(sizeof(int));
    w.pst = (RansacPair*)take(sizeof(RansacPair) * (size_t)B);
    w.hyp = (double*)take(sizeof(double) * 12 * H * (size_t)B);
    w.hflag = (int*)take(sizeof(int) * H * (size_t)B);
    w.work = (int2*)take(sizeof(int2) * H * nbt);
    w.part = (Partial*)take(sizeof(Partial) * H * nbt);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.total = off;
    return w;
}

}  // namespace

extern "C" {

size_t regtr_ransac_ws_bytes(int n_cap, int m_cap, int B, int max_iter, int first_chunk) {
    const int fc = first_chunk >= 1 && first_chunk <= REGTR_RANSAC_CHUNK_MAX ? first_chunk : 1;
    return carve_ransac(nullptr, n_cap > 0 ? n_cap : 1, m_cap > 0 ? m_cap : 1, B > 0 ? B : 1,
                        largest_chunk(max_iter > 0 ? max_iter : 0, fc)).total;
}

int regtr_ransac(const double* xyz, const int32_t* offs, int B, int n_cap, const double* corr_src,
                 const double* corr_tgt, const int32_t* coffs, const uint8_t* corr_mask, int m_cap, double max_dist,
                 float cell, const regtr_ransac_options* opt, double* pose_out, double* result, uint32_t* status,
                 void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !coffs || !opt || !pose_out || !result || !status || !ws || !state || B <= 0 || 2 * B > 32767 ||
        n_cap < 0 || m_cap < 0 || (n_cap > 0 && !xyz) || (m_cap > 0 && (!corr_src || !corr_tgt)) ||
        !(max_dist > 0.0) || !((double)cell > max_dist))
        return REGTR_ERR_ARG;
    const regtr_ransac_options o = *opt;
    if (o.max_iteration < 0 || !(o.confidence >= 0.0 && o.confidence <= 1.0) || o.ransac_n < 3 ||
        o.ransac_n > REGTR_RANSAC_MAX_N || !(o.edge_length >= 0.0 && o.edge_length <= DBL_MAX) ||
        !(o.distance >= 0.0 && o.distance <= DBL_MAX) || o.pair_base < 0 || o.first_chunk < 1 ||
        o.first_chunk > REGTR_RANSAC_CHUNK_MAX)
        return REGTR_ERR_ARG;
    const int nc = n_cap > 0 ? n_cap : 1, mc = m_cap > 0 ? m_cap : 1;
    const int hcap = largest_chunk(o.max_iteration, o.first_chunk);
    RansacWs w = carve_ransac(ws, nc, mc, B, hcap);
    if (ws_bytes < w.total || state_bytes < regtr_cellgrid_state_bytes(nc)) return REGTR_ERR_WORKSPACE;
    const double bound = regtr_overlap_coord_bound(max_dist, cell);
    const int T = 256;
    k_ransac_init<<<regtr_cdiv((nc > B + 1 ? nc : B + 1), T), T, 0, st>>>(xyz, offs, B, nc, bound, w.x32, w.tofs,
                                                                          w.bpre, w.work_count, status);
    REGTR_CHECK_LAUNCH();
    k_ransac_compact<<<B, VAL_THREADS, 0, st>>>(corr_src, corr_tgt, coffs, corr_mask, o.ransac_n, o.max_iteration,
                                                 w.ka, w.kc, w.pst, pose_out, result);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, w.tofs, B, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes,
                                        state, state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const CellSlot* table = grid_table(w.grid, (size_t)nc);
    const float4* sxyzi = grid_sxyzi(w.grid);
    const int log2t = cell_table_log2(nc), nbtot = n_blocks_cap(nc, B);
    const double log_conf = log(1.0 - o.confidence);
    const unsigned k0 = (unsigned)o.seed, k1 = (unsigned)(o.seed >> 32);
    long long s0 = 0;
    for (int c = 0; s0 < o.max_iteration; ++c) {
        const int hc = chunk_size(s0, o.first_chunk, c, o.max_iteration);
        k_ransac_generate<<<dim3(regtr_cdiv(hc, GEN_THREADS), B), GEN_THREADS, 0, st>>>(
            w.ka, w.kc, coffs, offs, w.bpre, w.pst, (int)s0, hc, hcap, o.ransac_n, o.edge_length, o.distance, k0, k1,
            o.pair_base, w.hyp, w.hflag, w.work, w.work_count);
        REGTR_CHECK_LAUNCH();
        k_ransac_validate<<<8 * REGTR_NUM_SMS, VAL_THREADS, 0, st>>>(xyz, offs, B, hcap, nbtot, w.bpre, w.hyp, w.work,
                                                                     w.work_count, table, log2t, sxyzi, cell,
                                                                     max_dist * max_dist, bound, w.part);
        REGTR_CHECK_LAUNCH();
        k_ransac_scan<<<regtr_cdiv(B, SCAN_WARPS), SCAN_WARPS * 32, 0, st>>>(
            offs, B, (int)s0, hc, hcap, nbtot, o.max_iteration, o.ransac_n, log_conf, w.bpre, w.hyp, w.hflag, w.part,
            w.pst, pose_out, result, w.work_count, status);
        REGTR_CHECK_LAUNCH();
        s0 += hc;
    }
    return REGTR_OK;
}

}  // extern "C"
