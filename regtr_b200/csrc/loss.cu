// RegTR's training losses on the packed coarse tokens (regtr.py:237-294 of the reference): the ground-truth overlap
// pyramid, the overlap BCE and the correspondence L1 with their gradients, and the InfoNCE feature loss
// (feature_loss.py:246-314) forward and backward.  Every launch count is independent of the number of pairs, nothing
// synchronises with the host, and every sum runs in a fixed order (no float atomics): two runs are bit-identical.
//
// Token layout: the N coarse tokens are the B source clouds followed by the B target clouds; offs (2B+1, int32, device)
// holds their starts.  Pair b is source cloud b against target cloud B + b.
//
// InfoNCE geometry rule.  The source key point is moved by the ground-truth pose in fp32, in the evaluation order of
// x @ R^T + t without contraction.  The squared distance to a target key point is the sum of the squared coordinate
// differences, taken in float64 from the fp32 coordinates, and is compared with r_p^2 and r_n^2 rounded from the
// doubles r_p and r_n.  The positive of a source token is its nearest target token of the same pair, ties to the lowest
// index; the token is an anchor when that distance is strictly below r_p; target tokens strictly inside r_n other than
// the positive are ignored.  torch.cdist's GEMM form can disagree with this only for distances within rounding of a
// threshold or of a tie.
//
// InfoNCE logits are fp32 FMA chains over the 256 channels in ascending order, one chain per (source, target) entry:
// the forward and both backward passes call the same tile function, so the recomputed softmax uses the very logits the
// stored log-sum-exp was built from.
#include <math.h>

#include "common.cuh"

static_assert(sizeof(regtr_loss_args) == 568, "regtr_loss_args layout");

namespace {

constexpr int D = REGTR_LOSS_DIM;   // 256 channels
constexpr int TM = 32;              // tile edge (rows owned by a CTA, rows streamed per step)
constexpr int KC = 64;              // channels of the streamed rows staged per step
constexpr int PW = 256;             // tokens per CTA of the pointwise kernel

// R x + t of pair b (inverse: R^T x - R^T t), the fp32 operations of losses.se3_transform_list / se3_inv in order.
__device__ __forceinline__ void gt_point(const float* __restrict__ pose, int b, bool inverse, const float* x,
                                         float out[3]) {
    const float* P = pose + 12 * b;
    float r[3][3], t[3];
    if (!inverse) {
        for (int j = 0; j < 3; ++j) {
            for (int k = 0; k < 3; ++k) r[j][k] = P[4 * j + k];
            t[j] = P[4 * j + 3];
        }
    } else {
        for (int j = 0; j < 3; ++j)
            for (int k = 0; k < 3; ++k) r[j][k] = P[4 * k + j];
        for (int j = 0; j < 3; ++j) {
            float s = __fmul_rn(r[j][0], P[3]);
            s = __fadd_rn(s, __fmul_rn(r[j][1], P[7]));
            s = __fadd_rn(s, __fmul_rn(r[j][2], P[11]));
            t[j] = -s;
        }
    }
    for (int j = 0; j < 3; ++j) {
        float s = __fmul_rn(x[0], r[j][0]);
        s = __fadd_rn(s, __fmul_rn(x[1], r[j][1]));
        s = __fadd_rn(s, __fmul_rn(x[2], r[j][2]));
        out[j] = __fadd_rn(s, t[j]);
    }
}

__device__ __forceinline__ double dist2(const float* a, const float* b) {
    const double dx = (double)a[0] - (double)b[0], dy = (double)a[1] - (double)b[1], dz = (double)a[2] - (double)b[2];
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// Sum over the block in a fixed order: xor-shuffle tree per warp, then thread 0 adds the warp sums in warp order.
// `red` holds one double per warp; the result is returned to every thread.
__device__ double block_sum(double v, double* red) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
    return s;
}

// ---------------------------------------------------------------------------------------------- overlap pyramid

__global__ void k_overlap_level(const float* __restrict__ prev, const int32_t* __restrict__ pool, int K, int n,
                                const int32_t* __restrict__ n_prev_dev, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int n_prev = *n_prev_dev;
    float s = 0.f;
    int cnt = 0;
    for (int k = 0; k < K; ++k) {
        const int j = pool[(long long)i * K + k];
        if (j >= 0 && j < n_prev) {
            s = __fadd_rn(s, prev[j]);
            ++cnt;
        }
    }
    const float v = __fdiv_rn(s, (float)cnt);          // 0 / 0 stays NaN
    out[i] = v < 0.f ? 0.f : (v > 1.f ? 1.f : v);
}

// ---------------------------------------------------------------------------------------------- symmetrised W

// Ws is written as the TF32 halves the 3xTF32 GEMM reads (Ws = hi + lo, the rounding of regtr_split_tf32): it is a
// fresh matrix every step, so splitting it here saves the separate pass over it.
__global__ void k_sym_weight(const float* __restrict__ W, float* __restrict__ hi, float* __restrict__ lo) {
    const int r = blockIdx.x, c = threadIdx.x;
    const float v = (c >= r ? W[r * D + c] : 0.f) + (r >= c ? W[c * D + r] : 0.f);
    const float h = regtr_tf32_rne(v);
    hi[r * D + c] = h;
    lo[r * D + c] = regtr_tf32_rne(v - h);
}

__global__ void k_sym_weight_bwd(const float* __restrict__ dWs, float* __restrict__ dW) {
    const int r = blockIdx.x, c = threadIdx.x;
    if (c >= r) dW[r * D + c] += dWs[r * D + c] + dWs[c * D + r];
}

// ---------------------------------------------------------------------------------------------- BCE and L1

// ws: [L][n_chunks][3] partial sums (bce, src w*err, tgt w*err), then the two denominators max(sum w, 1e-6).
__global__ void __launch_bounds__(PW) k_loss_pointwise(const regtr_loss_args a) {
    __shared__ double red[PW / 32];
    const int l = blockIdx.y, chunk = blockIdx.x, n_chunks = gridDim.x;
    const int n_src = a.offs[a.B];
    double ws = 0.0, wt = 0.0;
    for (int i = threadIdx.x; i < a.N; i += PW) {
        const double v = (double)a.w[i];
        if (i < n_src) ws += v; else wt += v;
    }
    const double den_s = fmax(block_sum(ws, red), 1e-6), den_t = fmax(block_sum(wt, red), 1e-6);
    const bool ov_on = a.ov_val[l] >= 0, corr_on = a.corr_val[l] >= 0;
    const int i = chunk * PW + threadIdx.x;
    double bce = 0.0, es = 0.0, et = 0.0;
    if (i < a.N) {
        const int c = regtr_cloud_of(a.offs, 2 * a.B, i);
        const bool src = c < a.B;
        const float y = a.w[i];
        const long long li = (long long)l * a.N + i;
        const float x = a.logit[li];
        if (ov_on) {
            bce = (double)(fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x))));
            a.dlogit[li] = (1.f / (1.f + expf(-x)) - y) / (float)a.N;
        } else {
            a.dlogit[li] = 0.f;
        }
        if (corr_on) {
            float g[3];
            gt_point(a.pose, src ? c : c - a.B, !src, a.xyz + 3 * (long long)i, g);
            const double den = src ? den_s : den_t;
            float err = 0.f;
            for (int j = 0; j < 3; ++j) {
                const float d = __fsub_rn(a.corr[3 * li + j], g[j]);
                err = __fadd_rn(err, fabsf(d));
                const float sg = d > 0.f ? 1.f : (d < 0.f ? -1.f : d);      // sign(0) = 0, NaN stays NaN
                a.dcorr[3 * li + j] = (float)((double)y * (double)sg / den);
            }
            (src ? es : et) = (double)y * (double)err;
        } else {
            for (int j = 0; j < 3; ++j) a.dcorr[3 * li + j] = 0.f;
        }
    }
    bce = block_sum(bce, red);
    es = block_sum(es, red);
    et = block_sum(et, red);
    if (threadIdx.x == 0) {
        double* p = a.ws + ((long long)l * n_chunks + chunk) * 3;
        p[0] = bce; p[1] = es; p[2] = et;
        if (l == 0 && chunk == 0) {
            double* den = a.ws + (long long)a.L * n_chunks * 3;
            den[0] = den_s; den[1] = den_t;
        }
    }
}

__global__ void k_loss_scale(const regtr_loss_args a) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)a.L * a.N) return;
    const int l = (int)(t / a.N);
    const float go = a.ov_val[l] >= 0 ? a.g[a.ov_val[l]] : 0.f;
    const float gc = a.corr_val[l] >= 0 ? a.g[a.corr_val[l]] : 0.f;
    a.dlogit_out[t] = a.ov_val[l] >= 0 ? go * a.dlogit[t] : 0.f;
    for (int j = 0; j < 3; ++j) a.dcorr_out[3 * t + j] = a.corr_val[l] >= 0 ? gc * a.dcorr[3 * t + j] : 0.f;
}

// ---------------------------------------------------------------------------------------------- InfoNCE geometry

__global__ void k_infonce_match(const regtr_loss_args a) {
    const int b = blockIdx.y;
    const int s0 = a.offs[b], s1 = a.offs[b + 1], t0 = a.offs[a.B + b], t1 = a.offs[a.B + b + 1];
    const int i = s0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s1) return;
    float g[3];
    gt_point(a.pose, b, false, a.xyz + 3 * (long long)i, g);
    for (int j = 0; j < 3; ++j) a.src_gt[3 * (long long)i + j] = g[j];
    int best = -1;
    double bd = INFINITY;
    for (int j = t0; j < t1; ++j) {
        const double d = dist2(g, a.xyz + 3 * (long long)j);
        if (d < bd || best < 0) { bd = d; best = j; }
    }
    a.pos[i] = best;
    a.anchor[i] = (best >= 0 && bd < a.rp2) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------- InfoNCE logits

struct Tile {
    float res[TM][D + 1];       // the CTA's own rows, all channels
    float chunk[TM][KC + 1];    // KC channels of the streamed rows
    float s[TM][TM + 1];        // [source row][target row]: logits, then gradient weights
    float gt[TM][3];            // moved source key points of the tile's source rows
    float txyz[TM][3];          // key points of the tile's target rows
    int pos[TM];
    float lse[TM], c[TM];
};

__device__ __forceinline__ void load_resident(Tile& T, const float* __restrict__ base, int n_rows) {
    for (int e = threadIdx.x; e < TM * D; e += blockDim.x) {
        const int r = e / D, k = e - r * D;
        T.res[r][k] = r < n_rows ? base[(long long)r * D + k] : 0.f;
    }
}

// acc[u][v] = <res[ro + u], streamed row co + v>: one fmaf chain per entry over the channels in ascending order, so
// the value does not depend on which side is resident.  Begins and ends with the block in step.
__device__ __forceinline__ void tile_dots(Tile& T, const float* __restrict__ stream, int n_stream, float acc[2][2]) {
    const int ro = 2 * (threadIdx.x >> 4), co = 2 * (threadIdx.x & 15);
    acc[0][0] = acc[0][1] = acc[1][0] = acc[1][1] = 0.f;
    for (int kc = 0; kc < D; kc += KC) {
        __syncthreads();
        for (int e = threadIdx.x; e < TM * KC; e += blockDim.x) {
            const int r = e / KC, k = e - r * KC;
            T.chunk[r][k] = r < n_stream ? stream[(long long)r * D + kc + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < KC; ++k) {
            const float r0 = T.res[ro][kc + k], r1 = T.res[ro + 1][kc + k];
            const float c0 = T.chunk[co][k], c1 = T.chunk[co + 1][k];
            acc[0][0] = fmaf(r0, c0, acc[0][0]);
            acc[0][1] = fmaf(r0, c1, acc[0][1]);
            acc[1][0] = fmaf(r1, c0, acc[1][0]);
            acc[1][1] = fmaf(r1, c1, acc[1][1]);
        }
    }
}

// The logit of (source row i, target row j) of the tile after the ignore mask: -inf outside the pair, and for a
// target strictly inside r_n that is not the positive.
__device__ __forceinline__ float masked(const Tile& T, float s, int i, int j, int n_i, int n_j, int j_global, double rn2) {
    if (i >= n_i || j >= n_j) return -INFINITY;
    if (j_global != T.pos[i] && dist2(T.gt[i], T.txyz[j]) < rn2) return -INFINITY;
    return s;
}

__device__ __forceinline__ void load_src_meta(Tile& T, const regtr_loss_args& a, int i0, int n_i) {
    if (threadIdx.x < TM) {
        const int r = threadIdx.x;
        const bool ok = r < n_i;
        T.pos[r] = ok ? a.pos[i0 + r] : -1;
        for (int j = 0; j < 3; ++j) T.gt[r][j] = ok ? a.src_gt[3 * (long long)(i0 + r) + j] : 0.f;
    }
}

__device__ __forceinline__ void load_tgt_meta(Tile& T, const regtr_loss_args& a, int j0, int n_j) {
    if (threadIdx.x >= 32 && threadIdx.x < 32 + TM) {
        const int r = threadIdx.x - 32;
        for (int j = 0; j < 3; ++j) T.txyz[r][j] = r < n_j ? a.xyz[3 * (long long)(j0 + r) + j] : 0.f;
    }
}

// Gradient weight c_i of a source row: anchor / (anchors of the pair * B) times the upstream gradient of the term.
__device__ __forceinline__ void load_src_grad(Tile& T, const regtr_loss_args& a, int term, int b, int i0, int n_i) {
    if (threadIdx.x >= 64 && threadIdx.x < 64 + TM) {
        const int r = threadIdx.x - 64;
        float c = 0.f, lse = 0.f;
        if (r < n_i && a.anchor[i0 + r]) {
            c = (float)((double)a.g[a.term_val[term]] / ((double)a.n_anchor[b] * (double)a.B));
            lse = a.lse[(long long)term * a.N + i0 + r];
        }
        T.c[r] = c;
        T.lse[r] = lse;
    }
}

__device__ __forceinline__ float grad_weight(const Tile& T, float s, int i, int j_global) {
    if (T.c[i] == 0.f || s == -INFINITY) return 0.f;
    return T.c[i] * (expf(s - T.lse[i]) - (j_global == T.pos[i] ? 1.f : 0.f));
}

__global__ void __launch_bounds__(256) k_infonce_fwd(const regtr_loss_args a) {
    __shared__ Tile T;
    const int term = blockIdx.z, b = blockIdx.y;
    const int s0 = a.offs[b], t0 = a.offs[a.B + b], n_t = a.offs[a.B + b + 1] - t0;
    const int i0 = s0 + blockIdx.x * TM, n_i = min(TM, a.offs[b + 1] - i0);
    if (n_i <= 0) return;
    const int ro = 2 * (threadIdx.x >> 4), co = 2 * (threadIdx.x & 15);
    load_resident(T, a.q[term] + (long long)i0 * D, n_i);
    load_src_meta(T, a, i0, n_i);
    float m = -INFINITY, spos = 0.f;                            // of row threadIdx.x (threads < TM)
    double sum = 0.0;                                           // fp64: ~600 sequential adds must not cost the lse bits
    for (int j0 = 0; j0 < n_t; j0 += TM) {
        const int n_j = min(TM, n_t - j0);
        __syncthreads();
        load_tgt_meta(T, a, t0 + j0, n_j);
        float acc[2][2];
        tile_dots(T, a.feat[term] + (long long)(t0 + j0) * D, n_j, acc);
        for (int u = 0; u < 2; ++u)
            for (int v = 0; v < 2; ++v)
                T.s[ro + u][co + v] = masked(T, acc[u][v], ro + u, co + v, n_i, n_j, t0 + j0 + co + v, a.rn2);
        __syncthreads();
        if (threadIdx.x < n_i) {
            const int r = threadIdx.x;
            float mt = -INFINITY;
            for (int j = 0; j < n_j; ++j) mt = fmaxf(mt, T.s[r][j]);
            if (mt > -INFINITY) {
                const float mn = fmaxf(m, mt);
                sum *= (double)expf(m - mn);
                for (int j = 0; j < n_j; ++j) sum += (double)expf(T.s[r][j] - mn);
                m = mn;
            }
            const int pj = T.pos[r] - (t0 + j0);
            if (pj >= 0 && pj < n_j) spos = T.s[r][pj];
        }
    }
    if (threadIdx.x < n_i) {
        const int r = threadIdx.x;
        const float lse = (float)((double)m + log(sum));
        a.lse[(long long)term * a.N + i0 + r] = lse;
        a.row_loss[(long long)term * a.N + i0 + r] = T.pos[r] >= 0 ? lse - spos : 0.f;
    }
}

// dQ = G P, one CTA per tile of source rows; thread c owns channel c of all its rows.
__global__ void __launch_bounds__(256) k_infonce_bwd_src(const regtr_loss_args a) {
    __shared__ Tile T;
    const int term = blockIdx.z, b = blockIdx.y;
    const int s0 = a.offs[b], t0 = a.offs[a.B + b], n_t = a.offs[a.B + b + 1] - t0;
    const int i0 = s0 + blockIdx.x * TM, n_i = min(TM, a.offs[b + 1] - i0);
    if (n_i <= 0) return;
    const int ro = 2 * (threadIdx.x >> 4), co = 2 * (threadIdx.x & 15), ch = threadIdx.x;
    load_resident(T, a.q[term] + (long long)i0 * D, n_i);
    load_src_meta(T, a, i0, n_i);
    load_src_grad(T, a, term, b, i0, n_i);
    float out[TM];
#pragma unroll
    for (int r = 0; r < TM; ++r) out[r] = 0.f;
    for (int j0 = 0; j0 < n_t; j0 += TM) {
        const int n_j = min(TM, n_t - j0);
        __syncthreads();
        load_tgt_meta(T, a, t0 + j0, n_j);
        float acc[2][2];
        const float* P = a.feat[term] + (long long)(t0 + j0) * D;
        tile_dots(T, P, n_j, acc);
        for (int u = 0; u < 2; ++u)
            for (int v = 0; v < 2; ++v) {
                const int jg = t0 + j0 + co + v;
                T.s[ro + u][co + v] = grad_weight(T, masked(T, acc[u][v], ro + u, co + v, n_i, n_j, jg, a.rn2), ro + u, jg);
            }
        __syncthreads();
        for (int j = 0; j < n_j; ++j) {
            const float p = P[(long long)j * D + ch];
#pragma unroll
            for (int r = 0; r < TM; ++r) out[r] = fmaf(T.s[r][j], p, out[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < TM; ++r)
        if (r < n_i) a.dq[term][(long long)(i0 + r) * D + ch] = out[r];
}

// dP = G^T Q, one CTA per tile of target rows, written into the term's packed feature gradient.
__global__ void __launch_bounds__(256) k_infonce_bwd_tgt(const regtr_loss_args a) {
    __shared__ Tile T;
    const int term = blockIdx.z, b = blockIdx.y;
    const int s0 = a.offs[b], n_s = a.offs[b + 1] - s0, t0 = a.offs[a.B + b];
    const int j0 = t0 + blockIdx.x * TM, n_j = min(TM, a.offs[a.B + b + 1] - j0);
    if (n_j <= 0) return;
    const int ro = 2 * (threadIdx.x >> 4), co = 2 * (threadIdx.x & 15), ch = threadIdx.x;
    load_resident(T, a.feat[term] + (long long)j0 * D, n_j);
    load_tgt_meta(T, a, j0, n_j);
    float out[TM];
#pragma unroll
    for (int r = 0; r < TM; ++r) out[r] = 0.f;
    for (int i0 = 0; i0 < n_s; i0 += TM) {
        const int n_i = min(TM, n_s - i0);
        __syncthreads();
        load_src_meta(T, a, s0 + i0, n_i);
        load_src_grad(T, a, term, b, s0 + i0, n_i);
        float acc[2][2];                                          // [target ro + u][source co + v]
        const float* Q = a.q[term] + (long long)(s0 + i0) * D;
        tile_dots(T, Q, n_i, acc);
        for (int u = 0; u < 2; ++u)
            for (int v = 0; v < 2; ++v) {
                const int jg = j0 + ro + u;
                T.s[co + v][ro + u] = grad_weight(T, masked(T, acc[u][v], co + v, ro + u, n_i, n_j, jg, a.rn2), co + v, jg);
            }
        __syncthreads();
        for (int i = 0; i < n_i; ++i) {
            const float q = Q[(long long)i * D + ch];
#pragma unroll
            for (int r = 0; r < TM; ++r) out[r] = fmaf(T.s[i][r], q, out[r]);
        }
    }
#pragma unroll
    for (int r = 0; r < TM; ++r)
        if (r < n_j) a.dfeat[term][(long long)(j0 + r) * D + ch] = out[r];
}

// ---------------------------------------------------------------------------------------------- loss values

__global__ void k_loss_finalize(const regtr_loss_args a, int n_chunks) {
    for (int b = threadIdx.x; b < a.B; b += blockDim.x) {
        int n = 0;
        for (int i = a.offs[b]; i < a.offs[b + 1]; ++i) n += a.anchor[i];
        a.n_anchor[b] = n;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < a.n_terms * a.B; e += blockDim.x) {
        const int t = e / a.B, b = e - t * a.B;
        double s = 0.0;
        for (int i = a.offs[b]; i < a.offs[b + 1]; ++i)
            if (a.anchor[i]) s += (double)a.row_loss[(long long)t * a.N + i];
        a.pair_loss[e] = s / (double)a.n_anchor[b];               // no anchor: 0 / 0 = NaN, as the reference
    }
    __syncthreads();
    for (int t = threadIdx.x; t < a.n_terms; t += blockDim.x) {
        double s = 0.0;
        for (int b = 0; b < a.B; ++b) s += a.pair_loss[t * a.B + b];
        a.vals[a.term_val[t]] = (float)(s / (double)a.B);
    }
    const double* den = a.ws + (long long)a.L * n_chunks * 3;
    for (int l = threadIdx.x; l < a.L; l += blockDim.x) {
        double bce = 0.0, es = 0.0, et = 0.0;
        for (int c = 0; c < n_chunks; ++c) {
            const double* p = a.ws + ((long long)l * n_chunks + c) * 3;
            bce += p[0]; es += p[1]; et += p[2];
        }
        if (a.ov_val[l] >= 0) a.vals[a.ov_val[l]] = (float)(bce / (double)a.N);
        if (a.corr_val[l] >= 0) a.vals[a.corr_val[l]] = (float)(es / den[0] + et / den[1]);
    }
}

int check_args(const regtr_loss_args* args) {
    if (!args) return REGTR_ERR_ARG;
    const regtr_loss_args& a = *args;
    if (a.N < 0 || a.B < 1 || a.L < 0 || a.L > REGTR_LOSS_MAX_LAYERS || a.n_terms < 0 ||
        a.n_terms > REGTR_LOSS_MAX_TERMS || a.max_src < 0 || a.max_tgt < 0 || !a.offs)
        return REGTR_ERR_ARG;
    return REGTR_OK;
}

int n_chunks_of(int N) { return N > 0 ? regtr_cdiv(N, PW) : 0; }

}  // namespace

extern "C" {

int regtr_overlap_pyramid(const regtr_overlap_pyr_args* args, void* stream_) {
    if (!args || args->n_levels < 1 || args->n_levels > REGTR_LOSS_MAX_LEVELS) return REGTR_ERR_ARG;
    for (int p = 1; p < args->n_levels; ++p) {
        if (args->n[p] < 0 || args->K[p] < 1 || !args->n_prev[p] || !args->pyr[p - 1]) return REGTR_ERR_ARG;
        if (args->n[p] == 0) continue;
        if (!args->pool[p] || !args->pyr[p]) return REGTR_ERR_ARG;
        k_overlap_level<<<regtr_cdiv(args->n[p], 256), 256, 0, (cudaStream_t)stream_>>>(
            args->pyr[p - 1], args->pool[p], args->K[p], args->n[p], args->n_prev[p], args->pyr[p]);
        REGTR_CHECK_LAUNCH();
    }
    return REGTR_OK;
}

int regtr_sym_weight(const float* W, float* Ws_hi, float* Ws_lo, void* stream_) {
    if (!W || !Ws_hi || !Ws_lo) return REGTR_ERR_ARG;
    k_sym_weight<<<D, D, 0, (cudaStream_t)stream_>>>(W, Ws_hi, Ws_lo);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_sym_weight_bwd(const float* dWs, float* dW, void* stream_) {
    if (!dWs || !dW) return REGTR_ERR_ARG;
    k_sym_weight_bwd<<<D, D, 0, (cudaStream_t)stream_>>>(dWs, dW);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_loss_ws_bytes(int N, int L) {
    return regtr_align(((size_t)(L > 0 ? L : 0) * n_chunks_of(N) * 3 + 2) * sizeof(double));
}

int regtr_loss_pointwise(const regtr_loss_args* args, void* stream_) {
    const int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (a.N == 0 || a.L == 0) return REGTR_OK;
    if (!a.xyz || !a.pose || !a.w || !a.logit || !a.corr || !a.dlogit || !a.dcorr || !a.ws) return REGTR_ERR_ARG;
    if (a.ws_bytes < regtr_loss_ws_bytes(a.N, a.L)) return REGTR_ERR_WORKSPACE;
    k_loss_pointwise<<<dim3(n_chunks_of(a.N), a.L), PW, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_loss_pointwise_bwd(const regtr_loss_args* args, void* stream_) {
    const int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (a.N == 0 || a.L == 0) return REGTR_OK;
    if (!a.g || !a.dlogit || !a.dcorr || !a.dlogit_out || !a.dcorr_out) return REGTR_ERR_ARG;
    k_loss_scale<<<regtr_cdiv((long long)a.L * a.N, 256), 256, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_infonce_match(const regtr_loss_args* args, void* stream_) {
    const int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (a.max_src == 0) return REGTR_OK;
    if (!a.xyz || !a.pose || !a.src_gt || !a.pos || !a.anchor) return REGTR_ERR_ARG;
    k_infonce_match<<<dim3(regtr_cdiv(a.max_src, 128), a.B), 128, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

static int check_terms(const regtr_loss_args& a, bool bwd) {
    if (!a.xyz || !a.src_gt || !a.pos || !a.anchor || !a.lse) return REGTR_ERR_ARG;
    for (int t = 0; t < a.n_terms; ++t) {
        if (!a.q[t] || !a.feat[t] || a.term_val[t] < 0 || a.term_val[t] >= a.n_vals) return REGTR_ERR_ARG;
        if (bwd && (!a.dq[t] || !a.dfeat[t])) return REGTR_ERR_ARG;
    }
    return REGTR_OK;
}

int regtr_infonce_fwd(const regtr_loss_args* args, void* stream_) {
    int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (a.n_terms == 0 || a.max_src == 0) return REGTR_OK;
    if ((rc = check_terms(a, false)) || !a.row_loss) return REGTR_ERR_ARG;
    k_infonce_fwd<<<dim3(regtr_cdiv(a.max_src, TM), a.B, a.n_terms), 256, 0, (cudaStream_t)stream_>>>(a);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_infonce_bwd(const regtr_loss_args* args, void* stream_) {
    int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (a.n_terms == 0) return REGTR_OK;
    if ((rc = check_terms(a, true)) || !a.g || !a.n_anchor) return REGTR_ERR_ARG;
    if (a.max_src > 0) {
        k_infonce_bwd_src<<<dim3(regtr_cdiv(a.max_src, TM), a.B, a.n_terms), 256, 0, (cudaStream_t)stream_>>>(a);
        REGTR_CHECK_LAUNCH();
    }
    if (a.max_tgt > 0) {
        k_infonce_bwd_tgt<<<dim3(regtr_cdiv(a.max_tgt, TM), a.B, a.n_terms), 256, 0, (cudaStream_t)stream_>>>(a);
        REGTR_CHECK_LAUNCH();
    }
    return REGTR_OK;
}

int regtr_loss_finalize(const regtr_loss_args* args, void* stream_) {
    const int rc = check_args(args);
    if (rc) return rc;
    const regtr_loss_args& a = *args;
    if (!a.vals || !a.anchor || !a.n_anchor || !a.pair_loss || !a.row_loss || !a.ws) return REGTR_ERR_ARG;
    if (a.ws_bytes < regtr_loss_ws_bytes(a.N, a.L)) return REGTR_ERR_WORKSPACE;
    for (int l = 0; l < a.L; ++l)
        if (a.ov_val[l] >= a.n_vals || a.corr_val[l] >= a.n_vals) return REGTR_ERR_ARG;
    k_loss_finalize<<<1, 256, 0, (cudaStream_t)stream_>>>(a, n_chunks_of(a.N));
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
