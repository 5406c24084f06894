// Backward kernels of the cross-encoder and the correspondence heads (training / fine-tuning path):
//   attention core, varlen, head_dim 32      -- FlashAttention-2 recurrence, softmax recomputed from the forward's lse
//   LayerNorm (+ position add) backward      -- transformers.py:117-119, 194-232
//   dense-layer weight gradient + ReLU mask  -- nn.Linear / nn.ReLU backward
// (paths relative to /root/reference/src).  Every reduction runs in a fixed order with no atomics: two backward
// passes over the same inputs are bit-identical.
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int HD = 32;        // head dim
constexpr int BT = 64;        // keys (dK/dV pass) or queries (dQ pass) per block: one row per thread
constexpr int CH = 32;        // rows of the other operand staged per shared-memory chunk
constexpr float LN2 = 0.6931471805599453f;

__device__ __forceinline__ float fast_exp2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__device__ __forceinline__ void load_row(const float* __restrict__ p, float (&r)[HD], float s = 1.f) {
#pragma unroll
    for (int d = 0; d < HD / 4; ++d) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p) + d);
        r[4 * d] = t.x * s; r[4 * d + 1] = t.y * s; r[4 * d + 2] = t.z * s; r[4 * d + 3] = t.w * s;
    }
}

__device__ __forceinline__ float dot_smem(const float (&a)[HD], const float* __restrict__ b) {
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < HD / 4; ++d) {
        const float4 t = reinterpret_cast<const float4*>(b)[d];
        s = fmaf(a[4 * d], t.x, s); s = fmaf(a[4 * d + 1], t.y, s);
        s = fmaf(a[4 * d + 2], t.z, s); s = fmaf(a[4 * d + 3], t.w, s);
    }
    return s;
}

__device__ __forceinline__ void axpy_smem(float (&acc)[HD], float a, const float* __restrict__ b) {
#pragma unroll
    for (int d = 0; d < HD / 4; ++d) {
        const float4 t = reinterpret_cast<const float4*>(b)[d];
        acc[4 * d] = fmaf(a, t.x, acc[4 * d]); acc[4 * d + 1] = fmaf(a, t.y, acc[4 * d + 1]);
        acc[4 * d + 2] = fmaf(a, t.z, acc[4 * d + 2]); acc[4 * d + 3] = fmaf(a, t.w, acc[4 * d + 3]);
    }
}

__device__ __forceinline__ void store_row(float* __restrict__ p, const float (&r)[HD], float s) {
#pragma unroll
    for (int d = 0; d < HD / 4; ++d)
        reinterpret_cast<float4*>(p)[d] = make_float4(r[4 * d] * s, r[4 * d + 1] * s, r[4 * d + 2] * s, r[4 * d + 3] * s);
}

// keys / values [r0, r0 + nk) of one head into shared memory
__device__ __forceinline__ void stage_kv(float (&sK)[CH][HD], float (&sV)[CH][HD], const float* __restrict__ Kp, int ldk,
                                         const float* __restrict__ Vp, int ldv, size_t r0, int nk, int col) {
    for (int f = threadIdx.x; f < nk * (HD / 4); f += BT) {
        const int r = f >> 3, c4 = f & 7;
        reinterpret_cast<float4*>(&sK[r][0])[c4] =
            __ldg(reinterpret_cast<const float4*>(Kp + (r0 + r) * ldk + col) + c4);
        reinterpret_cast<float4*>(&sV[r][0])[c4] =
            __ldg(reinterpret_cast<const float4*>(Vp + (r0 + r) * ldv + col) + c4);
    }
}

// s + c += x with the rounding error of the add carried in c (Knuth's TwoSum: exact for any order of magnitudes)
__device__ __forceinline__ void two_sum_add(float& s, float& c, float x) {
    const float t = __fadd_rn(s, x), b = __fsub_rn(t, s);       // _rn: never contracted into an FMA
    c = __fadd_rn(c, __fadd_rn(__fsub_rn(s, __fsub_rn(t, b)), __fsub_rn(x, b)));
    s = t;
}

// ---- attention backward ------------------------------------------------------------------------------------------
// Scores are recomputed exactly as the forward (k_mha_tf32x3) scales them: s = (q * scale*log2e) . k, in base 2, and
// p = exp2(s - lse) with the forward's ex2.approx.  The dot products run in fp32 FMA chains (round-to-nearest at every
// step), which is at least as accurate as the forward's 3xTF32 tensor-core products.
//
// The softmax is made self-consistent in the backward's own arithmetic.  The forward's lse comes from 3xTF32 scores,
// so sum_k p differs from 1 by about |s| * 1e-7, and rowsum(dO * O) from the forward's O differs from sum_k P dP by
// as much.  Neither cancels in sum_k dS, and dQ / dK pick that error up multiplied by whatever k / q share (the
// in-projection bias: softmax ignores a vector added to every key, so sum_k dK = 0 and dQ does not change).  So
// pass 1 first sweeps the keys: Z = sum_k p and D = sum_k p dP, both compensated sums, give the normalised
// P = p / Z and delta = D / Z = sum_k P dP from the very p and dP both passes use.
//
// Pass 1 (this kernel): block = (64-query tile, head, problem), one query per thread; keys stream through shared
// memory, twice.  dS = P * (dP - delta) with dP = dO . v;  dQ = scale * sum_k dS k.  delta and 1 / Z are stored for
// pass 2.  Every query row belongs to exactly one problem, so every dQ row is written exactly once.  A problem with an
// empty key range has Z = 0 and writes dQ = 0.
// DROP (attention-probability dropout, the regtr_mha_varlen_fwd forward with a dropout key): dP = dO . v becomes
// g = m * scale * dP in both sweeps, so D = sum_k p g and delta = D / Z are formed from the very g the second sweep
// uses and sum_k dS = 0 still holds in this arithmetic.  The 8 threads of an aligned 8-query group share one Philox
// block per key: per 8 keys each draws the block of one key and the bits are passed round with one shuffle per key.
template <bool DROP>
__global__ void __launch_bounds__(BT)
k_mha_bwd_dq(const float* __restrict__ Q, int ldq, const float* __restrict__ Kp, int ldk, const float* __restrict__ Vp,
             int ldv, const float* __restrict__ dO, int lddo, const float* __restrict__ lse, float* __restrict__ delta,
             float* __restrict__ rnorm, float* __restrict__ dQ, int lddq, const int32_t* __restrict__ q_start,
             const int32_t* __restrict__ q_len, const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len,
             float qscale, float scale, DropKey drop) {
    __shared__ __align__(16) float sK[CH][HD], sV[CH][HD];
    const int prob = blockIdx.z, head = blockIdx.y, tile = blockIdx.x, nh = gridDim.y;
    const int ql = q_len[prob];
    if (tile * BT >= ql) return;
    const int q0 = q_start[prob], k0 = k_start[prob], kl = k_len[prob];
    const int qi = tile * BT + threadIdx.x;
    const bool active = qi < ql;
    const size_t row = (size_t)q0 + min(qi, ql - 1);
    const int col = head * HD;

    float q[HD], g[HD], acc[HD];
    load_row(Q + row * ldq + col, q, qscale);
    load_row(dO + row * lddo + col, g);
    const float L = lse[row * nh + head];

    // compensated sums (TwoSum, and TwoProduct for p * dP): Z and D to about one rounding, whatever the key count
    float z = 0.f, zc = 0.f, dsum = 0.f, dc = 0.f;
    if constexpr (DROP) {
        const unsigned w1 = drop_word1(drop, prob, head), rg = (unsigned)qi >> 3, u = threadIdx.x & 7;
        const int gl = threadIdx.x & 24;                 // first lane of this thread's 8-query group
        for (int kb = 0; kb < kl; kb += CH) {
            const int nk = min(CH, kl - kb);
            __syncthreads();
            stage_kv(sK, sV, Kp, ldk, Vp, ldv, (size_t)(k0 + kb), nk, col);
            __syncthreads();
            for (int j0 = 0; j0 < nk; j0 += 8) {
                const unsigned mine = drop_keep8(drop, w1, rg, (unsigned)(kb + j0) + u);
                for (int jj = 0; jj < 8 && j0 + jj < nk; ++jj) {
                    const int j = j0 + jj;
                    const unsigned mb = __shfl_sync(0xffffffffu, mine, gl | jj);
                    const float p = fast_exp2(dot_smem(q, &sK[j][0]) - L);
                    two_sum_add(z, zc, p);
                    const float dp = ((mb >> u) & 1u) ? __fmul_rn(dot_smem(g, &sV[j][0]), drop.scale) : 0.f;
                    const float pr = __fmul_rn(p, dp);
                    dc += fmaf(p, dp, -pr);
                    two_sum_add(dsum, dc, pr);
                }
            }
        }
        z += zc;
        dsum += dc;
        const float rz = z > 0.f ? 1.f / z : 0.f;
        const float dl = z > 0.f ? dsum / z : 0.f;
        if (active) { delta[row * nh + head] = dl; rnorm[row * nh + head] = rz; }
#pragma unroll
        for (int d = 0; d < HD; ++d) acc[d] = 0.f;
        for (int kb = 0; kb < kl; kb += CH) {
            const int nk = min(CH, kl - kb);
            __syncthreads();
            stage_kv(sK, sV, Kp, ldk, Vp, ldv, (size_t)(k0 + kb), nk, col);
            __syncthreads();
            for (int j0 = 0; j0 < nk; j0 += 8) {
                const unsigned mine = drop_keep8(drop, w1, rg, (unsigned)(kb + j0) + u);
                for (int jj = 0; jj < 8 && j0 + jj < nk; ++jj) {
                    const int j = j0 + jj;
                    const unsigned mb = __shfl_sync(0xffffffffu, mine, gl | jj);
                    const float p = fast_exp2(dot_smem(q, &sK[j][0]) - L);
                    const float dp = ((mb >> u) & 1u) ? __fmul_rn(dot_smem(g, &sV[j][0]), drop.scale) : 0.f;
                    axpy_smem(acc, p * (dp - dl), &sK[j][0]);
                }
            }
        }
        if (active) store_row(dQ + (size_t)(q0 + qi) * lddq + col, acc, scale * rz);
        return;
    }
    for (int kb = 0; kb < kl; kb += CH) {
        const int nk = min(CH, kl - kb);
        __syncthreads();
        stage_kv(sK, sV, Kp, ldk, Vp, ldv, (size_t)(k0 + kb), nk, col);
        __syncthreads();
        for (int j = 0; j < nk; ++j) {
            const float p = fast_exp2(dot_smem(q, &sK[j][0]) - L);
            two_sum_add(z, zc, p);
            const float dp = dot_smem(g, &sV[j][0]);
            const float pr = __fmul_rn(p, dp);
            dc += fmaf(p, dp, -pr);
            two_sum_add(dsum, dc, pr);
        }
    }
    z += zc;
    dsum += dc;
    const float rz = z > 0.f ? 1.f / z : 0.f;
    const float dl = z > 0.f ? dsum / z : 0.f;
    if (active) { delta[row * nh + head] = dl; rnorm[row * nh + head] = rz; }

#pragma unroll
    for (int d = 0; d < HD; ++d) acc[d] = 0.f;
    for (int kb = 0; kb < kl; kb += CH) {
        const int nk = min(CH, kl - kb);
        __syncthreads();
        stage_kv(sK, sV, Kp, ldk, Vp, ldv, (size_t)(k0 + kb), nk, col);
        __syncthreads();
        for (int j = 0; j < nk; ++j) {
            const float p = fast_exp2(dot_smem(q, &sK[j][0]) - L);
            const float ds = p * (dot_smem(g, &sV[j][0]) - dl);
            axpy_smem(acc, ds, &sK[j][0]);
        }
    }
    if (active) store_row(dQ + (size_t)(q0 + qi) * lddq + col, acc, scale * rz);
}

// Pass 2: block = (64-key tile, head, problem), one key per thread; the problem's queries stream through shared
// memory.  P = exp2(s - lse) / Z with the same FMA chain for s as pass 1;  dV = sum_q P dO,  dK = scale * sum_q dS q.
// Row ownership (what makes this pass atomic-free): every key row is written by the one problem whose key range
// holds it.  In the self table each token is a key of exactly one problem (its own cloud); in the cross table each
// cloud is the key range of exactly one problem (its partner's).  Callers with other tables must keep the key
// ranges disjoint.  A key range whose problem has no queries gets dK = dV = 0.
// DROP: dV = sum_q m scale P dO and dP -> g = m scale dP; each thread draws one Philox block per 8 queries of its key.
template <bool DROP>
__global__ void __launch_bounds__(BT)
k_mha_bwd_dkv(const float* __restrict__ Q, int ldq, const float* __restrict__ Kp, int ldk, const float* __restrict__ Vp,
              int ldv, const float* __restrict__ dO, int lddo, const float* __restrict__ lse,
              const float* __restrict__ delta, const float* __restrict__ rnorm, float* __restrict__ dK, int lddk,
              float* __restrict__ dV, int lddv, const int32_t* __restrict__ q_start, const int32_t* __restrict__ q_len,
              const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len, float qscale, float kscale,
              DropKey drop) {
    __shared__ __align__(16) float sQ[CH][HD], sG[CH][HD];
    __shared__ float sL[CH], sD[CH], sR[CH];
    const int prob = blockIdx.z, head = blockIdx.y, tile = blockIdx.x, nh = gridDim.y;
    const int kl = k_len[prob];
    if (tile * BT >= kl) return;
    const int q0 = q_start[prob], ql = q_len[prob], k0 = k_start[prob];
    const int kj = tile * BT + threadIdx.x;
    const bool active = kj < kl;
    const size_t row = (size_t)k0 + min(kj, kl - 1);
    const int col = head * HD;

    float k[HD], v[HD], dk[HD], dv[HD];
    load_row(Kp + row * ldk + col, k);
    load_row(Vp + row * ldv + col, v);
#pragma unroll
    for (int d = 0; d < HD; ++d) { dk[d] = 0.f; dv[d] = 0.f; }

    for (int qb = 0; qb < ql; qb += CH) {
        const int nq = min(CH, ql - qb);
        __syncthreads();
        for (int f = threadIdx.x; f < nq * (HD / 4); f += BT) {
            const int r = f >> 3, c4 = f & 7;
            const size_t qr = (size_t)(q0 + qb + r);
            const float4 t = __ldg(reinterpret_cast<const float4*>(Q + qr * ldq + col) + c4);
            reinterpret_cast<float4*>(&sQ[r][0])[c4] = make_float4(t.x * qscale, t.y * qscale, t.z * qscale, t.w * qscale);
            reinterpret_cast<float4*>(&sG[r][0])[c4] = __ldg(reinterpret_cast<const float4*>(dO + qr * lddo + col) + c4);
        }
        if (threadIdx.x < nq) {
            const size_t qr = (size_t)(q0 + qb + threadIdx.x);
            sL[threadIdx.x] = lse[qr * nh + head];
            sD[threadIdx.x] = delta[qr * nh + head];
            sR[threadIdx.x] = rnorm[qr * nh + head];
        }
        __syncthreads();
        if constexpr (DROP) {
            const unsigned w1 = drop_word1(drop, prob, head);
            for (int i0 = 0; i0 < nq; i0 += 8) {
                const unsigned mb = drop_keep8(drop, w1, (unsigned)(qb + i0) >> 3, (unsigned)kj);
                for (int ii = 0; ii < 8 && i0 + ii < nq; ++ii) {
                    const int i = i0 + ii;
                    const bool keep = (mb >> ii) & 1u;
                    const float p = fast_exp2(dot_smem(k, &sQ[i][0]) - sL[i]) * sR[i];
                    axpy_smem(dv, keep ? __fmul_rn(p, drop.scale) : 0.f, &sG[i][0]);
                    const float dp = keep ? __fmul_rn(dot_smem(v, &sG[i][0]), drop.scale) : 0.f;
                    axpy_smem(dk, p * (dp - sD[i]), &sQ[i][0]);
                }
            }
            continue;
        }
        for (int i = 0; i < nq; ++i) {
            const float p = fast_exp2(dot_smem(k, &sQ[i][0]) - sL[i]) * sR[i];
            axpy_smem(dv, p, &sG[i][0]);
            const float ds = p * (dot_smem(v, &sG[i][0]) - sD[i]);
            axpy_smem(dk, ds, &sQ[i][0]);
        }
    }
    if (!active) return;
    // dk accumulated against q * scale*log2e: dK = scale * sum dS q = ln2 * dk
    store_row(dK + (size_t)(k0 + kj) * lddk + col, dk, kscale);
    store_row(dV + (size_t)(k0 + kj) * lddv + col, dv, 1.f);
}

// ---- LayerNorm backward ------------------------------------------------------------------------------------------
// y = (x - mean) * rstd * g + b (mean / rstd recomputed from x exactly as k_layernorm_pos does);  dy_total = dy + dy_pos;
//   dx = rstd * (dxh - mean(dxh) - xh * mean(dxh * xh)) + dres,   dxh = dy_total * g,   xh = (x - mean) * rstd
//   dg = sum_rows dy_total * xh,   db = sum_rows dy_total
// Block = 8 warps over LNB_ROWS consecutive rows (warp w: rows w, w + 8, ...); each lane keeps its columns' dg / db
// partials, the block adds its 8 warps in order and stores one partial row; k_colsum adds the blocks in order.
constexpr int LNB_WARPS = 8, LNB_ROWS = 64, LN_PER = 8;     // E <= 32 * LN_PER = 256

// DROP (regtr_layernorm_bwd with a dropout key): also dz = dx * m * scale, the gradient of the dropped residual branch.
template <bool DROP>
__global__ void __launch_bounds__(32 * LNB_WARPS)
k_layernorm_bwd(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ dy,
                const float* __restrict__ dyp, const float* __restrict__ dres, int n, int E, float eps,
                float* __restrict__ dx, float* __restrict__ part, float* __restrict__ dz,
                const int32_t* __restrict__ offs, DropKey drop) {
    __shared__ float red[LNB_WARPS][2][32 * LN_PER];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, per = E / 32;
    float gm[LN_PER], ag[LN_PER], ab[LN_PER];
#pragma unroll
    for (int j = 0; j < LN_PER; ++j) { gm[j] = j < per ? __ldg(gamma + j * 32 + lane) : 0.f; ag[j] = 0.f; ab[j] = 0.f; }
    const int r_end = min(n, (blockIdx.x + 1) * LNB_ROWS);
    for (int row = blockIdx.x * LNB_ROWS + warp; row < r_end; row += LNB_WARPS) {
        const size_t o = (size_t)row * E;
        float v[LN_PER], g[LN_PER];
#pragma unroll
        for (int j = 0; j < LN_PER; ++j)
            if (j < per) {
                const int c = j * 32 + lane;
                v[j] = x[o + c];
                g[j] = (dy ? dy[o + c] : 0.f) + (dyp ? dyp[o + c] : 0.f);
            }
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < LN_PER; ++j) if (j < per) s += v[j];
        const float mean = warp_sum(s) / (float)E;
        float ss = 0.f;
#pragma unroll
        for (int j = 0; j < LN_PER; ++j) if (j < per) { const float d = v[j] - mean; ss += d * d; }
        const float rstd = 1.f / sqrtf(warp_sum(ss) / (float)E + eps);
        float s1 = 0.f, s2 = 0.f;
#pragma unroll
        for (int j = 0; j < LN_PER; ++j)
            if (j < per) {
                v[j] = (v[j] - mean) * rstd;                    // x-hat
                const float h = g[j] * gm[j];
                s1 += h; s2 = fmaf(h, v[j], s2);
                ag[j] = fmaf(g[j], v[j], ag[j]); ab[j] += g[j];
            }
        s1 = warp_sum(s1) / (float)E; s2 = warp_sum(s2) / (float)E;
        unsigned w1 = 0, rr = 0;
        if constexpr (DROP) {
            const int c = regtr_cloud_of(offs, 2 * drop.n_pairs, row);
            w1 = drop_word1(drop, c, 0);
            rr = (unsigned)(row - offs[c]);
        }
#pragma unroll
        for (int j = 0; j < LN_PER; ++j)
            if (j < per) {
                const int c = j * 32 + lane;
                float d = rstd * (g[j] * gm[j] - s1 - v[j] * s2);
                if (dres) d += dres[o + c];
                dx[o + c] = d;
                if constexpr (DROP) dz[o + c] = drop_keep(drop, w1, rr, (unsigned)c) ? __fmul_rn(d, drop.scale) : 0.f;
            }
    }
#pragma unroll
    for (int j = 0; j < LN_PER; ++j) { red[warp][0][j * 32 + lane] = ag[j]; red[warp][1][j * 32 + lane] = ab[j]; }
    __syncthreads();
    for (int c = threadIdx.x; c < 2 * E; c += 32 * LNB_WARPS) {
        const int which = c >= E, cc = c - which * E;
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < LNB_WARPS; ++w) t += red[w][which][cc];
        part[(size_t)blockIdx.x * 2 * E + c] = t;
    }
}

// out[c] = sum_b part[b * ld + c] for c < n_cols, b ascending (fixed order)
__global__ void k_colsum(const float* __restrict__ part, int n_blocks, int ld, int n_cols, float* __restrict__ out0,
                         int split, float* __restrict__ out1) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_cols) return;
    float t = 0.f;
    for (int b = 0; b < n_blocks; ++b) t += part[(size_t)b * ld + c];
    if (c < split) out0[c] = t;
    else out1[c - split] = t;
}

// ---- dense layers ----------------------------------------------------------------------------------------------
// dH * scale where H > 0: the ReLU mask applied to an incoming gradient (H = the ReLU's output).  With the
// feed-forward dropout (site 5) H is the dropped ReLU output, positive exactly where the ReLU passed and the mask kept,
// and scale is the dropout's 1 / (1 - p); without it scale = 1 and dh * 1 is dh (no -ftz / fast-math in the build).
__global__ void k_relu_bwd(const float* __restrict__ dh, const float* __restrict__ h, long long n, float scale,
                           float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = h[i] > 0.f ? __fmul_rn(dh[i], scale) : 0.f;
}

__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t u = __float_as_uint(x);
    u += 0x0FFFu + ((u >> 13) & 1u);
    return __uint_as_float(u & 0xFFFFE000u);
}

// Transpose a row-major [M, C] matrix (leading dim ld) into [Cp, Mp] (zero beyond M / C).  SPLIT: write the two TF32
// halves (round-to-nearest, as regtr_split_tf32) of every value; ONES: row C of the output is 1 over the M real
// columns (the bias gradient rides along the weight-gradient GEMM as one more output column).
template <bool SPLIT, bool ONES>
__global__ void k_transpose(const float* __restrict__ X, int ld, int M, int C, int Mp, int Cp, float* __restrict__ hi,
                            float* __restrict__ lo) {
    __shared__ float t[32][33];
    const int m0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int m = m0 + r, c = c0 + threadIdx.x;
        float v = 0.f;
        if (m < M) v = c < C ? X[(size_t)m * ld + c] : (ONES && c == C ? 1.f : 0.f);
        t[r][threadIdx.x] = v;
    }
    __syncthreads();
    for (int r = threadIdx.y; r < 32; r += 8) {
        const int c = c0 + r, m = m0 + threadIdx.x;
        if (c >= Cp || m >= Mp) continue;
        const float v = t[threadIdx.x][r];
        const size_t o = (size_t)c * Mp + m;
        if (SPLIT) { const float h = tf32_rn(v); hi[o] = h; lo[o] = tf32_rn(v - h); }
        else hi[o] = v;
    }
}

// dW[n, k] = C[n, k] (k < K), db[n] = C[n, K]
__global__ void k_wgrad_extract(const float* __restrict__ Cw, int ldc, int N, int K, float* __restrict__ dW,
                                float* __restrict__ db) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)N * (K + 1)) return;
    const int n = (int)(i / (K + 1)), k = (int)(i % (K + 1));
    if (k < K) dW[(size_t)n * K + k] = Cw[(size_t)n * ldc + k];
    else if (db) db[n] = Cw[(size_t)n * ldc + K];
}

struct WgradLayout {
    int Mp, Kp;
    size_t o_xl, o_dyt, o_c, o_gemm, total;
};

WgradLayout wgrad_layout(int M, int N, int K) {
    WgradLayout w;
    w.Mp = (M + 3) & ~3;
    w.Kp = (K + 1 + 3) & ~3;
    const size_t xt = regtr_align((size_t)w.Kp * w.Mp * sizeof(float));
    w.o_xl = xt;
    w.o_dyt = 2 * xt;
    w.o_c = w.o_dyt + regtr_align((size_t)N * w.Mp * sizeof(float));
    w.o_gemm = w.o_c + regtr_align((size_t)N * w.Kp * sizeof(float));
    w.total = w.o_gemm + regtr_gemm_ws_bytes(N, w.Kp, w.Mp);
    return w;
}

}  // namespace

extern "C" {

size_t regtr_mha_varlen_bwd_ws_bytes(int n_rows, int n_heads) {
    return regtr_align(2 * (size_t)(n_rows > 0 ? n_rows : 1) * (size_t)(n_heads > 0 ? n_heads : 1) * sizeof(float));
}

int regtr_mha_varlen_bwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv, const float* O,
                         int ldo, const float* dO, int lddo, const float* lse, float* dQ, int lddq, float* dK, int lddk,
                         float* dV, int lddv, const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                         const int32_t* k_len, int n_problems, int n_rows, int max_q_len, int max_k_len, int n_heads,
                         int head_dim, float scale, const regtr_dropout_args* drop, void* ws, size_t ws_bytes,
                         void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    DropKey dk;
    if (drop && (drop_key_of(drop, dk) != REGTR_OK || n_heads > 16 || 2 * drop->n_pairs != n_problems))
        return REGTR_ERR_ARG;
    if (n_problems < 0 || n_rows < 0 || max_q_len < 0 || max_k_len < 0 || n_heads <= 0) return REGTR_ERR_ARG;
    if (head_dim != HD) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || n_rows == 0) return REGTR_OK;
    if (!Q || !K || !V || !O || !dO || !lse || !dQ || !dK || !dV || !q_start || !q_len || !k_start || !k_len)
        return REGTR_ERR_ARG;
    if ((ldq | ldk | ldv | ldo | lddo | lddq | lddk | lddv) % 4 != 0 || n_problems > 65535 || n_heads > 65535)
        return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_mha_varlen_bwd_ws_bytes(n_rows, n_heads)) return REGTR_ERR_WORKSPACE;
    float* delta = (float*)ws;
    float* rnorm = delta + (size_t)n_rows * n_heads;
    const float qscale = scale * 1.4426950408889634f;
    if (max_q_len > 0) {
        const dim3 grid(regtr_cdiv(max_q_len, BT), n_heads, n_problems);
        if (drop)
            k_mha_bwd_dq<true><<<grid, BT, 0, st>>>(Q, ldq, K, ldk, V, ldv, dO, lddo, lse, delta, rnorm, dQ, lddq, q_start,
                                                    q_len, k_start, k_len, qscale, scale, dk);
        else
            k_mha_bwd_dq<false><<<grid, BT, 0, st>>>(Q, ldq, K, ldk, V, ldv, dO, lddo, lse, delta, rnorm, dQ, lddq, q_start,
                                                     q_len, k_start, k_len, qscale, scale, DropKey{});
        REGTR_CHECK_LAUNCH();
    }
    if (max_k_len > 0) {
        const dim3 grid(regtr_cdiv(max_k_len, BT), n_heads, n_problems);
        if (drop)
            k_mha_bwd_dkv<true><<<grid, BT, 0, st>>>(Q, ldq, K, ldk, V, ldv, dO, lddo, lse, delta, rnorm, dK, lddk, dV,
                                                     lddv, q_start, q_len, k_start, k_len, qscale, LN2, dk);
        else
            k_mha_bwd_dkv<false><<<grid, BT, 0, st>>>(Q, ldq, K, ldk, V, ldv, dO, lddo, lse, delta, rnorm, dK, lddk, dV,
                                                      lddv, q_start, q_len, k_start, k_len, qscale, LN2, DropKey{});
        REGTR_CHECK_LAUNCH();
    }
    return REGTR_OK;
}

size_t regtr_layernorm_bwd_ws_bytes(int n, int E) {
    return regtr_align((size_t)regtr_cdiv(n > 0 ? n : 1, LNB_ROWS) * 2 * (size_t)(E > 0 ? E : 1) * sizeof(float));
}

int regtr_layernorm_bwd(const float* x, const float* gamma, const float* dy, const float* dy_pos, const float* dres,
                        int n, const int32_t* offs, int E, float eps, float* dx, float* dz, float* dgamma, float* dbeta,
                        const regtr_dropout_args* drop, void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs != !drop || !dz != !drop) return REGTR_ERR_ARG;            // offs, dz and drop come together
    DropKey dk;
    if (drop && drop_key_of(drop, dk) != REGTR_OK) return REGTR_ERR_ARG;
    if (n < 0 || E <= 0 || E % 32 != 0) return REGTR_ERR_ARG;
    if (E > 32 * LN_PER) return REGTR_ERR_UNSUPPORTED;
    // n = 0 (empty tensors, null pointers) still writes dgamma = dbeta = 0
    if (!gamma || !dgamma || !dbeta || (n > 0 && (!x || !dx))) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_layernorm_bwd_ws_bytes(n, E)) return REGTR_ERR_WORKSPACE;
    float* part = (float*)ws;
    const int nb = n > 0 ? regtr_cdiv(n, LNB_ROWS) : 0;
    if (nb > 0) {
        if (drop)
            k_layernorm_bwd<true><<<nb, 32 * LNB_WARPS, 0, st>>>(x, gamma, dy, dy_pos, dres, n, E, eps, dx, part, dz, offs,
                                                                 dk);
        else
            k_layernorm_bwd<false><<<nb, 32 * LNB_WARPS, 0, st>>>(x, gamma, dy, dy_pos, dres, n, E, eps, dx, part, nullptr,
                                                                  nullptr, DropKey{});
        REGTR_CHECK_LAUNCH();
    }
    k_colsum<<<regtr_cdiv(2 * E, 256), 256, 0, st>>>(part, nb, 2 * E, 2 * E, dgamma, E, dbeta);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_relu_bwd(const float* dh, const float* h, long long n, float scale, float* out, void* stream_) {
    if (n < 0) return REGTR_ERR_ARG;
    if (n == 0) return REGTR_OK;
    if (!dh || !h || !out) return REGTR_ERR_ARG;
    k_relu_bwd<<<regtr_cdiv(n, 256), 256, 0, (cudaStream_t)stream_>>>(dh, h, n, scale, out);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_linear_wgrad_ws_bytes(int M, int N, int K) {
    return wgrad_layout(M > 0 ? M : 1, N > 0 ? N : 1, K > 0 ? K : 1).total;
}

// dW[N,K] = dY^T X and db[N] = sum_rows dY as ONE 3xTF32 GEMM on regtr_gemm_tf32x3: wgmma takes TF32 operands
// K-major only, and for this product the reduction runs over the rows of X and dY, so both are first transposed
// (X^T also split into its TF32 halves, plus a row of ones that yields db as column K of the product).  The GEMM's
// split-K over the long token dimension is deterministic (fixed-order plane sums).
int regtr_linear_wgrad(const float* X, int ldx, const float* dY, int ldy, int M, int N, int K, float* dW, float* db,
                       void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (M < 0 || N <= 0 || K <= 0 || (M > 0 && (ldx < K || ldy < N))) return REGTR_ERR_ARG;
    if (!dW || (M > 0 && (!X || !dY))) return REGTR_ERR_ARG;      // no tokens: dW = 0, db = 0, X and dY unread
    const WgradLayout w = wgrad_layout(M > 0 ? M : 1, N, K);
    if (!ws || ((uintptr_t)ws & 255) || ws_bytes < w.total) return REGTR_ERR_WORKSPACE;
    char* base = (char*)ws;
    float *xh = (float*)base, *xl = (float*)(base + w.o_xl), *dyt = (float*)(base + w.o_dyt), *cw = (float*)(base + w.o_c);
    const dim3 blk(32, 8);
    k_transpose<true, true><<<dim3(regtr_cdiv(w.Mp, 32), regtr_cdiv(w.Kp, 32)), blk, 0, st>>>(X, ldx, M, K, w.Mp, w.Kp, xh, xl);
    REGTR_CHECK_LAUNCH();
    k_transpose<false, false><<<dim3(regtr_cdiv(w.Mp, 32), regtr_cdiv(N, 32)), blk, 0, st>>>(dY, ldy, M, N, w.Mp, N, dyt, nullptr);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_gemm_tf32x3(dyt, w.Mp, xh, xl, w.Mp, cw, w.Kp, nullptr, nullptr, 0, N, w.Kp, w.Mp, nullptr, 0,
                                     base + w.o_gemm, w.total - w.o_gemm, stream_);
    if (rc != REGTR_OK) return rc;
    k_wgrad_extract<<<regtr_cdiv((long long)N * (K + 1), 256), 256, 0, st>>>(cw, w.Kp, N, K, dW, db);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
