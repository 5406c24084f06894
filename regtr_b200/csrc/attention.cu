// Variable-length multi-head attention core, fp32-accurate parity path (mma.sync 3xTF32).
//
// Replaces the softmax(QK^T/sqrt(d))V core of nn.MultiheadAttention as called by
// TransformerCrossEncoderLayer.forward_pre (/root/reference/src/models/transformer/
// transformers.py:197-226).  The reference pads sequences to a common length and masks
// padded keys with -inf; here every (query range, key range) problem is explicit, which is
// equivalent because masked keys receive exactly zero weight.

#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int HD = 32;        // head dim

// linear tile index -> (problem, tile inside the problem); false beyond the last tile
__device__ __forceinline__ bool find_tile(const int32_t* __restrict__ tile_base, int n_prob, int& prob, int& tile) {
    if (tile >= tile_base[n_prob]) return false;
    int p = 0;
    while (p + 1 < n_prob && tile_base[p + 1] <= tile) ++p;
    prob = p;
    tile -= tile_base[p];
    return true;
}

// ---- tensor-core fp32-accurate core --------------------------------------------------------------
// Flash-attention on mma.sync m16n8k8 TF32 with the 3xTF32 split (x = hi + lo; hi*hi + hi*lo + lo*hi in
// fp32 accumulators), so scores and outputs keep fp32 accuracy while the 2 x 32 MACs per (query, key)
// run on the tensor cores.  Block = (problem, head, 64 queries): 4 warps x 16 query rows; keys stream
// through shared memory in chunks of 64, already split into hi/lo halves once per block.
//   S = Q K^T:  A = Q fragment (registers, pre-scaled by scale*log2e, split once), B = K[key g][d]
//   online softmax on the C fragments (rows g, g+8; quad shuffles for the row maxima; row sums stay
//   lane-local until the end)
//   O += P V:   the C fragment of S is reused as the A fragment of P under the key permutation
//               (A column t <-> key 2t, column t+4 <-> key 2t+1); B = V[key][d] with the same permutation.
// Row stride 36 floats makes every fragment LDS bank-conflict free.
// DROP (training with the attention-probability dropout, regtr_mha_varlen_fwd with a dropout key): the keep mask
// multiplies the P fragments in registers before the split for P V, and the output normalisation carries the dropout
// scale; the row sums l (hence lse) stay those of the undropped probabilities.  Per 64-key chunk every lane draws the
// blocks of key kb + lane and kb + 32 + lane for the warp's two 8-row groups (4 Philox blocks), and each lane fetches
// the bits of its two keys per n-tile with two shuffles.
constexpr int MQ = 64, MK = 64, MLD = 36;

__device__ __forceinline__ uint32_t tf32_head(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float fast_exp2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

template <bool DROP>
__global__ void __launch_bounds__(128)
k_mha_tf32x3(const float* __restrict__ Q, int ldq, const float* __restrict__ Kp, int ldk, const float* __restrict__ Vp,
             int ldv, float* __restrict__ O, int ldo, const int32_t* __restrict__ q_start,
             const int32_t* __restrict__ q_len, const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len,
             const int32_t* __restrict__ tile_base, int n_prob, float scale, float* __restrict__ lse, DropKey drop) {
    __shared__ __align__(16) float sKh[MK][MLD], sKl[MK][MLD], sVh[MK][MLD], sVl[MK][MLD];
    int prob = blockIdx.z, tile = blockIdx.x;
    const int head = blockIdx.y;
    if (tile_base && !find_tile(tile_base, n_prob, prob, tile)) return;
    const int ql = q_len[prob];
    if (tile * MQ >= ql) return;
    const int q0 = q_start[prob], k0 = k_start[prob], kl = k_len[prob];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int col = head * HD;
    const int r0 = tile * MQ + warp * 16 + g, r1 = r0 + 8;      // this lane's two query rows (within the problem)

    // Q fragments: a0 (r0, 8kk+t)  a1 (r1, 8kk+t)  a2 (r0, 8kk+t+4)  a3 (r1, 8kk+t+4)
    uint32_t qh[4][4], qlo[4][4];
    {
        const float* p0 = Q + (size_t)(q0 + min(r0, ql - 1)) * ldq + col;
        const float* p1 = Q + (size_t)(q0 + min(r1, ql - 1)) * ldq + col;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const float v[4] = {p0[8 * kk + t] * scale, p1[8 * kk + t] * scale, p0[8 * kk + t + 4] * scale,
                                p1[8 * kk + t + 4] * scale};
#pragma unroll
            for (int e = 0; e < 4; ++e) { qh[kk][e] = tf32_head(v[e]); qlo[kk][e] = tf32_head(v[e] - __uint_as_float(qh[kk][e])); }
        }
    }
    float acc[4][4];
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
    unsigned dw1 = 0, drg = 0;
    if constexpr (DROP) { dw1 = drop_word1(drop, prob, head); drg = (unsigned)(tile * MQ + warp * 16) >> 3; }

    for (int kb = 0; kb < kl; kb += MK) {
        __syncthreads();
        // stage + split one chunk of keys / values (zeros beyond the key range)
#pragma unroll
        for (int j = 0; j < (MK * 8) / 128; ++j) {
            const int f = threadIdx.x + 128 * j, r = f >> 3, c4 = f & 7;
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (kb + r < kl) {
                kv = __ldg(reinterpret_cast<const float4*>(Kp + (size_t)(k0 + kb + r) * ldk + col) + c4);
                vv = __ldg(reinterpret_cast<const float4*>(Vp + (size_t)(k0 + kb + r) * ldv + col) + c4);
            }
            const float kx[4] = {kv.x, kv.y, kv.z, kv.w}, vx[4] = {vv.x, vv.y, vv.z, vv.w};
            float kh[4], kl4[4], vh[4], vl4[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                // lo halves rounded to nearest TF32 too: the tensor core would truncate them (a one-sided bias)
                kh[e] = __uint_as_float(tf32_head(kx[e])); kl4[e] = __uint_as_float(tf32_head(kx[e] - kh[e]));
                vh[e] = __uint_as_float(tf32_head(vx[e])); vl4[e] = __uint_as_float(tf32_head(vx[e] - vh[e]));
            }
            *reinterpret_cast<float4*>(&sKh[r][4 * c4]) = make_float4(kh[0], kh[1], kh[2], kh[3]);
            *reinterpret_cast<float4*>(&sKl[r][4 * c4]) = make_float4(kl4[0], kl4[1], kl4[2], kl4[3]);
            *reinterpret_cast<float4*>(&sVh[r][4 * c4]) = make_float4(vh[0], vh[1], vh[2], vh[3]);
            *reinterpret_cast<float4*>(&sVl[r][4 * c4]) = make_float4(vl4[0], vl4[1], vl4[2], vl4[3]);
        }
        __syncthreads();

        // S = Q K^T over the chunk: 8 n-tiles of 8 keys
        float S[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
            for (int e = 0; e < 4; ++e) S[nt][e] = 0.f;
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const uint32_t bh0 = __float_as_uint(sKh[8 * nt + g][8 * kk + t]), bh1 = __float_as_uint(sKh[8 * nt + g][8 * kk + t + 4]);
                const uint32_t bl0 = __float_as_uint(sKl[8 * nt + g][8 * kk + t]), bl1 = __float_as_uint(sKl[8 * nt + g][8 * kk + t + 4]);
                mma_tf32(S[nt], qlo[kk], bh0, bh1);
                mma_tf32(S[nt], qh[kk], bl0, bl1);
                mma_tf32(S[nt], qh[kk], bh0, bh1);
            }
        }
        if (kb + MK > kl) {                      // last chunk: keys beyond the range get zero weight
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int key = kb + 8 * nt + 2 * t;
                if (key >= kl) { S[nt][0] = -INFINITY; S[nt][2] = -INFINITY; }
                if (key + 1 >= kl) { S[nt][1] = -INFINITY; S[nt][3] = -INFINITY; }
            }
        }
        // online softmax (base 2: the scores carry log2 e)
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            mx0 = fmaxf(mx0, fmaxf(S[nt][0], S[nt][1]));
            mx1 = fmaxf(mx1, fmaxf(S[nt][2], S[nt][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);       // finite: every chunk holds >= 1 valid key
        const float c0 = fast_exp2(m0 - mn0), c1 = fast_exp2(m1 - mn1);   // exp2(-inf) = 0 on the first chunk
        m0 = mn0; m1 = mn1;
        l0 *= c0; l1 *= c1;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            S[nt][0] = fast_exp2(S[nt][0] - mn0); S[nt][1] = fast_exp2(S[nt][1] - mn0);
            S[nt][2] = fast_exp2(S[nt][2] - mn1); S[nt][3] = fast_exp2(S[nt][3] - mn1);
            l0 += S[nt][0] + S[nt][1];
            l1 += S[nt][2] + S[nt][3];
        }
        unsigned mk0 = 0, mk1 = 0;              // keys kb + lane, kb + 32 + lane: bits 0-7 rows r0 - g.., 8-15 rows r1 - g..
        if constexpr (DROP) {
            const unsigned c0 = (unsigned)(kb + lane), c1 = c0 + 32u;
            mk0 = drop_keep8(drop, dw1, drg, c0) | (drop_keep8(drop, dw1, drg + 1u, c0) << 8);
            mk1 = drop_keep8(drop, dw1, drg, c1) | (drop_keep8(drop, dw1, drg + 1u, c1) << 8);
        }
        // O = O * c + P V.  The chunk's P V is accumulated from zero and added to the running output with a
        // round-to-nearest FMA: the tensor core truncates when it adds into its accumulator, and a chain through
        // every key of a 700-token cloud (264 MMAs) biased the outputs by ~1e-5 relative against float64.
        float pacc[4][4];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) pacc[j][e] = 0.f;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            // A fragment of P: a0 (r0, key 2t) a1 (r1, key 2t) a2 (r0, key 2t+1) a3 (r1, key 2t+1)
            float pv[4] = {S[nt][0], S[nt][2], S[nt][1], S[nt][3]};
            if constexpr (DROP) {
                const unsigned ma = __shfl_sync(0xffffffffu, nt < 4 ? mk0 : mk1, (8 * nt + 2 * t) & 31);
                const unsigned mb = __shfl_sync(0xffffffffu, nt < 4 ? mk0 : mk1, (8 * nt + 2 * t + 1) & 31);
                if (!((ma >> g) & 1u)) pv[0] = 0.f;
                if (!((ma >> (8 + g)) & 1u)) pv[1] = 0.f;
                if (!((mb >> g) & 1u)) pv[2] = 0.f;
                if (!((mb >> (8 + g)) & 1u)) pv[3] = 0.f;
            }
            uint32_t ph[4], pl[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { ph[e] = tf32_head(pv[e]); pl[e] = tf32_head(pv[e] - __uint_as_float(ph[e])); }
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t bh0 = __float_as_uint(sVh[8 * nt + 2 * t][8 * j + g]), bh1 = __float_as_uint(sVh[8 * nt + 2 * t + 1][8 * j + g]);
                const uint32_t bl0 = __float_as_uint(sVl[8 * nt + 2 * t][8 * j + g]), bl1 = __float_as_uint(sVl[8 * nt + 2 * t + 1][8 * j + g]);
                mma_tf32(pacc[j], pl, bh0, bh1);
                mma_tf32(pacc[j], ph, bl0, bl1);
                mma_tf32(pacc[j], ph, bh0, bh1);
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            acc[j][0] = fmaf(acc[j][0], c0, pacc[j][0]); acc[j][1] = fmaf(acc[j][1], c0, pacc[j][1]);
            acc[j][2] = fmaf(acc[j][2], c1, pacc[j][2]); acc[j][3] = fmaf(acc[j][3], c1, pacc[j][3]);
        }
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
    if constexpr (DROP) { i0 *= drop.scale; i1 *= drop.scale; }
    if (lse && t == 0) {                         // base-2 log-sum-exp of the scaled scores (-inf: empty key range)
        const int nh = gridDim.y;
        if (r0 < ql) lse[(size_t)(q0 + r0) * nh + head] = m0 + log2f(l0);
        if (r1 < ql) lse[(size_t)(q0 + r1) * nh + head] = m1 + log2f(l1);
    }
    // C fragment: (r0, 8j+2t), (r0, 8j+2t+1), (r1, 8j+2t), (r1, 8j+2t+1)
    if (r0 < ql) {
        float* dst = O + (size_t)(q0 + r0) * ldo + col + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[j][0] * i0, acc[j][1] * i0);
    }
    if (r1 < ql) {
        float* dst = O + (size_t)(q0 + r1) * ldo + col + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[j][2] * i1, acc[j][3] * i1);
    }
}

// ---- CorrespondenceDecoder.simple_attention (regtr.py:316-351) ---------------------------------------
// Single-head attention whose values are key COORDINATES: out[q] = sum_k softmax_k(Qp[q] . Kp[k] * scale) xyz[k],
// for every decoder layer l at once (rows l*n_rows + token of Qp/Kp).  Block = (16 queries, problem, layer):
// warp w owns queries 4w..4w+3, lane = key of the current 32-key chunk; keys and queries are staged
// TRANSPOSED ([d][key], [d][query]) so that the D-long dot products read conflict-free / broadcast.
constexpr int CQ = 16, CK = 32;

__global__ void __launch_bounds__(128)
k_corr_attention(const float* __restrict__ Qp, const float* __restrict__ Kp, int ld, const float* __restrict__ xyz,
                 float* __restrict__ out, const int32_t* __restrict__ q_start, const int32_t* __restrict__ q_len,
                 const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len, int n_rows, int D,
                 float scale) {
    extern __shared__ __align__(16) float smem_f[];
    float* sQt = smem_f;                       // [D][CQ]
    float* sKt = sQt + (size_t)D * CQ;          // [D][CK]
    float* sX = sKt + (size_t)D * CK;           // [CK][4]
    const int tile = blockIdx.x, prob = blockIdx.y, layer = blockIdx.z;
    const int ql = q_len[prob];
    if (tile * CQ >= ql) return;
    const int q0 = q_start[prob], k0 = k_start[prob], kl = k_len[prob];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t row_base = (size_t)layer * n_rows;
    const int d4 = D >> 2;
    for (int f = threadIdx.x; f < CQ * d4; f += 128) {          // queries, pre-scaled (softmax in base 2)
        const int r = f % CQ, c = f / CQ;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (tile * CQ + r < ql) v = __ldg(reinterpret_cast<const float4*>(Qp + (row_base + q0 + tile * CQ + r) * ld) + c);
        sQt[(4 * c + 0) * CQ + r] = v.x * scale; sQt[(4 * c + 1) * CQ + r] = v.y * scale;
        sQt[(4 * c + 2) * CQ + r] = v.z * scale; sQt[(4 * c + 3) * CQ + r] = v.w * scale;
    }
    float m[4], l[4], a[4][3];
#pragma unroll
    for (int i = 0; i < 4; ++i) { m[i] = -INFINITY; l[i] = 0.f; a[i][0] = a[i][1] = a[i][2] = 0.f; }

    for (int kb = 0; kb < kl; kb += CK) {
        __syncthreads();
        for (int f = threadIdx.x; f < CK * d4; f += 128) {
            const int r = f % CK, c = f / CK;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (kb + r < kl) v = __ldg(reinterpret_cast<const float4*>(Kp + (row_base + k0 + kb + r) * ld) + c);
            sKt[(4 * c + 0) * CK + r] = v.x; sKt[(4 * c + 1) * CK + r] = v.y;
            sKt[(4 * c + 2) * CK + r] = v.z; sKt[(4 * c + 3) * CK + r] = v.w;
        }
        if (threadIdx.x < CK) {
            const bool ok = kb + threadIdx.x < kl;
            const float* xr = xyz + (size_t)(k0 + kb + threadIdx.x) * 3;
            sX[4 * threadIdx.x + 0] = ok ? xr[0] : 0.f;
            sX[4 * threadIdx.x + 1] = ok ? xr[1] : 0.f;
            sX[4 * threadIdx.x + 2] = ok ? xr[2] : 0.f;
        }
        __syncthreads();
        float sc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
        for (int d = 0; d < D; ++d) {
            const float kv = sKt[d * CK + lane];
            const float4 q4 = *reinterpret_cast<const float4*>(sQt + d * CQ + 4 * warp);
            sc[0] = fmaf(kv, q4.x, sc[0]); sc[1] = fmaf(kv, q4.y, sc[1]);
            sc[2] = fmaf(kv, q4.z, sc[2]); sc[3] = fmaf(kv, q4.w, sc[3]);
        }
        const bool live = kb + lane < kl;
        const float vx = sX[4 * lane], vy = sX[4 * lane + 1], vz = sX[4 * lane + 2];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float sv = live ? sc[i] : -INFINITY;
            float mx = sv;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            const float mn = fmaxf(m[i], mx);                   // finite: the chunk holds >= 1 live key
            const float corr = exp2f(m[i] - mn), p = live ? exp2f(sv - mn) : 0.f;
            l[i] = l[i] * corr + p;
            a[i][0] = fmaf(p, vx, a[i][0] * corr); a[i][1] = fmaf(p, vy, a[i][1] * corr); a[i][2] = fmaf(p, vz, a[i][2] * corr);
            m[i] = mn;
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float r[4] = {l[i], a[i][0], a[i][1], a[i][2]};
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) r[e] += __shfl_xor_sync(0xffffffffu, r[e], o);
        const int qi = tile * CQ + 4 * warp + i;
        if (lane < 3 && qi < ql) {
            const float inv = r[0] > 0.f ? 1.f / r[0] : 0.f;
            out[(row_base + q0 + qi) * 3 + lane] = (lane == 0 ? r[1] : lane == 1 ? r[2] : r[3]) * inv;
        }
    }
}

// ---- head-averaged attention probabilities (analysis: TransformerCrossEncoder.get_attentions) -----------------
// P[q, k] = (1/H) sum_h softmax_k(q_h . k_h * scale), what nn.MultiheadAttention returns with its default
// average_attn_weights=True.  Block = (64-query tile, problem): 4 warps x 16 query rows, scores on mma.sync 3xTF32
// exactly as in k_mha_tf32x3 (same fragments, same split), keys staged per head in chunks of 64.
//   sweep 1: per head, the online row maximum m and sum l of exp2(s - m) over the whole key range; kept in shared
//            memory as (m, 1 / l) -- the log-sum-exp in two parts, so that exp2 reads s - m with m exact;
//   sweep 2: per key chunk, for every head the same scores again (bit for bit), exp2(s - m) / l summed over the heads
//            in registers, then written once, scaled by 1/H.
// No atomics: every output element has one writer.  Nothing outside [q_len x k_len] of a problem is written.
constexpr int PQ = 64, PK = 64, PH_MAX = 16;

__device__ __forceinline__ void probs_load_q(const float* __restrict__ Q, int ldq, int q0, int ql, int r0, int r1,
                                             int col, int t, float scale, uint32_t (&qh)[4][4], uint32_t (&qlo)[4][4]) {
    const float* p0 = Q + (size_t)(q0 + min(r0, ql - 1)) * ldq + col;
    const float* p1 = Q + (size_t)(q0 + min(r1, ql - 1)) * ldq + col;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        const float v[4] = {p0[8 * kk + t] * scale, p1[8 * kk + t] * scale, p0[8 * kk + t + 4] * scale,
                            p1[8 * kk + t + 4] * scale};
#pragma unroll
        for (int e = 0; e < 4; ++e) { qh[kk][e] = tf32_head(v[e]); qlo[kk][e] = tf32_head(v[e] - __uint_as_float(qh[kk][e])); }
    }
}

// stage keys [kb, kb + PK) of one head, split into TF32 (hi, lo); zeros beyond the key range
__device__ __forceinline__ void probs_stage_k(const float* __restrict__ Kp, int ldk, int k0, int kl, int kb, int col,
                                              float (*sKh)[MLD], float (*sKl)[MLD]) {
#pragma unroll
    for (int j = 0; j < (PK * 8) / 128; ++j) {
        const int f = threadIdx.x + 128 * j, r = f >> 3, c4 = f & 7;
        float4 kv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (kb + r < kl) kv = __ldg(reinterpret_cast<const float4*>(Kp + (size_t)(k0 + kb + r) * ldk + col) + c4);
        const float kx[4] = {kv.x, kv.y, kv.z, kv.w};
        float kh[4], kl4[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) { kh[e] = __uint_as_float(tf32_head(kx[e])); kl4[e] = __uint_as_float(tf32_head(kx[e] - kh[e])); }
        *reinterpret_cast<float4*>(&sKh[r][4 * c4]) = make_float4(kh[0], kh[1], kh[2], kh[3]);
        *reinterpret_cast<float4*>(&sKl[r][4 * c4]) = make_float4(kl4[0], kl4[1], kl4[2], kl4[3]);
    }
}

// S = Q K^T over one staged chunk (C fragments: (r0, 2t), (r0, 2t+1), (r1, 2t), (r1, 2t+1) of each 8-key n-tile);
// keys beyond the range get -inf
__device__ __forceinline__ void probs_scores(const uint32_t (&qh)[4][4], const uint32_t (&qlo)[4][4],
                                             const float (*sKh)[MLD], const float (*sKl)[MLD], int g, int t, int kb,
                                             int kl, float (&S)[8][4]) {
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
        for (int e = 0; e < 4; ++e) S[nt][e] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            const uint32_t bh0 = __float_as_uint(sKh[8 * nt + g][8 * kk + t]), bh1 = __float_as_uint(sKh[8 * nt + g][8 * kk + t + 4]);
            const uint32_t bl0 = __float_as_uint(sKl[8 * nt + g][8 * kk + t]), bl1 = __float_as_uint(sKl[8 * nt + g][8 * kk + t + 4]);
            mma_tf32(S[nt], qlo[kk], bh0, bh1);
            mma_tf32(S[nt], qh[kk], bl0, bl1);
            mma_tf32(S[nt], qh[kk], bh0, bh1);
        }
        const int key = kb + 8 * nt + 2 * t;
        if (key >= kl) { S[nt][0] = -INFINITY; S[nt][2] = -INFINITY; }
        if (key + 1 >= kl) { S[nt][1] = -INFINITY; S[nt][3] = -INFINITY; }
    }
}

__global__ void __launch_bounds__(128)
k_mha_probs_avg(const float* __restrict__ Q, int ldq, const float* __restrict__ Kp, int ldk, float* __restrict__ P,
                const int64_t* __restrict__ p_offset, const int32_t* __restrict__ p_pitch,
                const int32_t* __restrict__ q_start, const int32_t* __restrict__ q_len,
                const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len, int n_heads, float scale,
                float inv_heads) {
    __shared__ __align__(16) float sKh[PK][MLD], sKl[PK][MLD];
    __shared__ float sM[PH_MAX][PQ], sI[PH_MAX][PQ];
    const int tile = blockIdx.x, prob = blockIdx.y;
    const int ql = q_len[prob], kl = k_len[prob];
    if (tile * PQ >= ql || kl <= 0) return;                 // empty query or key range: nothing is written
    const int q0 = q_start[prob], k0 = k_start[prob];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int rl0 = warp * 16 + g, rl1 = rl0 + 8;              // rows inside the tile
    const int r0 = tile * PQ + rl0, r1 = tile * PQ + rl1;       // rows inside the problem
    uint32_t qh[4][4], qlo[4][4];
    float S[8][4];

    // sweep 1: row maximum and sum of every head
    for (int h = 0; h < n_heads; ++h) {
        probs_load_q(Q, ldq, q0, ql, r0, r1, h * HD, t, scale, qh, qlo);
        float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
        for (int kb = 0; kb < kl; kb += PK) {
            __syncthreads();
            probs_stage_k(Kp, ldk, k0, kl, kb, h * HD, sKh, sKl);
            __syncthreads();
            probs_scores(qh, qlo, sKh, sKl, g, t, kb, kl, S);
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                mx0 = fmaxf(mx0, fmaxf(S[nt][0], S[nt][1]));
                mx1 = fmaxf(mx1, fmaxf(S[nt][2], S[nt][3]));
            }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);   // finite: every chunk holds >= 1 valid key
            l0 *= exp2f(m0 - mn0); l1 *= exp2f(m1 - mn1);            // exp2(-inf) = 0 on the first chunk
            m0 = mn0; m1 = mn1;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                l0 += exp2f(S[nt][0] - mn0) + exp2f(S[nt][1] - mn0);
                l1 += exp2f(S[nt][2] - mn1) + exp2f(S[nt][3] - mn1);
            }
        }
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        if (t == 0) { sM[h][rl0] = m0; sI[h][rl0] = 1.f / l0; sM[h][rl1] = m1; sI[h][rl1] = 1.f / l1; }
    }

    // sweep 2: head-averaged probabilities, one key chunk at a time
    const int64_t base = p_offset[prob];
    const int pitch = p_pitch[prob];
    float* row0 = P + base + (int64_t)r0 * pitch;
    float* row1 = P + base + (int64_t)r1 * pitch;
    for (int kb = 0; kb < kl; kb += PK) {
        float acc[8][4];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
        for (int h = 0; h < n_heads; ++h) {
            probs_load_q(Q, ldq, q0, ql, r0, r1, h * HD, t, scale, qh, qlo);
            __syncthreads();                                   // also orders sweep 1's sM / sI stores before the loads
            probs_stage_k(Kp, ldk, k0, kl, kb, h * HD, sKh, sKl);
            __syncthreads();
            probs_scores(qh, qlo, sKh, sKl, g, t, kb, kl, S);
            const float m0 = sM[h][rl0], i0 = sI[h][rl0], m1 = sM[h][rl1], i1 = sI[h][rl1];
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                acc[nt][0] = fmaf(exp2f(S[nt][0] - m0), i0, acc[nt][0]);
                acc[nt][1] = fmaf(exp2f(S[nt][1] - m0), i0, acc[nt][1]);
                acc[nt][2] = fmaf(exp2f(S[nt][2] - m1), i1, acc[nt][2]);
                acc[nt][3] = fmaf(exp2f(S[nt][3] - m1), i1, acc[nt][3]);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int key = kb + 8 * nt + 2 * t;
            if (r0 < ql) {
                if (key < kl) row0[key] = acc[nt][0] * inv_heads;
                if (key + 1 < kl) row0[key + 1] = acc[nt][1] * inv_heads;
            }
            if (r1 < ql) {
                if (key < kl) row1[key] = acc[nt][2] * inv_heads;
                if (key + 1 < kl) row1[key + 1] = acc[nt][3] * inv_heads;
            }
        }
    }
}

// plan rows (pitch 2B + 1): q_start, q_len, cross k_start, cross k_len for cloud c of a (src x B, tgt x B) stack,
// then the exclusive prefix of the number of 64-query and 128-query tiles per problem (entry 2B = total): the
// attention kernels are launched over a LINEAR tile index and find their problem in this table, so that a
// capacity-shaped launch (the per-cloud lengths live on the device) does not pay for max_len / tile empty CTAs
// per problem.
__global__ void k_attention_plan(const int32_t* __restrict__ offs, int B, int32_t* __restrict__ plan) {
    const int n2 = 2 * B, ld = n2 + 1;
    for (int c = threadIdx.x; c < n2; c += blockDim.x) {
        const int o = c < B ? c + B : c - B;
        plan[0 * ld + c] = offs[c];
        plan[1 * ld + c] = offs[c + 1] - offs[c];
        plan[2 * ld + c] = offs[o];
        plan[3 * ld + c] = offs[o + 1] - offs[o];
    }
    if (threadIdx.x == 0) {
        int t64 = 0, t128 = 0;
        for (int c = 0; c < n2; ++c) {
            const int l = offs[c + 1] - offs[c];
            plan[4 * ld + c] = t64; plan[5 * ld + c] = t128;
            t64 += (l + 63) >> 6; t128 += (l + 127) >> 7;
        }
        plan[4 * ld + n2] = t64; plan[5 * ld + n2] = t128;
    }
}


}  // namespace

extern "C" int regtr_attention_plan(const int32_t* offs, int B, int32_t* plan, void* stream_) {
    if (B < 0) return REGTR_ERR_ARG;
    if (B == 0) return REGTR_OK;
    if (!offs || !plan) return REGTR_ERR_ARG;
    k_attention_plan<<<1, 128, 0, (cudaStream_t)stream_>>>(offs, B, plan);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// lse (training): the per-(row, head) base-2 log-sum-exp that the backward recomputes the softmax from.
extern "C" int regtr_mha_varlen_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                                    float* O, int ldo, float* lse, const int32_t* q_start, const int32_t* q_len,
                                    const int32_t* k_start, const int32_t* k_len, int n_problems, int max_q_len,
                                    const int32_t* tile_base, int max_tiles, int n_heads, int head_dim, float scale,
                                    const regtr_dropout_args* drop, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (tile_base && (lse || drop)) return REGTR_ERR_UNSUPPORTED;       // training launches have no tile table
    DropKey dk;
    if (drop && (!lse || drop_key_of(drop, dk) != REGTR_OK || n_heads > 16 || 2 * drop->n_pairs != n_problems))
        return REGTR_ERR_ARG;
    if (n_problems < 0 || max_q_len < 0 || n_heads <= 0 || max_tiles < 0) return REGTR_ERR_ARG;
    if (head_dim != HD) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || max_q_len == 0 || (tile_base && max_tiles == 0)) return REGTR_OK;
    if (!Q || !K || !V || !O || !q_start || !q_len || !k_start || !k_len) return REGTR_ERR_ARG;
    if ((ldq | ldk | ldv) % 4 != 0 || n_problems > 65535 || n_heads > 65535) return REGTR_ERR_ARG;
    if (ldo % 2) return REGTR_ERR_UNSUPPORTED;              // float2 output stores
    // with the tile table: linear 64-query tile index (max_tiles = host bound of the total); else one grid
    // column per problem sized by the longest sequence
    const dim3 grid = tile_base ? dim3(max_tiles, n_heads, 1) : dim3(regtr_cdiv(max_q_len, MQ), n_heads, n_problems);
    // softmax in base 2: q is pre-scaled by scale * log2(e)
    if (drop)
        k_mha_tf32x3<true><<<grid, 128, 0, st>>>(Q, ldq, K, ldk, V, ldv, O, ldo, q_start, q_len, k_start, k_len,
                                                 tile_base, n_problems, scale * 1.4426950408889634f, lse, dk);
    else
        k_mha_tf32x3<false><<<grid, 128, 0, st>>>(Q, ldq, K, ldk, V, ldv, O, ldo, q_start, q_len, k_start, k_len,
                                                  tile_base, n_problems, scale * 1.4426950408889634f, lse, DropKey{});
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

extern "C" int regtr_mha_probs_avg(const float* Q, int ldq, const float* K, int ldk, float* P,
                                   const int64_t* p_offset, const int32_t* p_pitch, const int32_t* q_start,
                                   const int32_t* q_len, const int32_t* k_start, const int32_t* k_len, int n_problems,
                                   int max_q_len, int n_heads, int head_dim, float scale, void* stream_) {
    if (n_problems < 0 || max_q_len < 0 || n_heads <= 0) return REGTR_ERR_ARG;
    if (head_dim != HD || n_heads > PH_MAX) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || max_q_len == 0) return REGTR_OK;
    if (!Q || !K || !P || !p_offset || !p_pitch || !q_start || !q_len || !k_start || !k_len) return REGTR_ERR_ARG;
    if (ldq % 4 != 0 || ldk % 4 != 0 || ldq < n_heads * HD || ldk < n_heads * HD) return REGTR_ERR_ARG;
    if (((uintptr_t)Q | (uintptr_t)K) % 16 != 0 || n_problems > 65535) return REGTR_ERR_ARG;
    const dim3 grid(regtr_cdiv(max_q_len, PQ), n_problems);
    k_mha_probs_avg<<<grid, 128, 0, (cudaStream_t)stream_>>>(Q, ldq, K, ldk, P, p_offset, p_pitch, q_start, q_len,
                                                            k_start, k_len, n_heads, scale * 1.4426950408889634f,
                                                            1.f / (float)n_heads);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

extern "C" int regtr_corr_decode_fwd(const float* Qp, const float* Kp, int ld, const float* xyz, float* out,
                                     const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                                     const int32_t* k_len, int n_problems, int max_q_len, int n_layers, int n_rows,
                                     int D, float scale, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_problems < 0 || max_q_len < 0 || n_layers < 0 || n_rows < 0 || D <= 0) return REGTR_ERR_ARG;
    if (D % 4 != 0 || ld % 4 != 0 || ld < D) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || max_q_len == 0 || n_layers == 0) return REGTR_OK;
    if (!Qp || !Kp || !xyz || !out || !q_start || !q_len || !k_start || !k_len) return REGTR_ERR_ARG;
    if (n_problems > 65535 || n_layers > 65535) return REGTR_ERR_ARG;
    const size_t smem = ((size_t)D * (CQ + CK) + 4 * CK) * sizeof(float);
    if (smem > 200 * 1024) return REGTR_ERR_UNSUPPORTED;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(k_corr_attention, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return -(1000 + (int)e);
    }
    dim3 grid(regtr_cdiv(max_q_len, CQ), n_problems, n_layers);
    k_corr_attention<<<grid, 128, smem, st>>>(Qp, Kp, ld, xyz, out, q_start, q_len, k_start, k_len, n_rows, D,
                                              scale * 1.4426950408889634f);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}
