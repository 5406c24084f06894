// fp32-accurate dense GEMM on the Hopper tensor cores (wgmma, 3xTF32 split).
//
//   C[M,N] = act( A[M,K] @ B[N,K]^T + bias[N] + R[M,N] )        (all row-major fp32)
//
// It replaces the cuBLAS SIMT sgemm calls behind every nn.Linear on the RegTR hot path (unary
// blocks kpconv_blocks.py:546-561, feat_proj regtr.py:145, attention in/out projections and FFN
// transformers.py:197-238, regressor MLP regtr.py:413-443) and the KPConv weight contraction
// (kpconv_blocks.py:401-406) while keeping the fp32 parity tolerance: a single TF32 pass moves
// the pose by 4e-3 (DESIGN.md), so every operand is split x = hi + lo with both halves exactly
// representable in TF32 and the product is accumulated as hi*hi + hi*lo + lo*hi in fp32
// (dropped term lo*lo ~ 2^-22 relative).  Kernel structure: see k_gemm_tf32x3_wg.
// B (weights) is split once on the host side of the ABI (regtr_split_tf32) and cached.
#include <cuda_bf16.h>


#include "common.cuh"
#include <stdlib.h>

#include "tc.cuh"

namespace {

// Optional bf16 epilogue for the attention in-projection: columns [0, split) are written row-major
// to `qk` (the q and k halves), columns >= split transposed to `vt` (one row per channel).
struct QkvOut {
    __nv_bfloat16* qk;
    int ld_qk;
    __nv_bfloat16* vt;
    int ld_vt;
    int split;
    // fp32 split epilogue for the 3xTF32 tensor-core attention core (attention_tf32_tc.cu): columns [0,E) = q (scaled by
    // qscale), [E,2E) = k, [2E,3E) = v; every value is written as its two TF32 halves:
    //   qk4 [M, 4E] = [Q_hi | Q_lo | K_hi | K_lo],  vt2 [2E, ld_vtf] = v transposed (hi rows, then lo rows)
    float* qk4;
    int ld4;
    float* vt2;
    int ld_vtf;
    int E;
    float qscale;
};
constexpr QkvOut NO_QKV = {nullptr, 0, nullptr, 0, 0, nullptr, 0, nullptr, 0, 0, 0.f};

// Optional InstanceNorm statistics of the OUTPUT (per cloud, per column: mean and 1/sqrt(var + eps) over the
// cloud's rows, kpconv_blocks.py:497-519) WITHOUT a separate pass over C: every epilogue warp reduces its 32 rows
// per column in a fixed shuffle tree (sum and sum of squares, fp32) and stores the pair to part[row / 32][column];
// k_in_finalize_part then adds the partials of the 32-row groups that lie inside a cloud in a fixed order (fp64) and
// reads the few rows of the groups that straddle a cloud boundary straight from C.  No atomics anywhere: the
// statistics are bit-identical from run to run.  (Two earlier versions accumulated with 64-bit integer atomics
// into per-(cloud, column) fixed-point accumulators: exact and order-independent, but ~10^4 warps adding to the
// same few hundred addresses made the level-0 GEMMs 2x slower than the separate statistics kernel they replaced.)

// v[j] of lane l -> lane j receives the sum over the lanes of v_l[j] (fixed butterfly: deterministic)
__device__ __forceinline__ float warp_transpose_sum(float (&v)[32], int lane) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < off; ++i) {
            const float mine = up ? v[i + off] : v[i];
            const float give = up ? v[i] : v[i + off];
            v[i] = mine + __shfl_xor_sync(0xffffffffu, give, off);
        }
    }
    return v[0];
}

// stats[c][col] = (mean, rstd) of cloud c.  grid (n_clouds, N / 32), block (32, 8): lane = column, 8 row lanes.
// direct_all: no partials (split-K launches of the small coarse levels): every row is read from C.
__global__ void __launch_bounds__(256)
k_in_finalize_part(const float2* __restrict__ part, const float* __restrict__ C, int ldc, const int32_t* __restrict__ offs,
                   int N, float eps, int direct_all, float2* __restrict__ stats) {
    __shared__ double red[8][32][2];
    const int c = blockIdx.x, col = blockIdx.y * 32 + threadIdx.x, w = threadIdx.y;
    const int a = offs[c], b = offs[c + 1];
    int g_lo = (a + 31) >> 5, g_hi = b >> 5;                    // 32-row groups [g_lo, g_hi) lie inside the cloud
    const bool full = !direct_all && g_lo < g_hi;
    const int head_end = full ? 32 * g_lo : b, tail_start = full ? 32 * g_hi : b;
    double s = 0.0, q = 0.0;
    if (col < N) {
        if (full)
            for (int g = g_lo + w; g < g_hi; g += 8) {
                const float2 p = part[(size_t)g * N + col];
                s += (double)p.x; q += (double)p.y;
            }
        for (int r = a + w; r < head_end; r += 8) { const double v = (double)C[(size_t)r * ldc + col]; s += v; q += v * v; }
        for (int r = tail_start + w; r < b; r += 8) { const double v = (double)C[(size_t)r * ldc + col]; s += v; q += v * v; }
    }
    red[w][threadIdx.x][0] = s; red[w][threadIdx.x][1] = q;
    __syncthreads();
    if (w == 0 && col < N) {
        for (int t = 1; t < 8; ++t) { s += red[t][threadIdx.x][0]; q += red[t][threadIdx.x][1]; }
        const int n = b - a;
        const double dn = n > 0 ? (double)n : 1.0;
        const double mean = s / dn;
        double var = q / dn - mean * mean;           // biased variance (InstanceNorm)
        var = var > 0.0 ? var : 0.0;
        stats[(size_t)c * N + col] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
}

constexpr int BM = 128;
constexpr int BK = 32;                       // fp32 elements = 128 bytes = one swizzle span
constexpr uint32_t HI_MASK = 0xFFFFE000u;    // keep sign, exponent and 10 mantissa bits

// round-to-nearest-even to TF32 precision (10 mantissa bits); unbiased, so split errors do not
// accumulate linearly along K as plain truncation does
__device__ __forceinline__ float tf32_hi(float x) {
    uint32_t u = __float_as_uint(x);
    u += 0x0FFFu + ((u >> 13) & 1u);
    return __uint_as_float(u & HI_MASK);
}

__global__ void k_split_tf32(const float* __restrict__ x, long long n, float* __restrict__ hi, float* __restrict__ lo) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float v = x[i], h = tf32_hi(v);
    hi[i] = h;
    lo[i] = tf32_hi(v - h);
}

// ---- Hopper warpgroup MMA ----------------------------------------------------------------------------------------
// A CTA walks output tiles blockIdx.x, + gridDim.x, ... (one tile per CTA for launches of up to REGTR_NUM_SMS tiles):
//   warp 8      TMA producer: A tile (fp32), B_hi tile, B_lo tile per 32-wide k-block (SWIZZLE_128B), STAGES deep;
//               its stage / phase counters run across tiles, so the next tile's loads fly under the epilogue
//   warps 0-7   two consumer warpgroups, rows [0, 64) and [64, 128) of the tile: each thread reads its tf32
//               A fragments from the swizzled stage, splits them into (hi, lo) in registers and issues
//               wgmma.m64nBNk8 with A from registers and B_hi / B_lo through shared-memory descriptors
// Every k-block is accumulated by the tensor core into a fresh register block (lo*hi + hi*lo + hi*hi, small terms
// first) that is then added to the running fp32 sum with round-to-nearest adds: the tensor core's own accumulation
// truncates, so its chains stay 12 MMAs long whatever K is.  lo = x - hi is exact in fp32 and rounded to nearest
// TF32 as well (a truncated lo is a one-sided 2^-21 bias that adds up linearly along K).
// The epilogue stages the tile through shared memory of its own: thread = tile row, 32 columns at a time, as
// bias / residual / ReLU -> global (+ optional InstanceNorm partial sums, + the attention in-projection's outputs).
constexpr int CONSUMER_THREADS = 256;
constexpr int GEMM_THREADS = CONSUMER_THREADS + 32;

template <int BN, int ST> struct CfgT {
    static constexpr int STAGES = ST;
    static constexpr int A_BYTES = BM * BK * 4;          // 16 KB (fp32 tile as loaded by TMA)
    static constexpr int B_BYTES = BN * BK * 4;
    static constexpr int STAGE_BYTES = A_BYTES + 2 * B_BYTES;
    static constexpr int LDT = BN + 4;                   // epilogue tile pitch (floats): row reads conflict-free
    static constexpr int TILE_BYTES = BM * LDT * 4;
    static constexpr int SMEM = STAGES * STAGE_BYTES + TILE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
    static constexpr int MIN_CTAS = SMEM <= 113 * 1024 ? 2 : 1;
};

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory"); }

template <int BN>
__device__ __forceinline__ void wgmma_tf32(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
    if constexpr (BN == 128) tc::wgmma_tf32_n128(d, a, bdesc, accumulate);
    else if constexpr (BN == 64) tc::wgmma_tf32_n64(d, a, bdesc, accumulate);
    else tc::wgmma_tf32_n32(d, a, bdesc, accumulate);
}

template <int BN, int ST>
__global__ void __launch_bounds__(GEMM_THREADS, CfgT<BN, ST>::MIN_CTAS)
k_gemm_tf32x3_wg(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
                 const __grid_constant__ CUtensorMap tmBlo, float* __restrict__ C, int ldc,
                 const float* __restrict__ bias, const float* __restrict__ R, int ldr, int M, int N, int K,
                 const int32_t* __restrict__ m_dev, int relu, int kb_per_split, size_t split_stride, QkvOut qkv,
                 float2* __restrict__ part) {
    using P = CfgT<BN, ST>;
    extern __shared__ unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (m_dev) M = min(M, *m_dev);
    const int tiles_n = (N + BN - 1) / BN;
    const int n_tiles = ((M + BM - 1) / BM) * tiles_n;       // tiles that hold real rows
    if ((int)blockIdx.x >= n_tiles) return;                  // capacity padding (uniform exit)

    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    auto stage_A = [&](int s) { return base + s * P::STAGE_BYTES; };
    auto stage_Bhi = [&](int s) { return base + s * P::STAGE_BYTES + P::A_BYTES; };
    auto stage_Blo = [&](int s) { return base + s * P::STAGE_BYTES + P::A_BYTES + P::B_BYTES; };
    float* ctile = reinterpret_cast<float*>(base + P::STAGES * P::STAGE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + P::STAGES * P::STAGE_BYTES + P::TILE_BYTES);
    uint64_t* full = bars;                    // TMA bytes landed                        (count 1 + tx)
    uint64_t* empty = bars + P::STAGES;       // every consumer warp is done with stage  (count 8)

    const int nkb_total = (K + BK - 1) / BK;
    const int kb0 = blockIdx.z * kb_per_split;
    const int nkb = min(kb_per_split, nkb_total - kb0);
    if (warp == 8 && lane == 0) {
        for (int s = 0; s < P::STAGES; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], CONSUMER_THREADS / 32); }
        tc::fence_barrier_init();
        tc::tma_prefetch_desc(&tmA); tc::tma_prefetch_desc(&tmBhi); tc::tma_prefetch_desc(&tmBlo);
    }
    __syncthreads();
    C += (size_t)blockIdx.z * split_stride;

    if (warp == 8) {
        if (lane == 0) {
            int it = 0;                                         // k-block counter across tiles
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int s = it % P::STAGES;
                    const uint32_t ph = (it / P::STAGES) & 1;
                    tc::mbar_wait(&empty[s], ph ^ 1);
                    tc::mbar_arrive_expect_tx(&full[s], P::A_BYTES + 2 * P::B_BYTES);
                    tc::tma_load_2d(stage_A(s), &tmA, &full[s], (kb0 + kb) * BK, m0);
                    tc::tma_load_2d(stage_Bhi(s), &tmBhi, &full[s], (kb0 + kb) * BK, n0);
                    tc::tma_load_2d(stage_Blo(s), &tmBlo, &full[s], (kb0 + kb) * BK, n0);
                }
            }
        }
        return;
    }

    const int g = lane >> 2, t = lane & 3;
    const int fr = (warp >> 2) * 64 + (warp & 3) * 16 + g;   // this thread's fragment rows: fr and fr + 8
    const int q = warp & 3;                                  // epilogue: rows 32q .. 32q + 31 (thread = row)
    const int r = q * 32 + lane;
    int it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int m0 = (tile / tiles_n) * BM, n0 = (tile % tiles_n) * BN;
        float acc[BN / 2], blk[BN / 2];
#pragma unroll
        for (int j = 0; j < BN / 2; ++j) acc[j] = 0.f;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
            const int s = it % P::STAGES;
            tc::mbar_wait(&full[s], (it / P::STAGES) & 1);
            // SWIZZLE_128B tile: 16-byte chunk c of row x sits at chunk (c ^ (x & 7)) of its 128-byte row
            const unsigned char* sa = stage_A(s);
            uint32_t ahi[BK / 8][4], alo[BK / 8][4];
#pragma unroll
            for (int k = 0; k < BK / 8; ++k)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int x = fr + (i & 1) * 8, chunk = 2 * k + (i >> 1);
                    const float f = *reinterpret_cast<const float*>(sa + x * 128 + ((chunk ^ (x & 7)) << 4) + 4 * t);
                    const uint32_t h = (__float_as_uint(f) + 0x1000u) & HI_MASK;             // RN (ties away) to TF32
                    ahi[k][i] = h;
                    alo[k][i] = (__float_as_uint(f - __uint_as_float(h)) + 0x1000u) & HI_MASK;   // RN: unbiased
                }
            const uint64_t dBhi = tc::gmma_desc_sw128(tc::smem_u32(stage_Bhi(s)));
            const uint64_t dBlo = tc::gmma_desc_sw128(tc::smem_u32(stage_Blo(s)));
            tc::wgmma_fence();
#pragma unroll
            for (int k = 0; k < BK / 8; ++k) {                     // k-step = 8 tf32 = 32 bytes of the swizzled row
                const uint64_t adv = (uint64_t)(2 * k);
                wgmma_tf32<BN>(blk, alo[k], dBhi + adv, k != 0);   // small terms first
                wgmma_tf32<BN>(blk, ahi[k], dBlo + adv, 1);
                wgmma_tf32<BN>(blk, ahi[k], dBhi + adv, 1);
            }
            tc::wgmma_commit();
            tc::wgmma_wait<0>();
            __syncwarp();
            if (lane == 0) tc::mbar_arrive(&empty[s]);            // A read into registers, B read by the MMAs
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) acc[j] += blk[j];
        }
        // ---- epilogue of this tile: fragments -> shared tile -> thread-per-row chunks of 32 columns
        consumer_sync();                                           // the previous tile's epilogue is done reading
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            *reinterpret_cast<float2*>(ctile + fr * P::LDT + 8 * j + 2 * t) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(ctile + (fr + 8) * P::LDT + 8 * j + 2 * t) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        consumer_sync();
        const int row = m0 + r;
        const bool row_ok = row < M;
        float* crow = C + (size_t)row * ldc;
        const float* rrow = (R && row_ok) ? R + (size_t)row * ldr : nullptr;
        const int row_base = m0 + q * 32;
#pragma unroll 1
        for (int c0 = 32 * (warp >> 2); c0 < BN; c0 += 64) {
            const int col0 = n0 + c0;
            if (col0 >= N) continue;                           // warp-uniform
            const float* tq = ctile + q * 32 * P::LDT + c0;    // this warp's 32 x 32 block
            float v[32];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 o = *reinterpret_cast<const float4*>(tq + lane * P::LDT + 4 * j);
                v[4 * j] = o.x; v[4 * j + 1] = o.y; v[4 * j + 2] = o.z; v[4 * j + 3] = o.w;
            }
            if (qkv.qk) {                                      // bf16 epilogue (N % 32 == 0 guaranteed by the host)
                if (!row_ok) continue;
                if (bias) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] += bias[col0 + j];
                }
                if (col0 < qkv.split) {
                    uint32_t pk[16];
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const __nv_bfloat162 b = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
                        pk[j] = *reinterpret_cast<const uint32_t*>(&b);
                    }
                    uint4* dstq = reinterpret_cast<uint4*>(qkv.qk + (size_t)row * qkv.ld_qk + col0);
#pragma unroll
                    for (int j = 0; j < 4; ++j) dstq[j] = make_uint4(pk[4 * j], pk[4 * j + 1], pk[4 * j + 2], pk[4 * j + 3]);
                } else {
#pragma unroll
                    for (int j = 0; j < 32; ++j)
                        qkv.vt[(size_t)(col0 - qkv.split + j) * qkv.ld_vt + row] = __float2bfloat16_rn(v[j]);
                }
                continue;
            }
            if (qkv.qk4) {                                     // fp32 split epilogue (N = 3E, E % 32 == 0)
                // q / k leave as 128-byte row segments per 8 lanes, v transposed with lane = token
                const int sec = col0 / qkv.E, cin = col0 - sec * qkv.E;
                if (sec < 2) {
                    const int cq = lane & 7, rsub = lane >> 3;
                    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (bias) b4 = *reinterpret_cast<const float4*>(bias + col0 + 4 * cq);
                    const float sc = sec == 0 ? qkv.qscale : 1.f;
#pragma unroll
                    for (int it = 0; it < 8; ++it) {
                        const int rr = it * 4 + rsub, rg = row_base + rr;
                        const float4 o = *reinterpret_cast<const float4*>(tq + rr * P::LDT + 4 * cq);
                        const float f[4] = {(o.x + b4.x) * sc, (o.y + b4.y) * sc, (o.z + b4.z) * sc, (o.w + b4.w) * sc};
                        float h[4], l[4];
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            h[e] = __uint_as_float((__float_as_uint(f[e]) + 0x1000u) & HI_MASK);
                            l[e] = __uint_as_float((__float_as_uint(f[e] - h[e]) + 0x1000u) & HI_MASK);
                        }
                        if (rg < M) {
                            float* dst = qkv.qk4 + (size_t)rg * qkv.ld4 + sec * 2 * qkv.E + cin + 4 * cq;
                            *reinterpret_cast<float4*>(dst) = make_float4(h[0], h[1], h[2], h[3]);
                            *reinterpret_cast<float4*>(dst + qkv.E) = make_float4(l[0], l[1], l[2], l[3]);
                        }
                    }
                } else {
                    const int rg = row_base + lane;
#pragma unroll 4
                    for (int j = 0; j < 32; ++j) {
                        const float f = tq[lane * P::LDT + j] + (bias ? bias[col0 + j] : 0.f);
                        const float h = __uint_as_float((__float_as_uint(f) + 0x1000u) & HI_MASK);
                        const float l = __uint_as_float((__float_as_uint(f - h) + 0x1000u) & HI_MASK);
                        if (rg < M) {
                            qkv.vt2[(size_t)(cin + j) * qkv.ld_vtf + rg] = h;
                            qkv.vt2[(size_t)(qkv.E + cin + j) * qkv.ld_vtf + rg] = l;
                        }
                    }
                }
                continue;
            }
            if (col0 + 32 <= N && (ldc & 3) == 0 && (!R || (ldr & 3) == 0)) {
                // the block's rows leave as 128-byte row segments, 4 rows per warp instruction -- 4 memory wavefronts
                // instead of 32 per store, and the residual is read the same way
                const int cq = lane & 7, rsub = lane >> 3;
                float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
                if (bias) b4 = *reinterpret_cast<const float4*>(bias + col0 + 4 * cq);
#pragma unroll
                for (int it = 0; it < 8; ++it) {
                    const int rr = it * 4 + rsub, rg = row_base + rr;
                    float4 o = *reinterpret_cast<const float4*>(tq + rr * P::LDT + 4 * cq);
                    if (rg < M) {
                        o.x += b4.x; o.y += b4.y; o.z += b4.z; o.w += b4.w;
                        if (R) {
                            const float4 rv = *reinterpret_cast<const float4*>(R + (size_t)rg * ldr + col0 + 4 * cq);
                            o.x += rv.x; o.y += rv.y; o.z += rv.z; o.w += rv.w;
                        }
                        if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                        *reinterpret_cast<float4*>(C + (size_t)rg * ldc + col0 + 4 * cq) = o;
                    }
                }
            } else {
#pragma unroll
                for (int j = 0; j < 32; ++j) {
                    if (col0 + j < N) {
                        if (bias) v[j] += bias[col0 + j];
                        if (rrow) v[j] += rrow[col0 + j];
                        if (relu) v[j] = fmaxf(v[j], 0.f);
                        if (row_ok) crow[col0 + j] = v[j];
                    }
                }
            }
            if (part) {                                        // host guarantees N % 32 == 0 in this mode
                // per-column sum / sum of squares over this warp's 32 rows (fixed shuffle tree), one float2 per
                // (32-row group, column); groups that straddle a cloud boundary or M are ignored by the finaliser
                float sq[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) sq[j] = v[j] * v[j];
                const float s1 = warp_transpose_sum(v, lane);
                const float s2 = warp_transpose_sum(sq, lane);
                part[(size_t)((m0 >> 5) + q) * N + col0 + lane] = make_float2(s1, s2);
            }
        }
    }
}

// C = act(sum_z P[z] + bias + R): deterministic split-K reduction (fixed order), 4 columns / thread
__global__ void k_splitk_reduce(const float* __restrict__ P, int splits, size_t split_stride, float* __restrict__ C,
                                int ldc, const float* __restrict__ bias, const float* __restrict__ R, int ldr, int M,
                                int N, const int32_t* __restrict__ m_dev, int relu) {
    if (m_dev) M = min(M, *m_dev);
    const int n4 = N >> 2;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)M * n4) return;
    int r, c;
    regtr_row_col((unsigned)t, (unsigned)n4, r, c);
    c *= 4;
    const float* p0 = P + (size_t)r * N + c;
    float4 acc = *reinterpret_cast<const float4*>(p0);
    int z = 1;
    for (; z + 4 <= splits; z += 4) {                  // four planes in flight; the sum keeps the plane order
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = *reinterpret_cast<const float4*>(p0 + (size_t)(z + u) * split_stride);
#pragma unroll
        for (int u = 0; u < 4; ++u) { acc.x += v[u].x; acc.y += v[u].y; acc.z += v[u].z; acc.w += v[u].w; }
    }
    for (; z < splits; ++z) {
        const float4 v = *reinterpret_cast<const float4*>(p0 + (size_t)z * split_stride);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (bias) { acc.x += bias[c]; acc.y += bias[c + 1]; acc.z += bias[c + 2]; acc.w += bias[c + 3]; }
    if (R) {
        const float* rr = R + (size_t)r * ldr + c;
        acc.x += rr[0]; acc.y += rr[1]; acc.z += rr[2]; acc.w += rr[3];
    }
    if (relu) { acc.x = fmaxf(acc.x, 0.f); acc.y = fmaxf(acc.y, 0.f); acc.z = fmaxf(acc.z, 0.f); acc.w = fmaxf(acc.w, 0.f); }
    float* o = C + (size_t)r * ldc + c;
    o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
}

// CUDA-core reference (REGTR_GEMM_IMPL=ffma; A/B accuracy measurements only, tests/diag_accuracy.py): one thread
// per output element, sequential round-to-nearest FMA over K -- what an fp32 SGEMM computes.
__global__ void k_gemm_ffma(const float* __restrict__ A, int lda, const float* __restrict__ Bhi,
                            const float* __restrict__ Blo, int ldb, float* __restrict__ C, int ldc,
                            const float* __restrict__ bias, const float* __restrict__ R, int ldr, int M, int N, int K,
                            const int32_t* __restrict__ m_dev, int relu) {
    if (m_dev) M = min(M, *m_dev);
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    for (int m = blockIdx.y; m < M; m += gridDim.y) {
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc = fmaf(A[(size_t)m * lda + k], Bhi[(size_t)n * ldb + k] + Blo[(size_t)n * ldb + k], acc);
        if (bias) acc += bias[n];
        if (R) acc += R[(size_t)m * ldr + n];
        if (relu) acc = fmaxf(acc, 0.f);
        C[(size_t)m * ldc + n] = acc;
    }
}

// split count: only for skinny problems (few output tiles) with a long K, to fill the machine
// (ceil(REGTR_NUM_SMS / tiles) planes, each of at least 8 k-blocks); the planes are summed in a fixed order by the
// reduction kernel.  At most 16 k-blocks (K = 512) per plane keeps the split's partial sums short as well.
int choose_splits(int M, int N, int K, int bn) {
    const int tiles = regtr_cdiv(M, BM) * regtr_cdiv(N, bn);
    const int nkb = regtr_cdiv(K, BK);
    if (tiles >= REGTR_NUM_SMS / 2 || nkb < 16 || (N & 3)) return 1;
    int s = regtr_cdiv(REGTR_NUM_SMS, tiles);
    if (s > nkb / 8) s = nkb / 8;
    if (s > 8) s = 8;
    const int s_acc = regtr_cdiv(nkb, 16);
    if (s < s_acc) s = s_acc;
    if (s > 16) s = 16;
    return s < 1 ? 1 : s;
}

// Widest tile that covers N: the pipeline keeps several independent pairs in flight, so the machine is
// filled by OTHER forwards and what counts is the total CTA time (A is streamed / split once per N-tile).
int choose_bn(int M, int N) {
    (void)M;
    return N > 64 ? 128 : (N > 32 ? 64 : 32);
}

// ---- host: tensor maps (driver entry point resolved through the runtime, no libcuda link)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// row-major fp32 matrix [rows, cols] with leading dimension ld; box = [box_rows, 32 cols], 128B swizzle
bool make_map(CUtensorMap* m, const float* ptr, int rows, int cols, int ld, int box_rows) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * sizeof(float)};
    cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int BN, int ST>
int launch_gemm(const float* A, int lda, const float* Bhi, const float* Blo, int ldb, float* C, int ldc,
                const float* bias, const float* R, int ldr, int M, int N, int K, const int32_t* m_dev, int relu,
                int splits, float* ws, cudaStream_t st, QkvOut qkv = NO_QKV, float2* part = nullptr) {
    using P = CfgT<BN, ST>;
    CUtensorMap tA, tBh, tBl;
    if (!make_map(&tA, A, M, K, lda, BM) || !make_map(&tBh, Bhi, N, K, ldb, BN) || !make_map(&tBl, Blo, N, K, ldb, BN))
        return REGTR_ERR_ARG;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(k_gemm_tf32x3_wg<BN, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, P::SMEM);
        if (e != cudaSuccess) return -(1000 + (int)e);
        attr_set = true;
    }
    const int nkb = regtr_cdiv(K, BK);
    const int tiles = regtr_cdiv(M, BM) * regtr_cdiv(N, BN);
    if (splits <= 1) {
        // Launches of several waves walk their tiles with fewer CTAs: ~4 tiles per CTA, between half and twice the SM
        // count, so that one set-up serves several tiles and the other forwards' kernels still find free SMs.
        int grid = tiles;
        if (tiles > REGTR_NUM_SMS / 4) {
            grid = tiles / 4;
            grid = grid < REGTR_NUM_SMS / 2 ? REGTR_NUM_SMS / 2 : (grid > 2 * REGTR_NUM_SMS ? 2 * REGTR_NUM_SMS : grid);
            if (grid > tiles) grid = tiles;
        }
        k_gemm_tf32x3_wg<BN, ST><<<grid, GEMM_THREADS, P::SMEM, st>>>(tA, tBh, tBl, C, ldc, bias, R, ldr, M, N, K, m_dev,
                                                                      relu, nkb, 0, qkv, part);
        REGTR_CHECK_LAUNCH();
        return REGTR_OK;
    }
    const int per = regtr_cdiv(nkb, splits);
    const int z = regtr_cdiv(nkb, per);                     // every plane gets >= 1 k-block
    const size_t stride = (size_t)M * N;
    k_gemm_tf32x3_wg<BN, ST><<<dim3(tiles, 1, z), GEMM_THREADS, P::SMEM, st>>>(tA, tBh, tBl, ws, N, nullptr, nullptr, 0, M, N,
                                                                               K, m_dev, 0, per, stride, NO_QKV, nullptr);
    REGTR_CHECK_LAUNCH();
    k_splitk_reduce<<<regtr_cdiv((long long)M * (N / 4), 256), 256, 0, st>>>(ws, z, stride, C, ldc, bias, R, ldr, M, N,
                                                                            m_dev, relu);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // namespace

extern "C" {

int regtr_split_tf32(const float* x, long long n, float* hi, float* lo, void* stream_) {
    if (n < 0) return REGTR_ERR_ARG;
    if (n == 0) return REGTR_OK;
    if (!x || !hi || !lo) return REGTR_ERR_ARG;
    k_split_tf32<<<regtr_cdiv(n, 256), 256, 0, (cudaStream_t)stream_>>>(x, n, hi, lo);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_gemm_ws_bytes(int M, int N, int K) {
    if (M <= 0 || N <= 0 || K <= 0) return 256;
    const int s = choose_splits(M, N, K, choose_bn(M, N));
    return s > 1 ? regtr_align((size_t)s * M * N * sizeof(float)) : 256;
}

static int gemm_dispatch(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb, float* C, int ldc,
                         const float* bias, const float* R, int ldr, int M, int N, int K, const int32_t* m_dev,
                         int relu, void* ws, size_t ws_bytes, void* stream_, float2* part, int* used_splits) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (M < 0 || N <= 0 || K <= 0) return REGTR_ERR_ARG;
    if (M == 0) return REGTR_OK;
    if (!A || !B_hi || !B_lo || !C) return REGTR_ERR_ARG;
    // TMA: 16-byte aligned bases and row pitches
    if ((lda & 3) || (ldb & 3) || ((uintptr_t)A & 15) || ((uintptr_t)B_hi & 15) || ((uintptr_t)B_lo & 15))
        return REGTR_ERR_UNSUPPORTED;
    {
        const char* impl = getenv("REGTR_GEMM_IMPL");
        if (impl && impl[0] == 'f') {
            if (used_splits) *used_splits = 2;                  // statistics: read every row from C
            k_gemm_ffma<<<dim3(regtr_cdiv(N, 128), M < 32768 ? M : 32768), 128, 0, st>>>(A, lda, B_hi, B_lo, ldb, C, ldc, bias, R, ldr, M, N, K,
                                                                    m_dev, relu);
            REGTR_CHECK_LAUNCH();
            return REGTR_OK;
        }
    }
    const int bn = choose_bn(M, N);
    int splits = choose_splits(M, N, K, bn);
    if (used_splits) *used_splits = splits;
    if (splits > 1 && (!ws || ws_bytes < regtr_gemm_ws_bytes(M, N, K))) return REGTR_ERR_WORKSPACE;
    float2* p = splits > 1 ? nullptr : part;
    // Stages: as deep as keeps the epilogue tile beside them; the 32-wide tile takes 3 so that two CTAs share an SM.
    if (bn == 128) return launch_gemm<128, 3>(A, lda, B_hi, B_lo, ldb, C, ldc, bias, R, ldr, M, N, K, m_dev, relu, splits, (float*)ws, st, NO_QKV, p);
    if (bn == 64) return launch_gemm<64, 4>(A, lda, B_hi, B_lo, ldb, C, ldc, bias, R, ldr, M, N, K, m_dev, relu, splits, (float*)ws, st, NO_QKV, p);
    return launch_gemm<32, 3>(A, lda, B_hi, B_lo, ldb, C, ldc, bias, R, ldr, M, N, K, m_dev, relu, splits, (float*)ws, st, NO_QKV, p);
}

int regtr_gemm_tf32x3(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb, float* C, int ldc,
                      const float* bias, const float* R, int ldr, int M, int N, int K, const int32_t* m_dev,
                      int relu, void* ws, size_t ws_bytes, void* stream_) {
    return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, bias, R, ldr, M, N, K, m_dev, relu, ws, ws_bytes, stream_,
                         nullptr, nullptr);
}

size_t regtr_instnorm_part_bytes(int M, int N) {
    return sizeof(float2) * (size_t)(regtr_cdiv(M > 0 ? M : 1, 128) * 4) * (size_t)(N > 0 ? N : 1);
}

int regtr_gemm_tf32x3_instats(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb, float* C, int ldc,
                              int M, int N, int K, const int32_t* m_dev, const int32_t* offs, int n_clouds, float eps,
                              void* part, float* stats, void* ws, size_t ws_bytes, void* stream_) {
    if (!offs || n_clouds <= 0 || !part || !stats) return REGTR_ERR_ARG;
    if (N % 32 != 0 || ((uintptr_t)part & 7)) return REGTR_ERR_UNSUPPORTED;
    if (M <= 0) return M < 0 ? REGTR_ERR_ARG : REGTR_OK;
    int splits = 1;
    const int rc = gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, nullptr, nullptr, 0, M, N, K, m_dev, 0, ws, ws_bytes,
                                 stream_, (float2*)part, &splits);
    if (rc != REGTR_OK) return rc;
    k_in_finalize_part<<<dim3(n_clouds, N / 32), dim3(32, 8), 0, (cudaStream_t)stream_>>>(
        (const float2*)part, C, ldc, offs, N, eps, splits > 1 ? 1 : 0, (float2*)stats);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// In-projection of the attention block with the bf16 epilogue consumed by regtr_mha_bf16_tc_fwd:
// qk_out [M, split] bf16 (ld_qk), vt_out [N - split, ld_vt] bf16 (transposed v), bias added first.
int regtr_gemm_tf32x3_qkv_bf16(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                               const float* bias, int M, int N, int K, int split, void* qk_out, int ld_qk,
                               void* vt_out, int ld_vt, const int32_t* m_dev, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (M < 0 || N <= 0 || K <= 0 || split <= 0 || split > N) return REGTR_ERR_ARG;
    if (M == 0) return REGTR_OK;
    if (!A || !B_hi || !B_lo || !qk_out || !vt_out) return REGTR_ERR_ARG;
    if ((N & 31) || (split & 31) || (ld_qk & 7) || ((uintptr_t)qk_out & 15) || (lda & 3) || (ldb & 3) ||
        ((uintptr_t)A & 15) || ((uintptr_t)B_hi & 15) || ((uintptr_t)B_lo & 15) || ld_vt < M)
        return REGTR_ERR_UNSUPPORTED;
    QkvOut q = NO_QKV;
    q.qk = (__nv_bfloat16*)qk_out; q.ld_qk = ld_qk; q.vt = (__nv_bfloat16*)vt_out; q.ld_vt = ld_vt; q.split = split;
    float* dummy = reinterpret_cast<float*>(qk_out);      // C is never written in this mode
    const int bn = choose_bn(M, N);
    if (bn == 128) return launch_gemm<128, 3>(A, lda, B_hi, B_lo, ldb, dummy, 0, bias, nullptr, 0, M, N, K, m_dev, 0, 1, nullptr, st, q);
    if (bn == 64) return launch_gemm<64, 4>(A, lda, B_hi, B_lo, ldb, dummy, 0, bias, nullptr, 0, M, N, K, m_dev, 0, 1, nullptr, st, q);
    return launch_gemm<32, 3>(A, lda, B_hi, B_lo, ldb, dummy, 0, bias, nullptr, 0, M, N, K, m_dev, 0, 1, nullptr, st, q);
}

// In-projection of the attention block with the fp32 split epilogue consumed by regtr_mha_tf32_tc_fwd (see QkvOut).
int regtr_gemm_tf32x3_qkv_split(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                                const float* bias, int M, int N, int K, int E, float qscale, float* qk4, int ld4,
                                float* vt2, int ld_vt, const int32_t* m_dev, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (M < 0 || N <= 0 || K <= 0 || E <= 0 || N != 3 * E) return REGTR_ERR_ARG;
    if (M == 0) return REGTR_OK;
    if (!A || !B_hi || !B_lo || !qk4 || !vt2) return REGTR_ERR_ARG;
    if ((E & 31) || (ld4 & 3) || ld4 < 4 * E || ((uintptr_t)qk4 & 15) || (lda & 3) || (ldb & 3) || ((uintptr_t)A & 15) ||
        ((uintptr_t)B_hi & 15) || ((uintptr_t)B_lo & 15) || ld_vt < M)
        return REGTR_ERR_UNSUPPORTED;
    QkvOut q = NO_QKV;
    q.qk4 = qk4; q.ld4 = ld4; q.vt2 = vt2; q.ld_vtf = ld_vt; q.E = E; q.qscale = qscale;
    return launch_gemm<128, 3>(A, lda, B_hi, B_lo, ldb, qk4, 0, bias, nullptr, 0, M, N, K, m_dev, 0, 1, nullptr, st, q);
}

}  // extern "C"
