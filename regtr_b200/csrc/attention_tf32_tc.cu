// fp32-accurate variable-length multi-head attention core on the Hopper tensor cores (3xTF32 split, fp32
// accumulation, fp32 softmax): the parity-mode MHA core of TransformerCrossEncoderLayer.forward_pre
// (reference src/models/transformer/transformers.py:197-226) with both contractions -- S = Q K^T and
// O = P V -- fed by TMA and issued as wgmma.m64nNk8 tf32.  head_dim = 32.
//
// Inputs come from the in-projection GEMM's split epilogue (gemm_tc.cu, regtr_gemm_tf32x3_qkv_split):
//   qk4 [N_tokens, 4E] fp32 : [Q_hi | Q_lo | K_hi | K_lo], q pre-scaled by scale * log2(e); x = hi + lo with both
//                             halves exactly representable in TF32                       (TMA, SWIZZLE_128B)
//   vt2 [2E, ld_vt]    fp32 : v TRANSPOSED (rows = channels, hi then lo; tokens contiguous), so that P V is a
//                             K-major x K-major MMA                                       (TMA, SWIZZLE_128B)
// CTA = (problem, head, tile of 128 queries); 9 warps:
//   warp 8     TMA producer (Q_hi / Q_lo once; per 64-key tile K_hi [+ K_lo, Vt_hi, Vt_lo in pass 2], 2 stages)
//   warps 0-7  two consumer warpgroups, queries [0, 64) and [64, 128) of the tile; S and O live in registers
// Two passes over the keys:
//   pass 1  S ~ Q_hi K_hi^T (one TF32 MMA per k-step: the row maximum only stabilises the exponentials, any
//           value within a few per cent of it serves) -> row maximum m;
//   pass 2  S = Q_lo K_hi^T + Q_hi K_lo^T + Q_hi K_hi^T (fp32-accurate), p = exp2(s - m), row sums in registers,
//           p moved from the accumulator layout into the A-fragment layout with quad shuffles and split into
//           (hi, lo) TF32 halves there: O_tile = P_lo V_hi + P_hi V_lo + P_hi V_hi, added to the running O with
//           round-to-nearest fp32 adds.  P never touches shared memory, the accumulator is never rescaled.
#include "common.cuh"
#include "tc.cuh"

namespace {

constexpr int HD = 32;          // head dim (floats: one 128-byte swizzle row)
constexpr int BQ = 128;         // queries per CTA
constexpr int BKEY = 64;        // keys per tile
constexpr int THREADS = 288;

constexpr int Q_BYTES = BQ * HD * 4;        // 16 KB per half (hi / lo)
constexpr int K_BYTES = BKEY * HD * 4;      // 8 KB per half
constexpr int V_HALF = HD * 32 * 4;         // 4 KB: 32 channel rows x 32 keys; a 64-key tile = 2 halves per (hi / lo)
constexpr int STAGE_BYTES = 2 * K_BYTES + 4 * V_HALF;      // K_hi K_lo | Vt_hi(0,1) Vt_lo(0,1) = 32 KB
constexpr int SMEM_BYTES = 2 * Q_BYTES + 2 * STAGE_BYTES + 1024 + 256;
constexpr uint32_t HI_MASK = 0xFFFFE000u;

__device__ __forceinline__ uint32_t tf32_rn(float x) { return (__float_as_uint(x) + 0x1000u) & HI_MASK; }
__device__ __forceinline__ float fast_exp2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__global__ void __launch_bounds__(THREADS, 1)
k_mha_tf32_tc(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
              const __grid_constant__ CUtensorMap tmVt, float* __restrict__ O, int ldo, int E,
              const int32_t* __restrict__ q_start, const int32_t* __restrict__ q_len,
              const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len,
              const int32_t* __restrict__ tile_base, int n_prob) {
    extern __shared__ unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int prob = blockIdx.z, qt = blockIdx.x;
    const int head = blockIdx.y;
    if (tile_base) {                                             // linear 128-query tile index -> (problem, tile)
        if (qt >= tile_base[n_prob]) return;
        int p = 0;
        while (p + 1 < n_prob && tile_base[p + 1] <= qt) ++p;
        prob = p;
        qt -= tile_base[p];
    }
    const int ql = q_len[prob];
    if (qt * BQ >= ql) return;                                   // uniform exit
    const int q0 = q_start[prob] + qt * BQ, k0 = k_start[prob], kl = k_len[prob];
    if (kl <= 0) {                                                // no keys: zero rows (uniform exit)
        for (int t = threadIdx.x; t < BQ * HD; t += blockDim.x) {
            const int r = t / HD, d = t % HD;
            if (qt * BQ + r < ql) O[(size_t)(q0 + r) * ldo + head * HD + d] = 0.f;
        }
        return;
    }
    // Key tiles start at a token index aligned to 4 (16 bytes of fp32): the inner TMA coordinate of the transposed
    // V must be 16-byte aligned; keys outside [k0, k0 + kl) are masked in the softmax.
    const int ka = k0 & ~3;
    const int n_kt = (k0 - ka + kl + BKEY - 1) / BKEY;
    const int n_it = 2 * n_kt;                                   // pass 1 (max) + pass 2 (exp, PV)

    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* sQhi = base;
    unsigned char* sQlo = base + Q_BYTES;
    auto stage = [&](int s) { return base + 2 * Q_BYTES + s * STAGE_BYTES; };
    auto sKhi = [&](int s) { return stage(s); };
    auto sKlo = [&](int s) { return stage(s) + K_BYTES; };
    auto sVhi = [&](int s, int h) { return stage(s) + 2 * K_BYTES + h * V_HALF; };
    auto sVlo = [&](int s, int h) { return stage(s) + 2 * K_BYTES + (2 + h) * V_HALF; };
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + 2 * Q_BYTES + 2 * STAGE_BYTES);
    uint64_t* q_full = bars;            // 1
    uint64_t* kv_full = bars + 1;       // [2] TMA landed
    uint64_t* kv_empty = bars + 3;      // [2] every consumer warp's MMAs that read the stage retired (8 arrivals)

    if (warp == 8 && lane == 0) {
        tc::mbar_init(q_full, 1);
        for (int i = 0; i < 2; ++i) { tc::mbar_init(&kv_full[i], 1); tc::mbar_init(&kv_empty[i], 8); }
        tc::fence_barrier_init();
        tc::tma_prefetch_desc(&tmQ); tc::tma_prefetch_desc(&tmK); tc::tma_prefetch_desc(&tmVt);
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            tc::mbar_arrive_expect_tx(q_full, 2 * Q_BYTES);
            tc::tma_load_2d(sQhi, &tmQ, q_full, head * HD, q0);
            tc::tma_load_2d(sQlo, &tmQ, q_full, E + head * HD, q0);
            for (int it = 0; it < n_it; ++it) {
                const int s = it & 1;
                const uint32_t ph = (it >> 1) & 1;
                const int kt = it < n_kt ? it : it - n_kt;
                const int key0 = ka + kt * BKEY;
                tc::mbar_wait(&kv_empty[s], ph ^ 1);
                if (it < n_kt) {                                 // pass 1: K_hi only
                    tc::mbar_arrive_expect_tx(&kv_full[s], K_BYTES);
                    tc::tma_load_2d(sKhi(s), &tmK, &kv_full[s], 2 * E + head * HD, key0);
                } else {
                    tc::mbar_arrive_expect_tx(&kv_full[s], 2 * K_BYTES + 4 * V_HALF);
                    tc::tma_load_2d(sKhi(s), &tmK, &kv_full[s], 2 * E + head * HD, key0);
                    tc::tma_load_2d(sKlo(s), &tmK, &kv_full[s], 3 * E + head * HD, key0);
                    tc::tma_load_2d(sVhi(s, 0), &tmVt, &kv_full[s], key0, head * HD);
                    tc::tma_load_2d(sVhi(s, 1), &tmVt, &kv_full[s], key0 + 32, head * HD);
                    tc::tma_load_2d(sVlo(s, 0), &tmVt, &kv_full[s], key0, E + head * HD);
                    tc::tma_load_2d(sVlo(s, 1), &tmVt, &kv_full[s], key0 + 32, E + head * HD);
                }
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;             // this thread's query rows: row0 and row0 + 8
    const int src_a = (lane & ~3) | (t >> 1), src_b = src_a + 2; // quad lanes holding columns t and t + 4
    const bool odd = t & 1;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[HD / 2];
#pragma unroll
    for (int j = 0; j < HD / 2; ++j) o[j] = 0.f;
    tc::mbar_wait(q_full, 0);
    const uint64_t dQhi = tc::gmma_desc_sw128(tc::smem_u32(sQhi + wg * 64 * 128));
    const uint64_t dQlo = tc::gmma_desc_sw128(tc::smem_u32(sQlo + wg * 64 * 128));
    float sc[BKEY / 2];
    for (int it = 0; it < n_kt; ++it) {                           // pass 1
        const int s = it & 1;
        const int jlo = max(0, k0 - (ka + it * BKEY));          // keys [jlo, jhi) of this tile belong to the problem
        const int jhi = min(BKEY, k0 + kl - (ka + it * BKEY));
        tc::mbar_wait(&kv_full[s], (it >> 1) & 1);
        const uint64_t dKhi = tc::gmma_desc_sw128(tc::smem_u32(sKhi(s)));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 8; ++k)                          // k-step = 8 tf32 = 32 bytes
            tc::wgmma_tf32_ss_n64(sc, dQhi + (uint64_t)(2 * k), dKhi + (uint64_t)(2 * k), k != 0);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&kv_empty[s]);
#pragma unroll
        for (int i = 0; i < BKEY / 2; ++i) {
            const int j = 8 * (i >> 2) + 2 * t + (i & 1);
            if (j >= jlo && j < jhi) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], sc[i]);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {                                 // row maximum over the quad that shares the row
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
    }
    for (int it = n_kt; it < n_it; ++it) {                        // pass 2
        const int s = it & 1;
        const int kt = it - n_kt;
        const int jlo = max(0, k0 - (ka + kt * BKEY));
        const int jhi = min(BKEY, k0 + kl - (ka + kt * BKEY));
        tc::mbar_wait(&kv_full[s], (it >> 1) & 1);
        const uint64_t dKhi = tc::gmma_desc_sw128(tc::smem_u32(sKhi(s)));
        const uint64_t dKlo = tc::gmma_desc_sw128(tc::smem_u32(sKlo(s)));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 8; ++k) {
            const uint64_t adv = (uint64_t)(2 * k);
            tc::wgmma_tf32_ss_n64(sc, dQlo + adv, dKhi + adv, k != 0);      // small terms first
            tc::wgmma_tf32_ss_n64(sc, dQhi + adv, dKlo + adv, 1);
            tc::wgmma_tf32_ss_n64(sc, dQhi + adv, dKhi + adv, 1);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < BKEY / 2; ++i) {
            const int j = 8 * (i >> 2) + 2 * t + (i & 1);
            const float p = (j >= jlo && j < jhi) ? fast_exp2(sc[i] - m[(i >> 1) & 1]) : 0.f;
            l[(i >> 1) & 1] += p;
            sc[i] = p;
        }
        // accumulator layout (row g: columns 8j + 2t, +1) -> A fragments of k-step j (row g: columns t, t + 4)
        uint32_t phi[BKEY / 8][4], plo[BKEY / 8][4];
#pragma unroll
        for (int j = 0; j < BKEY / 8; ++j)
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                const float e0 = sc[4 * j + 2 * r], e1 = sc[4 * j + 2 * r + 1];
                const float xa0 = __shfl_sync(0xffffffffu, e0, src_a), xa1 = __shfl_sync(0xffffffffu, e1, src_a);
                const float xb0 = __shfl_sync(0xffffffffu, e0, src_b), xb1 = __shfl_sync(0xffffffffu, e1, src_b);
                const float pa = odd ? xa1 : xa0, pb = odd ? xb1 : xb0;
                phi[j][r] = tf32_rn(pa);
                plo[j][r] = tf32_rn(pa - __uint_as_float(phi[j][r]));
                phi[j][2 + r] = tf32_rn(pb);
                plo[j][2 + r] = tf32_rn(pb - __uint_as_float(phi[j][2 + r]));
            }
        float ot[HD / 2];
        tc::wgmma_fence();
#pragma unroll
        for (int j = 0; j < BKEY / 8; ++j) {
            const int h = j >> 2;
            const uint64_t adv = (uint64_t)(2 * (j & 3));
            const uint64_t dVhi = tc::gmma_desc_sw128(tc::smem_u32(sVhi(s, h))) + adv;
            const uint64_t dVlo = tc::gmma_desc_sw128(tc::smem_u32(sVlo(s, h))) + adv;
            tc::wgmma_tf32_n32(ot, plo[j], dVhi, j != 0);
            tc::wgmma_tf32_n32(ot, phi[j], dVlo, 1);
            tc::wgmma_tf32_n32(ot, phi[j], dVhi, 1);
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(&kv_empty[s]);
#pragma unroll
        for (int j = 0; j < HD / 2; ++j) o[j] += ot[j];
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = row0 + 8 * r;
        if (qt * BQ + row >= ql) continue;
        const float inv = l[r] > 0.f ? 1.f / l[r] : 0.f;
        float* dst = O + (size_t)(q0 + row) * ldo + head * HD;
#pragma unroll
        for (int j = 0; j < HD / 8; ++j)
            *reinterpret_cast<float2*>(dst + 8 * j + 2 * t) = make_float2(o[4 * j + 2 * r] * inv, o[4 * j + 2 * r + 1] * inv);
    }
}

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

// row-major fp32 matrix [rows, cols] with leading dimension ld; box = [32 cols, box_rows], 128-byte swizzle
bool make_map_f32(CUtensorMap* m, const void* ptr, long long rows, long long cols, long long ld, int box_rows) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {32u, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

extern "C" int regtr_mha_tf32_tc_fwd(const float* qk4, int ld4, const float* vt2, int ld_vt, int n_tokens, float* O,
                                     int ldo, const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                                     const int32_t* k_len, int n_problems, int max_q_len, const int32_t* tile_base,
                                     int max_tiles, int n_heads, int head_dim, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_problems < 0 || max_q_len < 0 || n_heads <= 0 || n_tokens < 0 || max_tiles < 0) return REGTR_ERR_ARG;
    if (head_dim != HD) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || max_q_len == 0 || n_tokens == 0 || (tile_base && max_tiles == 0)) return REGTR_OK;
    if (!qk4 || !vt2 || !O || !q_start || !q_len || !k_start || !k_len) return REGTR_ERR_ARG;
    const int E = n_heads * HD;
    if ((ld4 & 3) || (ld_vt & 3) || ld4 < 4 * E || ((uintptr_t)qk4 & 15) || ((uintptr_t)vt2 & 15) || (ldo & 3) ||
        n_problems > 65535)
        return REGTR_ERR_UNSUPPORTED;
    CUtensorMap tQ, tK, tV;
    if (!make_map_f32(&tQ, qk4, n_tokens, 4 * E, ld4, BQ) || !make_map_f32(&tK, qk4, n_tokens, 4 * E, ld4, BKEY) ||
        !make_map_f32(&tV, vt2, 2 * E, ld_vt, ld_vt, HD))
        return REGTR_ERR_ARG;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(k_mha_tf32_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
        if (e != cudaSuccess) return -(1000 + (int)e);
        attr_set = true;
    }
    const dim3 grid = tile_base ? dim3(max_tiles, n_heads, 1) : dim3(regtr_cdiv(max_q_len, BQ), n_heads, n_problems);
    k_mha_tf32_tc<<<grid, THREADS, SMEM_BYTES, st>>>(tQ, tK, tV, O, ldo, E, q_start, q_len, k_start, k_len, tile_base,
                                                 n_problems);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}
