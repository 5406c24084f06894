// Variable-length multi-head attention core on the Hopper tensor cores (bf16 operands, fp32 accumulation,
// fp32 softmax) -- the "fast" precision mode of the MHA core of TransformerCrossEncoderLayer.forward_pre
// (reference src/models/transformer/transformers.py:197-226).  head_dim = 32.
//
// Inputs come from the in-projection GEMM's bf16 epilogue (gemm_tc.cu, mode QKV_BF16):
//   QK  [N_tokens, 2E] bf16 row-major : columns [0,E) = q, [E,2E) = k          (TMA, SWIZZLE_64B)
//   Vt  [E, ld_vt]     bf16           : v transposed (one row per head-dim channel, tokens
//                                        contiguous) so that P*V is a K-major x K-major MMA (TMA, SWIZZLE_128B)
// CTA = (problem, head, tile of 128 queries); 9 warps:
//   warp 8     TMA producer (Q once; K / Vt tiles of 64 keys, 2 stages)
//   warps 0-7  two consumer warpgroups, queries [0, 64) and [64, 128): S = Q K^T (wgmma m64n64k16, both operands
//              from shared memory), O += P V (m64n32k16, P from registers: the bf16 A fragment of a 16-key step is
//              exactly the accumulator layout of the two 8-key column blocks it covers)
// Two passes over the keys -- pass 1: exact row maximum; pass 2: p = exp2((s - max) * scale*log2e), row sums in
// registers -- so the accumulator never needs an online-softmax rescale.
#include <cuda_bf16.h>

#include "common.cuh"
#include "tc.cuh"

namespace {

constexpr int HD = 32;          // head dim
constexpr int BQ = 128;         // queries per CTA
constexpr int BKEY = 64;        // keys per tile
constexpr int THREADS = 288;

constexpr int Q_BYTES = BQ * HD * 2;        // 8 KB   (rows of 64 B)
constexpr int K_BYTES = BKEY * HD * 2;      // 4 KB
constexpr int V_BYTES = HD * BKEY * 2;      // 4 KB   (32 rows of 128 B)
constexpr int SMEM_BYTES = Q_BYTES + 2 * K_BYTES + 2 * V_BYTES + 1024 + 256;

__global__ void __launch_bounds__(THREADS, 2)
k_mha_bf16_tc(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
              const __grid_constant__ CUtensorMap tmVt, float* __restrict__ O, int ldo, int E,
              const int32_t* __restrict__ q_start, const int32_t* __restrict__ q_len,
              const int32_t* __restrict__ k_start, const int32_t* __restrict__ k_len, float scale_log2e) {
    extern __shared__ unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int prob = blockIdx.z, head = blockIdx.y, qt = blockIdx.x;
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
    // Key tiles start at a token index aligned to 8 (16 bytes of bf16): the inner TMA coordinate of
    // the transposed V must be 16-byte aligned; keys outside [k0, k0+kl) are masked in the softmax.
    const int ka = k0 & ~7;
    const int n_kt = (k0 - ka + kl + BKEY - 1) / BKEY;
    const int n_it = 2 * n_kt;                                   // pass 1 (max) + pass 2 (exp, PV)

    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* sQ = base;
    auto sK = [&](int s) { return base + Q_BYTES + s * K_BYTES; };
    auto sV = [&](int s) { return base + Q_BYTES + 2 * K_BYTES + s * V_BYTES; };
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + Q_BYTES + 2 * K_BYTES + 2 * V_BYTES);
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
            tc::mbar_arrive_expect_tx(q_full, Q_BYTES);
            tc::tma_load_2d(sQ, &tmQ, q_full, head * HD, q0);
            for (int it = 0; it < n_it; ++it) {
                const int s = it & 1;
                const uint32_t ph = (it >> 1) & 1;
                const int kt = it < n_kt ? it : it - n_kt;
                tc::mbar_wait(&kv_empty[s], ph ^ 1);
                const bool second = it >= n_kt;
                tc::mbar_arrive_expect_tx(&kv_full[s], K_BYTES + (second ? V_BYTES : 0));
                tc::tma_load_2d(sK(s), &tmK, &kv_full[s], E + head * HD, ka + kt * BKEY);
                if (second) tc::tma_load_2d(sV(s), &tmVt, &kv_full[s], ka + kt * BKEY, head * HD);
            }
        }
        return;
    }

    const int wg = warp >> 2;
    const int g = lane >> 2, t = lane & 3;
    const int row0 = wg * 64 + (warp & 3) * 16 + g;             // this thread's query rows: row0 and row0 + 8
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    float o[HD / 2];
#pragma unroll
    for (int j = 0; j < HD / 2; ++j) o[j] = 0.f;
    tc::mbar_wait(q_full, 0);
    const uint64_t dQ = tc::gmma_desc_sw64(tc::smem_u32(sQ + wg * 64 * 64));
    float sc[BKEY / 2];
    for (int it = 0; it < n_kt; ++it) {                           // pass 1
        const int s = it & 1;
        const int jlo = max(0, k0 - (ka + it * BKEY));          // keys [jlo, jhi) of this tile belong to the problem
        const int jhi = min(BKEY, k0 + kl - (ka + it * BKEY));
        tc::mbar_wait(&kv_full[s], (it >> 1) & 1);
        const uint64_t dK = tc::gmma_desc_sw64(tc::smem_u32(sK(s)));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; ++k)                         // k-step = 16 bf16 = 32 bytes
            tc::wgmma_bf16_ss_n64(sc, dQ + (uint64_t)(2 * k), dK + (uint64_t)(2 * k), k != 0);
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
    const float mm[2] = {m[0] * scale_log2e, m[1] * scale_log2e};
    for (int it = n_kt; it < n_it; ++it) {                        // pass 2
        const int s = it & 1;
        const int kt = it - n_kt;
        const int jlo = max(0, k0 - (ka + kt * BKEY));
        const int jhi = min(BKEY, k0 + kl - (ka + kt * BKEY));
        tc::mbar_wait(&kv_full[s], (it >> 1) & 1);
        const uint64_t dK = tc::gmma_desc_sw64(tc::smem_u32(sK(s)));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < HD / 16; ++k)
            tc::wgmma_bf16_ss_n64(sc, dQ + (uint64_t)(2 * k), dK + (uint64_t)(2 * k), k != 0);
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        uint32_t pa[BKEY / 16][4];                                // A fragments of the four 16-key steps
#pragma unroll
        for (int i = 0; i < BKEY / 2; i += 2) {
            const int j = 8 * (i >> 2) + 2 * t, r = (i >> 1) & 1;
            const float p0 = (j >= jlo && j < jhi) ? exp2f(fmaf(sc[i], scale_log2e, -mm[r])) : 0.f;
            const float p1 = (j + 1 >= jlo && j + 1 < jhi) ? exp2f(fmaf(sc[i + 1], scale_log2e, -mm[r])) : 0.f;
            const __nv_bfloat162 b = __floats2bfloat162_rn(p0, p1);
            // the row sum uses the SAME rounded values the tensor core multiplies with V
            l[r] += __low2float(b) + __high2float(b);
            pa[i >> 3][(i >> 1) & 3] = *reinterpret_cast<const uint32_t*>(&b);
        }
        float ot[HD / 2];
        const uint64_t dV = tc::gmma_desc_sw128(tc::smem_u32(sV(s)));
        tc::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BKEY / 16; ++k) tc::wgmma_bf16_n32(ot, pa[k], dV + (uint64_t)(2 * k), k != 0);
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

bool make_map_bf16(CUtensorMap* m, const void* ptr, long long rows, long long cols, long long ld, int box_cols,
                   int box_rows, CUtensorMapSwizzle sw) {
    EncodeTiledFn enc = encode_fn();
    if (!enc) return false;
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
    cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

extern "C" int regtr_mha_bf16_tc_fwd(const void* QK, int ld_qk, const void* Vt, int ld_vt, int n_tokens, float* O,
                                     int ldo, const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                                     const int32_t* k_len, int n_problems, int max_q_len, int n_heads, int head_dim,
                                     float scale, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_problems < 0 || max_q_len < 0 || n_heads <= 0 || n_tokens < 0) return REGTR_ERR_ARG;
    if (head_dim != HD) return REGTR_ERR_UNSUPPORTED;
    if (n_problems == 0 || max_q_len == 0 || n_tokens == 0) return REGTR_OK;
    if (!QK || !Vt || !O || !q_start || !q_len || !k_start || !k_len) return REGTR_ERR_ARG;
    const int E = n_heads * HD;
    if ((ld_qk & 7) || (ld_vt & 7) || ((uintptr_t)QK & 15) || ((uintptr_t)Vt & 15) || (ldo & 3) || n_problems > 65535)
        return REGTR_ERR_UNSUPPORTED;
    CUtensorMap tQ, tK, tV;
    if (!make_map_bf16(&tQ, QK, n_tokens, 2 * E, ld_qk, HD, BQ, CU_TENSOR_MAP_SWIZZLE_64B) ||
        !make_map_bf16(&tK, QK, n_tokens, 2 * E, ld_qk, HD, BKEY, CU_TENSOR_MAP_SWIZZLE_64B) ||
        !make_map_bf16(&tV, Vt, E, ld_vt, ld_vt, BKEY, HD, CU_TENSOR_MAP_SWIZZLE_128B))
        return REGTR_ERR_ARG;
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(k_mha_bf16_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
        if (e != cudaSuccess) return -(1000 + (int)e);
        attr_set = true;
    }
    dim3 grid(regtr_cdiv(max_q_len, BQ), n_heads, n_problems);
    k_mha_bf16_tc<<<grid, THREADS, SMEM_BYTES, st>>>(tQ, tK, tV, O, ldo, E, q_start, q_len, k_start, k_len,
                                                 scale * 1.4426950408889634f);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}
