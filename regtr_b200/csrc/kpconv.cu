// KPConv encoder kernels: neighbour gather + kernel-point influence + aggregation
// (the HBM-bound "gather" of the north star), max-pool gather, and the
// [Nq, 15*Cin] x [15*Cin, Cout] weight contraction.
//
// Reference behaviour replaced (paths relative to /root/reference/src):
//   models/backbone_kpconv/kpconv_blocks.py:269-414  KPConv.forward (rigid, linear, sum)
//   models/backbone_kpconv/kpconv_blocks.py:127-143  max_pool
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int KP = 15;          // kernel points (config num_kernel_points)
constexpr int KPP = 16;         // padded
constexpr int AGG_WARPS = 8;

// flags[r] = (sum_c x[r,c] > 0): the reference counts a neighbour only when its feature
// row sums to a positive number (kpconv_blocks.py:409-412).  Summed in fp64 so that the
// sign is the mathematically exact one whenever |sum| is above fp32 rounding noise.
__global__ void k_row_flags(const float* __restrict__ x, int n, int C, uint8_t* __restrict__ flags) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n) return;
    double acc = 0.0;
    for (int c = lane; c < C; c += 32) acc += (double)x[(size_t)warp * C + c];
    acc = warp_sum(acc);
    if (lane == 0) flags[warp] = acc > 0.0;
}

// Capacity-shaped launches: rows at or beyond the real count n are padding.  Their only consumer is a GEMM
// that works in 128-row tiles, skips tiles beyond n and never stores rows >= n, so padding rows need
// defined (zero) contents only inside the tile that straddles n; the rest of the capacity is left untouched.
__device__ __forceinline__ int pad_band_end(int n) { return (n + 127) & ~127; }

// Phase 1 (lanes own neighbours): compact the valid (non-shadow) neighbours of one query into
// shared memory as (relative position, id) and count those whose feature row sums to > 0.
// Phase 2 (lanes own (neighbour, kernel point) pairs, 16 per neighbour so that all 32 lanes stay
// busy): linear influence  h = max(0, 1 - |rel - kp| / extent)  into w_s[k][16] (slot 15 = 0).
__device__ __forceinline__ void stage_neighbours(const float* __restrict__ s, const int32_t* __restrict__ idx_row,
                                                 const uint8_t* __restrict__ flags, const float* __restrict__ kp_s,
                                                 float qx, float qy, float qz, int Ns, int K, float inv_extent,
                                                 float* __restrict__ w_s, float4* __restrict__ rel_s,
                                                 int* __restrict__ id_s, int lane, int& n_valid, int& n_counted) {
    int base = 0, counted = 0;
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int kk = k0 + lane;
        int id = Ns;
        if (kk < K) id = idx_row[kk];
        const bool valid = (id >= 0) && (id < Ns);
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const int pos = base + __popc(m & ((1u << lane) - 1u));
            rel_s[pos] = make_float4(s[3 * id + 0] - qx, s[3 * id + 1] - qy, s[3 * id + 2] - qz, 0.f);
            id_s[pos] = id;
            counted += flags[id];
        }
        base += __popc(m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) counted += __shfl_xor_sync(0xffffffffu, counted, o);
    // pad the neighbour list to a multiple of 4 with copies of a valid id and ZERO influences, so that
    // the aggregation loop needs no bounds predicates
    const int padded = (base + 3) & ~3;
    if (lane < padded - base) { id_s[base + lane] = base > 0 ? id_s[0] : 0; rel_s[base + lane] = make_float4(0.f, 0.f, 0.f, 0.f); }
    __syncwarp();
    // lane -> fixed kernel point p = lane & 15 (held in registers), neighbours k = (lane >> 4) + 2 r
    const int p = lane & 15;
    const bool real = p < KP;
    const float kx = real ? kp_s[3 * p + 0] : 0.f, ky = real ? kp_s[3 * p + 1] : 0.f, kz = real ? kp_s[3 * p + 2] : 0.f;
    for (int k = lane >> 4; k < padded; k += 2) {
        float w = 0.f;
        if (real && k < base) {
            const float4 r = rel_s[k];
            const float dx = r.x - kx, dy = r.y - ky, dz = r.z - kz;
            const float d2 = dx * dx + dy * dy + dz * dz;
            const float d = d2 > 0.f ? d2 * rsqrtf(d2) : 0.f;          // |.|: <= 2 ulp, far inside the tolerance
            w = fmaxf(0.f, 1.f - d * inv_extent);
        }
        w_s[k * KPP + p] = w;
    }
    __syncwarp();
    n_valid = base;
    n_counted = counted;
}

// ---- aggregation on the tensor cores ---------------------------------------------------------------
// Per query the aggregation is a tiny GEMM  wf[15, Cin] = H[15, n] @ X[n, Cin]  (H = influences of the
// n <= K valid neighbours, X = their gathered feature rows).  One warp per query runs it as
// mma.sync m16n8k8 (M = 16 kernel-point rows, k-step = 8 neighbours) with both operands built
// directly in the fragment layout -- no shared-memory staging of H and one 128-byte row read per
// neighbour (LDG.128: lane (g,t) reads channels 4g..4g+3 of neighbours t and t+4):
//   A (H^T, 16x8):  lane (g,t) computes the influences of kernel points g, g+8 on neighbours t, t+4
//   B (X, 8x8):     n-tile j takes column n=g from channel 32h + 4g + j  (a fixed channel permutation)
//   D (16x8):       lane (g,t) ends up with 8 contiguous channels 32h + 8t .. 8t+7 of rows g and g+8
// fp32 accuracy comes from the 3xTF32 split (lo*hi + hi*lo + hi*hi, round-to-nearest hi), like the GEMMs.
// round-to-nearest (ties away) TF32 head of a finite fp32 value: two integer ops instead of cvt.rna's
// special-case sequence; the tail x - head is exact in fp32 and the tensor core truncates it to TF32.
__device__ __forceinline__ uint32_t tf32_head(float x) { return (__float_as_uint(x) + 0x1000u) & 0xffffe000u; }
__device__ __forceinline__ void mma_tf32_16x8x8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// linear influence max(0, 1 - |rel - kp| / extent); sqrt.approx: one MUFU, exact 0 at 0, <= 1 ulp
__device__ __forceinline__ float influence(const float4 r, float kx, float ky, float kz, float inv_extent) {
    const float dx = r.x - kx, dy = r.y - ky, dz = r.z - kz;
    const float d2 = dx * dx + dy * dy + dz * dz;
    float d;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(d) : "f"(d2));
    return fmaxf(0.f, fmaf(-d, inv_extent, 1.f));
}

// NH = 32-channel groups per warp; blockIdx.y selects the warp's channel slice [32 NH y, 32 NH (y+1)) so
// that small levels with wide features still fill the machine (each slice repeats the cheap staging).
template <int NH, int MINB>
__global__ void __launch_bounds__(AGG_WARPS * 32, MINB)
k_kpconv_agg_mma(const float* __restrict__ q, const float* __restrict__ s, const int32_t* __restrict__ idx,
                 const float* __restrict__ x, const uint8_t* __restrict__ flags, const float* __restrict__ kp,
                 int Nq, int Ns, const int32_t* __restrict__ nq_dev, const int32_t* __restrict__ ns_dev, int K, int Cin,
                 float inv_extent, float* __restrict__ wf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Kp = (K + 7) & ~7;
    // per warp: rows[Kp][32 NH] (staged feature rows, 16-byte chunks swizzled) | rel[Kp] (float4) | id[Kp]
    constexpr int ROW = 32 * NH;                  // floats per staged row
    float* rows_s = reinterpret_cast<float*>(smem_raw) + (size_t)warp * Kp * (ROW + 5);
    float4* rel_s = reinterpret_cast<float4*>(rows_s + Kp * ROW);
    int* id_s = reinterpret_cast<int*>(rows_s + Kp * (ROW + 4));
    const int qi = blockIdx.x * AGG_WARPS + warp;
    if (qi >= Nq) return;
    if (ns_dev) Ns = min(Ns, *ns_dev);
    const int c_base = blockIdx.y * (32 * NH);
    const int g = lane >> 2, t = lane & 3;
    float* out = wf + (size_t)qi * (KP * Cin) + c_base;
    if (nq_dev && qi >= *nq_dev) {               // capacity padding row
        if (qi < pad_band_end(*nq_dev))
            for (int p = g; p < KP; p += 8)
#pragma unroll
                for (int h = 0; h < NH; ++h) {
                    reinterpret_cast<float4*>(out + p * Cin + 32 * h + 8 * t)[0] = make_float4(0.f, 0.f, 0.f, 0.f);
                    reinterpret_cast<float4*>(out + p * Cin + 32 * h + 8 * t)[1] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
        return;
    }
    // compact the valid (non-shadow) neighbours; count those whose feature row sums to > 0
    const float qx = q[3 * qi], qy = q[3 * qi + 1], qz = q[3 * qi + 2];
    const int32_t* idx_row = idx + (size_t)qi * K;
    int base = 0, counted = 0;
#pragma unroll 1
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int kk = k0 + lane;
        int id = Ns;
        if (kk < K) id = idx_row[kk];
        const bool valid = (id >= 0) && (id < Ns);
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const int pos = base + __popc(m & ((1u << lane) - 1u));
            rel_s[pos] = make_float4(s[3 * id + 0] - qx, s[3 * id + 1] - qy, s[3 * id + 2] - qz, 0.f);
            id_s[pos] = id;
            counted += flags[id];
        }
        base += __popc(m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) counted += __shfl_xor_sync(0xffffffffu, counted, o);
    // pad to a whole k-step with a loadable row id and a far-away position (influence exactly 0)
    const int padded = (base + 7) & ~7;
    if (lane < padded - base) { id_s[base + lane] = base > 0 ? id_s[0] : 0; rel_s[base + lane] = make_float4(1e6f, 1e6f, 1e6f, 0.f); }
    __syncwarp();

    // stage ALL neighbour rows of the query with cp.async (16 bytes per lane): every row is in flight at
    // once instead of one k-step at a time.  Chunk c of row n lands in slot (c + 2 (n & 3)) & 7 of its
    // 128-byte group so that the LDS.128 fragment reads below are bank-conflict free.
    {
        constexpr int CPR = 8 * NH, RPI = 32 / CPR;            // 16-byte chunks per row, rows per warp instruction
        const int c = lane % CPR, rg = lane / CPR;
        const float* xs = x + c_base + 4 * c;
        uint32_t dst = (uint32_t)__cvta_generic_to_shared(rows_s) + (uint32_t)(rg * ROW + (c & ~7) * 4) * 4u;
        for (int n = rg; n < padded; n += RPI, dst += RPI * ROW * 4) {
            const float* src = xs + (size_t)id_s[n] * Cin;
            asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(((c + 2 * n) & 7) * 16)), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }

    const float ax = __ldg(kp + 3 * g), ay = __ldg(kp + 3 * g + 1), az = __ldg(kp + 3 * g + 2);
    const bool row_b = g + 8 < KP;                // M = 16 rows, kernel points 0..14; row 15: far away -> 0
    const float bx = row_b ? __ldg(kp + 3 * g + 24) : -1e6f, by = row_b ? __ldg(kp + 3 * g + 25) : -1e6f,
                bz = row_b ? __ldg(kp + 3 * g + 26) : -1e6f;

    float acc[NH][4][4];
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[h][j][e] = 0.f;

    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncwarp();
    for (int k0 = 0; k0 < padded; k0 += 8) {
        const int n0 = k0 + t, n1 = n0 + 4;        // n0 & 3 == n1 & 3 == t
        const float* row0 = rows_s + n0 * ROW + 4 * ((g + 2 * t) & 7);
        const float* row1 = rows_s + n1 * ROW + 4 * ((g + 2 * t) & 7);
        float4 v0[NH], v1[NH];
#pragma unroll
        for (int h = 0; h < NH; ++h) {
            v0[h] = *reinterpret_cast<const float4*>(row0 + 32 * h);
            v1[h] = *reinterpret_cast<const float4*>(row1 + 32 * h);
        }
        const float4 r0 = rel_s[n0], r1 = rel_s[n1];
        const float w[4] = {influence(r0, ax, ay, az, inv_extent), influence(r0, bx, by, bz, inv_extent),
                            influence(r1, ax, ay, az, inv_extent), influence(r1, bx, by, bz, inv_extent)};
        uint32_t a_hi[4], a_lo[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) { a_hi[e] = tf32_head(w[e]); a_lo[e] = __float_as_uint(w[e] - __uint_as_float(a_hi[e])); }
#pragma unroll
        for (int h = 0; h < NH; ++h) {
            const float b0f[4] = {v0[h].x, v0[h].y, v0[h].z, v0[h].w};
            const float b1f[4] = {v1[h].x, v1[h].y, v1[h].z, v1[h].w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const uint32_t h0 = tf32_head(b0f[j]), h1 = tf32_head(b1f[j]);
                const uint32_t l0 = __float_as_uint(b0f[j] - __uint_as_float(h0));
                const uint32_t l1 = __float_as_uint(b1f[j] - __uint_as_float(h1));
                mma_tf32_16x8x8(acc[h][j], a_lo, h0, h1);
                mma_tf32_16x8x8(acc[h][j], a_hi, l0, l1);
                mma_tf32_16x8x8(acc[h][j], a_hi, h0, h1);
            }
        }
    }

    float inv;                                    // 1 / max(count, 1): one MUFU (<= 1 ulp)
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"((float)max(counted, 1)));
#pragma unroll
    for (int h = 0; h < NH; ++h) {
        float* o = out + g * Cin + 32 * h + 8 * t;
        reinterpret_cast<float4*>(o)[0] = make_float4(acc[h][0][0] * inv, acc[h][1][0] * inv, acc[h][2][0] * inv, acc[h][3][0] * inv);
        reinterpret_cast<float4*>(o)[1] = make_float4(acc[h][0][1] * inv, acc[h][1][1] * inv, acc[h][2][1] * inv, acc[h][3][1] * inv);
        if (row_b) {
            float* o2 = o + 8 * Cin;
            reinterpret_cast<float4*>(o2)[0] = make_float4(acc[h][0][2] * inv, acc[h][1][2] * inv, acc[h][2][2] * inv, acc[h][3][2] * inv);
            reinterpret_cast<float4*>(o2)[1] = make_float4(acc[h][0][3] * inv, acc[h][1][3] * inv, acc[h][2][3] * inv, acc[h][3][3] * inv);
        }
    }
}

// ---- software-pipelined persistent variant (the default for Cin % 32 == 0, K <= 64) -------------------------
// k_kpconv_agg_mma above runs one query per warp start to finish: index row -> support coordinates -> feature
// rows are three DEPENDENT global round trips (~2000 cycles) in front of ~800 issue slots of work, and the
// profile showed the SM idle 47 % of the time waiting on them (long-scoreboard 3.7 warps per issue).  Here
// every warp is persistent and walks a strided list of work items (query, 32-channel slice) with the chain
// pipelined ACROSS items: while item i runs on the tensor cores, the feature rows of item i+1 are in flight
// (cp.async into the other half of a double buffer), the coordinates of item i+2 are being loaded into
// registers and the index row of item i+3 has been requested.  Same fragment construction, same arithmetic
// and the same output as k_kpconv_agg_mma<1>.
constexpr int PIPE_WARPS = 4;

struct AggItem {            // registers that travel with an item through the load stages
    int id0, id1;           // neighbour ids of lanes (lane, lane + 32) of the index row
    float x0, y0, z0, x1, y1, z1;
    float qx, qy, qz;
    int f0, f1;             // "row sums to > 0" flags of the two neighbours
};

// NH: 32-channel halves per work item.  NH = 2 (Cin % 64 == 0) shares the index / coordinate / influence work of a
// query between two channel halves: 65 instead of 92 issue slots per (8 neighbours, 32 channels) in the main loop.
template <int NH>
__global__ void __launch_bounds__(PIPE_WARPS * 32, NH == 1 ? 4 : 2)
k_kpconv_agg_pipe(const float* __restrict__ q, const float* __restrict__ s, const int32_t* __restrict__ idx,
                  const float* __restrict__ x, const uint8_t* __restrict__ flags, const float* __restrict__ kp,
                  int Nq, int Ns, const int32_t* __restrict__ nq_dev, const int32_t* __restrict__ ns_dev, int K, int Cin,
                  int log2_slices, float inv_extent, float* __restrict__ wf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Kp = (K + 7) & ~7;
    constexpr int ROW = 32 * NH;
    // per warp, two buffers of: rows[Kp][32 NH] (16-byte chunks swizzled per 128-byte group) | rel[Kp] (float4) | id[Kp]
    const int buf_floats = Kp * (ROW + 5);
    float* wbase = reinterpret_cast<float*>(smem_raw) + (size_t)warp * 2 * buf_floats;
    if (ns_dev) Ns = min(Ns, *ns_dev);
    const int nq_real = nq_dev ? min(Nq, *nq_dev) : Nq;
    const int W = gridDim.x * PIPE_WARPS, w = blockIdx.x * PIPE_WARPS + warp;
    const int g = lane >> 2, t = lane & 3;
    // capacity padding rows: zero the band up to the next multiple of 128 (the consumer GEMM's last tile)
    if (nq_dev) {
        const int band_end = min(pad_band_end(nq_real), Nq);
        for (int r = nq_real + w; r < band_end; r += W) {
            float4* o = reinterpret_cast<float4*>(wf + (size_t)r * (KP * Cin));
            for (int i = lane; i < KP * Cin / 4; i += 32) o[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    const long long n_items = (long long)nq_real << log2_slices;
    const int slice_mask = (1 << log2_slices) - 1;

    const float ax = __ldg(kp + 3 * g), ay = __ldg(kp + 3 * g + 1), az = __ldg(kp + 3 * g + 2);
    const bool row_b = g + 8 < KP;                // M = 16 rows, kernel points 0..14; row 15: far away -> 0
    const float bx = row_b ? __ldg(kp + 3 * g + 24) : -1e6f, by = row_b ? __ldg(kp + 3 * g + 25) : -1e6f,
                bz = row_b ? __ldg(kp + 3 * g + 26) : -1e6f;

    // ---- stage A: request the index row of item `it`
    auto stage_idx = [&](long long it, AggItem& a) {
        a.id0 = Ns; a.id1 = Ns;
        if (it < n_items) {
            const int32_t* row = idx + (size_t)(it >> log2_slices) * K;
            if (lane < K) a.id0 = __ldg(row + lane);
            if (lane + 32 < K) a.id1 = __ldg(row + lane + 32);
        }
    };
    // ---- stage B: request the support coordinates / flags of the item's neighbours and its query point
    auto stage_coords = [&](long long it, AggItem& a) {
        const bool v0 = a.id0 >= 0 && a.id0 < Ns, v1 = a.id1 >= 0 && a.id1 < Ns;
        a.x0 = a.y0 = a.z0 = a.x1 = a.y1 = a.z1 = 0.f; a.f0 = a.f1 = 0;
        if (v0) { a.x0 = __ldg(s + 3 * a.id0); a.y0 = __ldg(s + 3 * a.id0 + 1); a.z0 = __ldg(s + 3 * a.id0 + 2); a.f0 = flags[a.id0]; }
        if (v1) { a.x1 = __ldg(s + 3 * a.id1); a.y1 = __ldg(s + 3 * a.id1 + 1); a.z1 = __ldg(s + 3 * a.id1 + 2); a.f1 = flags[a.id1]; }
        if (!v0) a.id0 = -1;
        if (!v1) a.id1 = -1;
        a.qx = a.qy = a.qz = 0.f;
        if (it < n_items) {
            const int qi = (int)(it >> log2_slices);
            a.qx = __ldg(q + 3 * qi); a.qy = __ldg(q + 3 * qi + 1); a.qz = __ldg(q + 3 * qi + 2);
        }
    };
    // ---- stage C: compact the valid neighbours into buffer `b`, start the cp.async of their feature rows.
    // Returns (padded neighbour count, counted neighbours) of the item.
    auto stage_rows = [&](long long it, const AggItem& a, int b, int& padded, int& counted) {
        float* rows_s = wbase + b * buf_floats;
        float4* rel_s = reinterpret_cast<float4*>(rows_s + Kp * ROW);
        int* id_s = reinterpret_cast<int*>(rows_s + Kp * (ROW + 4));
        const bool v0 = a.id0 >= 0, v1 = a.id1 >= 0;
        const unsigned m0 = __ballot_sync(0xffffffffu, v0), m1 = __ballot_sync(0xffffffffu, v1);
        const unsigned lt = (1u << lane) - 1u;
        const int n0 = __popc(m0);
        if (v0) { const int p = __popc(m0 & lt); rel_s[p] = make_float4(a.x0 - a.qx, a.y0 - a.qy, a.z0 - a.qz, 0.f); id_s[p] = a.id0; }
        if (v1) { const int p = n0 + __popc(m1 & lt); rel_s[p] = make_float4(a.x1 - a.qx, a.y1 - a.qy, a.z1 - a.qz, 0.f); id_s[p] = a.id1; }
        const int base = n0 + __popc(m1);
        counted = __popc(__ballot_sync(0xffffffffu, v0 && a.f0)) + __popc(__ballot_sync(0xffffffffu, v1 && a.f1));
        // pad to a whole k-step: a loadable row (row 0 exists whenever there is a valid neighbour) and a far-away
        // position, i.e. an influence of exactly 0
        padded = (base + 7) & ~7;
        if (lane < padded - base) { id_s[base + lane] = 0; rel_s[base + lane] = make_float4(1e6f, 1e6f, 1e6f, 0.f); }
        __syncwarp();
        if (it < n_items) {
            constexpr int CPR = 8 * NH, RPI = 32 / CPR;              // 16-byte chunks per row, rows per warp instruction
            const int c = lane % CPR, rg = lane / CPR;
            const float* xs = x + (size_t)((int)it & slice_mask) * ROW + 4 * c;
            uint32_t dst = (uint32_t)__cvta_generic_to_shared(rows_s) + (uint32_t)(rg * ROW + (c & ~7) * 4) * 4u;
            for (int n = rg; n < padded; n += RPI, dst += RPI * ROW * 4) {
                const float* src = xs + (size_t)id_s[n] * Cin;
                asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(dst + (uint32_t)(((c + 2 * n) & 7) * 16)), "l"(src) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    // ---- prologue: fill the pipeline
    AggItem a1, a2;                          // a1: item i+1 (coordinates requested), a2: item i+2 (index row requested)
    int pad_cur = 0, cnt_cur = 0, pad_nxt = 0, cnt_nxt = 0;
    long long it = w;
    {
        AggItem a0;
        stage_idx(it, a0); stage_idx(it + W, a1); stage_idx(it + 2LL * W, a2);
        stage_coords(it, a0); stage_coords(it + W, a1);
        stage_rows(it, a0, 0, pad_cur, cnt_cur);
    }
    int b = 0;
    for (; it < n_items; it += W, b ^= 1) {
        // rows of item i+1 (coordinates arrived during the previous item), coordinates of i+2, index row of i+3
        stage_rows(it + W, a1, b ^ 1, pad_nxt, cnt_nxt);
        a1 = a2;
        stage_coords(it + 2LL * W, a1);
        stage_idx(it + 3LL * W, a2);

        // ---- item i on the tensor cores (rows landed: only the newest cp.async group may still be in flight)
        asm volatile("cp.async.wait_group 1;" ::: "memory");
        __syncwarp();
        const float* rows_s = wbase + b * buf_floats;
        const float4* rel_s = reinterpret_cast<const float4*>(rows_s + Kp * ROW);
        float acc[NH][4][4];
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[h][j][e] = 0.f;
        for (int k0 = 0; k0 < pad_cur; k0 += 8) {
            const int n0 = k0 + t, n1 = n0 + 4;        // n0 & 3 == n1 & 3 == t
            const float* row0 = rows_s + n0 * ROW + 4 * ((g + 2 * t) & 7);
            const float* row1 = rows_s + n1 * ROW + 4 * ((g + 2 * t) & 7);
            float4 v0[NH], v1[NH];
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                v0[h] = *reinterpret_cast<const float4*>(row0 + 32 * h);
                v1[h] = *reinterpret_cast<const float4*>(row1 + 32 * h);
            }
            const float4 r0 = rel_s[n0], r1 = rel_s[n1];
            const float hw[4] = {influence(r0, ax, ay, az, inv_extent), influence(r0, bx, by, bz, inv_extent),
                                 influence(r1, ax, ay, az, inv_extent), influence(r1, bx, by, bz, inv_extent)};
            uint32_t a_hi[4], a_lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) { a_hi[e] = tf32_head(hw[e]); a_lo[e] = __float_as_uint(hw[e] - __uint_as_float(a_hi[e])); }
#pragma unroll
            for (int h = 0; h < NH; ++h) {
                const float b0f[4] = {v0[h].x, v0[h].y, v0[h].z, v0[h].w};
                const float b1f[4] = {v1[h].x, v1[h].y, v1[h].z, v1[h].w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const uint32_t h0 = tf32_head(b0f[j]), h1 = tf32_head(b1f[j]);
                    const uint32_t l0 = __float_as_uint(b0f[j] - __uint_as_float(h0));
                    const uint32_t l1 = __float_as_uint(b1f[j] - __uint_as_float(h1));
                    mma_tf32_16x8x8(acc[h][j], a_lo, h0, h1);
                    mma_tf32_16x8x8(acc[h][j], a_hi, l0, l1);
                    mma_tf32_16x8x8(acc[h][j], a_hi, h0, h1);
                }
            }
        }
        float inv;                                    // 1 / max(count, 1): one MUFU (<= 1 ulp)
        asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"((float)max(cnt_cur, 1)));
#pragma unroll
        for (int h = 0; h < NH; ++h) {
            float* o = wf + (size_t)(it >> log2_slices) * (KP * Cin) + ((int)it & slice_mask) * ROW + g * Cin + 32 * h + 8 * t;
            reinterpret_cast<float4*>(o)[0] = make_float4(acc[h][0][0] * inv, acc[h][1][0] * inv, acc[h][2][0] * inv, acc[h][3][0] * inv);
            reinterpret_cast<float4*>(o)[1] = make_float4(acc[h][0][1] * inv, acc[h][1][1] * inv, acc[h][2][1] * inv, acc[h][3][1] * inv);
            if (row_b) {
                float* o2 = o + 8 * Cin;
                reinterpret_cast<float4*>(o2)[0] = make_float4(acc[h][0][2] * inv, acc[h][1][2] * inv, acc[h][2][2] * inv, acc[h][3][2] * inv);
                reinterpret_cast<float4*>(o2)[1] = make_float4(acc[h][0][3] * inv, acc[h][1][3] * inv, acc[h][2][3] * inv, acc[h][3][3] * inv);
            }
        }
        __syncwarp();                                 // all lanes are done with buffer b before it is refilled
        pad_cur = pad_nxt; cnt_cur = cnt_nxt;
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
}

// Cin = 1 (the first block: a constant-1 input feature).  Per query the whole op is
//   wf[p] = sum_k h(rel_k - kp_p) * x[id_k] / #{k : x[id_k] > 0}       (15 numbers)
// and, FUSEd, out[c] = sum_p wf[p] W[p, c].  Lane (p = lane & 15, half = lane >> 4) sums its kernel point over
// every second neighbour straight from the staged (rel, x) quadruples: no influence table, no gather in the loop.
template <bool FUSE>
__global__ void __launch_bounds__(AGG_WARPS * 32)
k_kpconv_c1(const float* __restrict__ q, const float* __restrict__ s, const int32_t* __restrict__ idx,
            const float* __restrict__ x, const float* __restrict__ kp, const float* __restrict__ W, int Nq, int Ns,
            const int32_t* __restrict__ nq_dev, const int32_t* __restrict__ ns_dev, int K, int Cout, float inv_extent,
            float* __restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float4* rel_s = reinterpret_cast<float4*>(smem_raw) + warp * K;
    float* W_s = reinterpret_cast<float*>(reinterpret_cast<float4*>(smem_raw) + AGG_WARPS * K);
    if (FUSE) {
        for (int t = threadIdx.x; t < KP * Cout; t += blockDim.x) W_s[t] = W[t];
        __syncthreads();
    }
    if (ns_dev) Ns = min(Ns, *ns_dev);
    const int width = FUSE ? Cout : KP;
    const int nq_real = nq_dev ? min(Nq, *nq_dev) : Nq;
    const int p = lane & 15;
    const bool real = p < KP;                    // slot 15: a far-away kernel point, influence exactly 0
    const float kx = real ? __ldg(kp + 3 * p) : -1e6f, ky = real ? __ldg(kp + 3 * p + 1) : -1e6f,
                kz = real ? __ldg(kp + 3 * p + 2) : -1e6f;
    // persistent warps: the weights are staged once per CTA, the kernel points once per warp
    for (int qi = blockIdx.x * AGG_WARPS + warp; qi < Nq; qi += gridDim.x * AGG_WARPS) {
    float* o = out + (size_t)qi * width;
    if (qi >= nq_real) {                         // capacity padding row
        if (qi < pad_band_end(nq_real))
            for (int t = lane; t < width; t += 32) o[t] = 0.f;
        continue;
    }
    const float qx = q[3 * qi], qy = q[3 * qi + 1], qz = q[3 * qi + 2];
    const int32_t* idx_row = idx + (size_t)qi * K;
    int base = 0, counted = 0;
#pragma unroll 1
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int kk = k0 + lane;
        int id = Ns;
        if (kk < K) id = idx_row[kk];
        const bool valid = (id >= 0) && (id < Ns);
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const float xv = x[id];
            rel_s[base + __popc(m & ((1u << lane) - 1u))] =
                make_float4(s[3 * id + 0] - qx, s[3 * id + 1] - qy, s[3 * id + 2] - qz, xv);
            counted += xv > 0.f;                 // the reference counts rows whose feature sum is > 0
        }
        base += __popc(m);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) counted += __shfl_xor_sync(0xffffffffu, counted, off);
    __syncwarp();
    float acc = 0.f;
    for (int k = lane >> 4; k < base; k += 2) {
        const float4 r = rel_s[k];
        acc = fmaf(influence(r, kx, ky, kz, inv_extent), r.w, acc);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 16);
    float inv;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"((float)max(counted, 1)));
    const float v = acc * inv;
    if constexpr (!FUSE) {
        if (lane < KP) o[lane] = v;
    } else {
        for (int c0 = 0; c0 < Cout; c0 += 32) {  // warp-uniform trip count: the shuffles stay convergent
            const int c = c0 + lane;
            float r = 0.f;
#pragma unroll
            for (int pp = 0; pp < KP; ++pp) {
                const float wv = __shfl_sync(0xffffffffu, v, pp);
                if (c < Cout) r = fmaf(wv, W_s[pp * Cout + c], r);
            }
            if (c < Cout) o[c] = r;
        }
    }
    __syncwarp();                                // rel_s is refilled for the next query of this warp
    }
}

// Small Cin (2..16): neighbours and influences staged by stage_neighbours; then lane
// (p, half) sums w[k][p] * x[id_k][c] over its half of the neighbours, halves combined by shuffle.
__global__ void __launch_bounds__(AGG_WARPS * 32)
k_kpconv_agg_small(const float* __restrict__ q, const float* __restrict__ s, const int32_t* __restrict__ idx,
                   const float* __restrict__ x, const uint8_t* __restrict__ flags, const float* __restrict__ kp,
                   int Nq, int Ns, const int32_t* __restrict__ nq_dev, const int32_t* __restrict__ ns_dev, int K, int Cin,
                   float extent, float* __restrict__ wf) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* kp_s = reinterpret_cast<float*>(smem_raw);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int Kp = (K + 3) & ~3;
    float* w_s = kp_s + 48 + warp * (Kp * (KPP + 4 + 1));
    float4* rel_s = reinterpret_cast<float4*>(w_s + Kp * KPP);
    int* id_s = reinterpret_cast<int*>(w_s + Kp * (KPP + 4));
    if (threadIdx.x < 3 * KP) kp_s[threadIdx.x] = kp[threadIdx.x];
    __syncthreads();
    const int qi = blockIdx.x * AGG_WARPS + warp;
    if (qi >= Nq) return;
    if (ns_dev) Ns = min(Ns, *ns_dev);
    float* out = wf + (size_t)qi * (KP * Cin);
    if (nq_dev && qi >= *nq_dev) {
        if (qi < pad_band_end(*nq_dev))
            for (int t = lane; t < KP * Cin; t += 32) out[t] = 0.f;
        return;
    }
    int n_valid, n_counted;
    stage_neighbours(s, idx + (size_t)qi * K, flags, kp_s, q[3 * qi], q[3 * qi + 1], q[3 * qi + 2], Ns, K,
                     1.f / extent, w_s, rel_s, id_s, lane, n_valid, n_counted);
    const float inv = 1.f / (float)max(n_counted, 1);
    const int p = lane & 15, half = lane >> 4;
    for (int c = 0; c < Cin; ++c) {
        float acc = 0.f;
        for (int k = half; k < n_valid; k += 2) acc = fmaf(w_s[k * KPP + p], __ldg(x + (size_t)id_s[k] * Cin + c), acc);
        acc += __shfl_xor_sync(0xffffffffu, acc, 16);
        if (lane < KP) out[lane * Cin + c] = acc * inv;
    }
}

// out[q, c] = max(0-shadow, x[idx[q,k], c]) ; 4 channels per thread.
__global__ void k_max_pool(const float* __restrict__ x, const int32_t* __restrict__ idx, int Nq, int Ns,
                           const int32_t* __restrict__ ns_dev, int K, int C, float* __restrict__ out) {
    const int c4 = C >> 2;
    if (ns_dev) Ns = min(Ns, *ns_dev);
    const unsigned total = (unsigned)Nq * (unsigned)c4, stride = gridDim.x * blockDim.x;
    for (unsigned t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += stride) {     // grid-stride: long-lived CTAs
        int qi, cc;
        regtr_row_col(t, (unsigned)c4, qi, cc);
        float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
        for (int k = 0; k < K; ++k) {
            const int id = idx[(size_t)qi * K + k];
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (id >= 0 && id < Ns) v = __ldg(reinterpret_cast<const float4*>(x + (size_t)id * C) + cc);
            m.x = fmaxf(m.x, v.x); m.y = fmaxf(m.y, v.y); m.z = fmaxf(m.z, v.z); m.w = fmaxf(m.w, v.w);
        }
        reinterpret_cast<float4*>(out + (size_t)qi * C)[cc] = m;
    }
}

__global__ void k_max_pool_scalar(const float* __restrict__ x, const int32_t* __restrict__ idx, int Nq, int Ns,
                                  const int32_t* __restrict__ ns_dev, int K, int C, float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)Nq * C) return;
    if (ns_dev) Ns = min(Ns, *ns_dev);
    int qi, c;
    regtr_row_col((unsigned)t, (unsigned)C, qi, c);
    float m = -INFINITY;
    for (int k = 0; k < K; ++k) {
        const int id = idx[(size_t)qi * K + k];
        m = fmaxf(m, (id >= 0 && id < Ns) ? x[(size_t)id * C + c] : 0.f);
    }
    out[(size_t)qi * C + c] = m;
}

// out[n, o] = sum_k a[n, k] * W[k, o] for a tiny K (the first block: K = 15 * in_feats_dim = 15, which
// breaks the 16-byte TMA pitch of the tensor-core GEMM).  One thread per 4 outputs, W in smem.
__global__ void k_gemm_smallk(const float* __restrict__ a, const float* __restrict__ W, int n, int K, int Cout,
                              const int32_t* __restrict__ n_dev, float* __restrict__ out) {
    extern __shared__ float w_s[];
    for (int t = threadIdx.x; t < K * Cout; t += blockDim.x) w_s[t] = W[t];
    __syncthreads();
    if (n_dev) n = min(n, *n_dev);
    const int c4 = Cout >> 2;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * c4) return;
    int r, c;
    regtr_row_col((unsigned)t, (unsigned)c4, r, c);
    c *= 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int k = 0; k < K; ++k) {
        const float av = a[(size_t)r * K + k];
        const float4 wv = *reinterpret_cast<const float4*>(w_s + k * Cout + c);
        acc.x = fmaf(av, wv.x, acc.x); acc.y = fmaf(av, wv.y, acc.y); acc.z = fmaf(av, wv.z, acc.z); acc.w = fmaf(av, wv.w, acc.w);
    }
    *reinterpret_cast<float4*>(out + (size_t)r * Cout + c) = acc;
}

// W[K, N] (row-major) -> TF32 (hi, lo) halves of W^T, [N, K] row-major: the B operand layout of the GEMM
__global__ void k_split_transpose(const float* __restrict__ W, int K, int N, float* __restrict__ hi, float* __restrict__ lo) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)K * N) return;
    const int n = (int)(t / K), k = (int)(t % K);
    const float v = W[(size_t)k * N + n];
    uint32_t u = __float_as_uint(v);
    u += 0x0FFFu + ((u >> 13) & 1u);
    const float h = __uint_as_float(u & 0xFFFFE000u);
    float l = v - h;
    uint32_t ul = __float_as_uint(l);
    ul += 0x0FFFu + ((ul >> 13) & 1u);
    hi[t] = h;
    lo[t] = __uint_as_float(ul & 0xFFFFE000u);
}

size_t agg_smem_bytes(int K) {
    const int Kp = (K + 3) & ~3;
    return sizeof(float) * 48 + (size_t)AGG_WARPS * Kp * (KPP + 4 + 1) * sizeof(float);
}

// k_kpconv_agg_mma: per warp, Kp staged rows of 32 NH floats plus a float4 and an id per neighbour
size_t agg_mma_smem_bytes(int K, int nh) {
    const int Kp = (K + 7) & ~7;
    return (size_t)AGG_WARPS * Kp * (32 * nh + 5) * sizeof(float);
}

template <int NH, int MINB>
int launch_agg_mma(const float* q, const float* s, const int32_t* idx, const float* x, const uint8_t* flags,
                   const float* kp, int Nq, int Ns, const int32_t* nq_dev, const int32_t* ns_dev, int K, int Cin,
                   float extent, float* wf, cudaStream_t st) {
    const size_t smem = agg_mma_smem_bytes(K, NH);
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(k_kpconv_agg_mma<NH, MINB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return REGTR_ERR_UNSUPPORTED;       // K too large for the staged kernel
    }
    const dim3 grid(regtr_cdiv(Nq, AGG_WARPS), Cin / (32 * NH));
    k_kpconv_agg_mma<NH, MINB><<<grid, AGG_WARPS * 32, smem, st>>>(q, s, idx, x, flags, kp, Nq, Ns, nq_dev, ns_dev, K, Cin,
                                                                   1.f / extent, wf);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// Channel slicing of k_kpconv_agg_mma: the grid keeps at least this many warps (from the level-size sweep).
constexpr long long AGG_MMA_MIN_WARPS = 8192;
constexpr size_t SMEM_OPTIN = 227 * 1024;           // sm_90 opt-in shared memory per block

// channel groups per warp: as wide as possible while the grid still has >= AGG_MMA_MIN_WARPS warps and the staged
// rows fit in shared memory (NH = 2 up to K = 104)
int agg_mma_nh(int Nq, int K, int Cin) {
    int nh = Cin / 32 > 2 ? 2 : Cin / 32;      // staged rows: 128 NH bytes of smem per neighbour and warp
    while (nh > 1 && ((long long)Nq * (Cin / (32 * nh)) < AGG_MMA_MIN_WARPS || agg_mma_smem_bytes(K, nh) > SMEM_OPTIN))
        nh >>= 1;
    return nh;
}

}  // namespace

static inline int c1_grid(int Nq) {
    const int b = regtr_cdiv(Nq, AGG_WARPS);
    return b < 8 * REGTR_NUM_SMS ? b : 8 * REGTR_NUM_SMS;
}

extern "C" {

// wf | row flags  (what regtr_kpconv_aggregate needs; regtr_kpconv_fwd adds regtr_kpconv_fwd_ws_bytes)
size_t regtr_kpconv_ws_bytes(int Nq, int Ns, int Cin) {
    return regtr_align(sizeof(float) * (size_t)(Nq > 0 ? Nq : 1) * KP * (size_t)Cin) +
           regtr_align((size_t)(Ns > 0 ? Ns : 1));
}

// + split W^T (hi, lo) + the GEMM's own workspace
size_t regtr_kpconv_fwd_ws_bytes(int Nq, int Ns, int Cin, int Cout) {
    const size_t w = regtr_align(sizeof(float) * (size_t)KP * (size_t)(Cin > 0 ? Cin : 1) * (size_t)(Cout > 0 ? Cout : 1));
    return regtr_kpconv_ws_bytes(Nq, Ns, Cin) + 2 * w + regtr_gemm_ws_bytes(Nq, Cout, KP * Cin);
}

int regtr_kpconv_aggregate(const float* q, const float* s, const int32_t* idx, const float* x, const float* kp,
                           int Nq, int Ns, const int32_t* nq_dev, const int32_t* ns_dev, int K, int Cin, float extent,
                           float* wf, uint8_t* rowflag_ws, int flags_ready, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Nq < 0 || Ns < 0 || K <= 0 || K > 128 || Cin <= 0 || !(extent > 0.f)) return REGTR_ERR_ARG;
    if (!(Cin <= 16 || (Cin % 32 == 0 && Cin <= 256 && (Cin / 32 == 1 || Cin / 32 == 2 || Cin / 32 == 4 || Cin / 32 == 8))))
        return REGTR_ERR_UNSUPPORTED;
    if (Nq == 0) return REGTR_OK;
    if (!q || !s || !idx || !x || !kp || !wf || !rowflag_ws) return REGTR_ERR_ARG;
    if (Cin == 1 && (size_t)AGG_WARPS * K * sizeof(float4) <= 48 * 1024) {      // flags come from x itself
        k_kpconv_c1<false><<<c1_grid(Nq), AGG_WARPS * 32, (size_t)AGG_WARPS * K * sizeof(float4), st>>>(
            q, s, idx, x, kp, nullptr, Nq, Ns, nq_dev, ns_dev, K, 0, 1.f / extent, wf);
        REGTR_CHECK_LAUNCH();
        return REGTR_OK;
    }
    if (Ns > 0 && !flags_ready) {
        k_row_flags<<<regtr_cdiv((long long)Ns * 32, 256), 256, 0, st>>>(x, Ns, Cin, rowflag_ws);
        REGTR_CHECK_LAUNCH();
    }
    if (Cin <= 16) {
        const size_t smem = agg_smem_bytes(K);      // 84 KB at K = 128: above K = 73 it needs the opt-in
        static size_t attr_smem = 0;
        if (smem > 48 * 1024 && smem > attr_smem) {
            if (cudaFuncSetAttribute(k_kpconv_agg_small, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
                cudaSuccess)
                return REGTR_ERR_UNSUPPORTED;
            attr_smem = smem;
        }
        k_kpconv_agg_small<<<regtr_cdiv(Nq, AGG_WARPS), AGG_WARPS * 32, smem, st>>>(q, s, idx, x, rowflag_ws, kp, Nq,
                                                                                   Ns, nq_dev, ns_dev, K, Cin, extent, wf);
        REGTR_CHECK_LAUNCH();
        return REGTR_OK;
    }
    {   // software-pipelined persistent kernel up to K = 64
        const int nh = (Cin % 64 == 0) ? 2 : 1;
        const int S = Cin / (32 * nh);
        if (K <= 64 && Cin % 32 == 0 && (S & (S - 1)) == 0) {
            const int Kp = (K + 7) & ~7;
            const size_t smem = (size_t)PIPE_WARPS * 2 * Kp * (32 * nh + 5) * sizeof(float);
            if (smem > 200 * 1024) return REGTR_ERR_UNSUPPORTED;
            static size_t attr_smem[2] = {0, 0};
            if (smem > 48 * 1024 && smem > attr_smem[nh - 1]) {
                const cudaError_t ea = nh == 1
                    ? cudaFuncSetAttribute(k_kpconv_agg_pipe<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                    : cudaFuncSetAttribute(k_kpconv_agg_pipe<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                if (ea != cudaSuccess) return REGTR_ERR_UNSUPPORTED;
                attr_smem[nh - 1] = smem;
            }
            int log2s = 0;
            while ((1 << log2s) < S) ++log2s;
            const long long items = (long long)Nq * S;
            const int fit = (int)((220 * 1024) / (smem + 1024));
            const int per_sm = std::max(1, std::min(nh == 1 ? 4 : 2, fit));
            const int grid = (int)std::min<long long>((long long)REGTR_NUM_SMS * per_sm, (items + PIPE_WARPS - 1) / PIPE_WARPS);
            if (nh == 1)
                k_kpconv_agg_pipe<1><<<grid, PIPE_WARPS * 32, smem, st>>>(q, s, idx, x, rowflag_ws, kp, Nq, Ns, nq_dev, ns_dev, K,
                                                                         Cin, log2s, 1.f / extent, wf);
            else
                k_kpconv_agg_pipe<2><<<grid, PIPE_WARPS * 32, smem, st>>>(q, s, idx, x, rowflag_ws, kp, Nq, Ns, nq_dev, ns_dev, K,
                                                                         Cin, log2s, 1.f / extent, wf);
            REGTR_CHECK_LAUNCH();
            return REGTR_OK;
        }
    }
    // longer neighbour lists: the staged kernel, one query per warp
    if (agg_mma_nh(Nq, K, Cin) == 2)
        return launch_agg_mma<2, 2>(q, s, idx, x, rowflag_ws, kp, Nq, Ns, nq_dev, ns_dev, K, Cin, extent, wf, st);
    return launch_agg_mma<1, 4>(q, s, idx, x, rowflag_ws, kp, Nq, Ns, nq_dev, ns_dev, K, Cin, extent, wf, st);
}

int regtr_kpconv_fwd(const float* q, const float* s, const int32_t* idx, const float* x, const float* W,
                     const float* kp, int Nq, int Ns, const int32_t* nq_dev, const int32_t* ns_dev, int K, int Cin,
                     int Cout, float extent, float* out, void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Cout <= 0 || Cin <= 0 || Nq < 0 || Ns < 0) return REGTR_ERR_ARG;
    if (Nq == 0) return REGTR_OK;
    if (!W || !out || !ws) return REGTR_ERR_ARG;
    if (ws_bytes < regtr_kpconv_ws_bytes(Nq, Ns, Cin)) return REGTR_ERR_WORKSPACE;
    if (Cin == 1) {                               // first block: gather + aggregation + 15 x Cout contraction, one kernel
        if (K <= 0 || K > 128 || !(extent > 0.f)) return REGTR_ERR_ARG;
        if (!q || !s || !idx || !x || !kp) return REGTR_ERR_ARG;
        const size_t smem = (size_t)AGG_WARPS * K * sizeof(float4) + (size_t)KP * Cout * sizeof(float);
        if (smem <= 48 * 1024) {
            k_kpconv_c1<true><<<c1_grid(Nq), AGG_WARPS * 32, smem, st>>>(
                q, s, idx, x, kp, W, Nq, Ns, nq_dev, ns_dev, K, Cout, 1.f / extent, out);
            REGTR_CHECK_LAUNCH();
            return REGTR_OK;
        }
    }
    float* wf = (float*)ws;
    uint8_t* flags = (uint8_t*)ws + regtr_align(sizeof(float) * (size_t)Nq * KP * (size_t)Cin);
    int rc = regtr_kpconv_aggregate(q, s, idx, x, kp, Nq, Ns, nq_dev, ns_dev, K, Cin, extent, wf, flags, 0, stream_);
    if (rc != REGTR_OK) return rc;
    const int KDs = KP * Cin;
    if (KDs <= 64 && Cout % 4 == 0 && (size_t)KDs * Cout * sizeof(float) <= 48 * 1024) {
        k_gemm_smallk<<<regtr_cdiv((long long)Nq * (Cout / 4), 256), 256, (size_t)KDs * Cout * sizeof(float), st>>>(
            wf, W, Nq, KDs, Cout, nq_dev, out);
        REGTR_CHECK_LAUNCH();
        return REGTR_OK;
    }
    // out[Nq,Cout] = wf[Nq,15*Cin] @ W[15*Cin,Cout] on the library's own 3xTF32 wgmma GEMM: split + transpose
    // W into the workspace tail, then regtr_gemm_tf32x3 (the Python front end caches the split instead)
    const int KD = KP * Cin;
    if (KD % 4) return REGTR_ERR_UNSUPPORTED;
    char* p = (char*)ws + regtr_align(sizeof(float) * (size_t)Nq * KP * (size_t)Cin) + regtr_align((size_t)(Ns > 0 ? Ns : 1));
    float* w_hi = (float*)p;
    float* w_lo = (float*)(p + regtr_align(sizeof(float) * (size_t)KD * Cout));
    void* gws = p + 2 * regtr_align(sizeof(float) * (size_t)KD * Cout);
    const size_t used = (size_t)((char*)gws - (char*)ws);
    const size_t gws_bytes = regtr_gemm_ws_bytes(Nq, Cout, KD);
    if (ws_bytes < used + gws_bytes) return REGTR_ERR_WORKSPACE;
    k_split_transpose<<<regtr_cdiv((long long)KD * Cout, 256), 256, 0, st>>>(W, KD, Cout, w_hi, w_lo);
    REGTR_CHECK_LAUNCH();
    return regtr_gemm_tf32x3(wf, KD, w_hi, w_lo, KD, out, Cout, nullptr, nullptr, 0, Nq, Cout, KD, nq_dev, 0, gws,
                             gws_bytes, stream_);
}

int regtr_max_pool(const float* x, const int32_t* idx, int Nq, int Ns, const int32_t* ns_dev, int K, int C,
                   float* out, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Nq < 0 || Ns < 0 || K <= 0 || C <= 0) return REGTR_ERR_ARG;
    if ((long long)Nq * C >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;               // 32-bit work-item index
    if (Nq == 0) return REGTR_OK;
    if (!x || !idx || !out) return REGTR_ERR_ARG;
    if (C % 4 == 0) {
        const int mp_blocks = regtr_cdiv((long long)Nq * (C / 4), 256);
        k_max_pool<<<mp_blocks < 8 * REGTR_NUM_SMS ? mp_blocks : 8 * REGTR_NUM_SMS, 256, 0, st>>>(x, idx, Nq, Ns, ns_dev, K, C, out);
    } else {
        k_max_pool_scalar<<<regtr_cdiv((long long)Nq * C, 256), 256, 0, st>>>(x, idx, Nq, Ns, ns_dev, K, C, out);
    }
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
