// Normalisation / embedding kernels around the GEMMs:
//   per-cloud InstanceNorm (+ residual, + LeakyReLU)  -- kpconv_blocks.py:474-530, 546-561
//   LayerNorm (+ position add)                         -- transformers.py:117-119, 194-232
//   3-D sine position embedding                        -- position_embedding.py:29-50
// (paths relative to /root/reference/src)
#include "common.cuh"
#include "philox.cuh"

namespace {

constexpr int IN_CH = 128;    // rows per statistics chunk
constexpr int IN_TY = 8;      // row lanes per block (block = 32 x 8 threads, 4 channels per thread)
constexpr int IN_CT = 128;    // channels per block

// chunk id -> (cloud, first row, last row) ; chunks never straddle clouds.
__device__ __forceinline__ bool chunk_of(const int32_t* __restrict__ offs, int n_clouds, int chunk, int& cloud,
                                         int& r0, int& r1, int& first, int& count) {
    int acc = 0;
    for (int c = 0; c < n_clouds; ++c) {
        const int a = offs[c], b = offs[c + 1];
        const int nc = (b - a + IN_CH - 1) / IN_CH;
        if (chunk < acc + nc) {
            cloud = c;
            r0 = a + (chunk - acc) * IN_CH;
            r1 = min(r0 + IN_CH, b);
            first = acc;                         // the cloud's chunks are [first, first + count)
            count = nc;
            return true;
        }
        acc += nc;
    }
    return false;
}

// partial[chunk][c] = (sum, sum of squares) in fp64 over the chunk's rows.  C % 4 == 0.
// With `counters` (one int per (cloud, channel tile), zero on entry and left zero): the LAST block of a
// (cloud, channel tile) to finish also reduces that group's partials to stats[cloud][c] = (mean, rstd) --
// same fixed summation order as k_in_finalize, so the result does not depend on which block that is --
// and the separate finalize launch disappears.
__global__ void __launch_bounds__(32 * IN_TY)
k_in_stats(const float* __restrict__ x, const int32_t* __restrict__ offs, int n_clouds, int C,
           double2* __restrict__ partial, int32_t* __restrict__ counters, float eps, float2* __restrict__ stats) {
    __shared__ double red[IN_TY][32][8];
    __shared__ int s_last;
    int cloud, r0, r1, first, count;
    if (!chunk_of(offs, n_clouds, blockIdx.x, cloud, r0, r1, first, count)) return;
    const int c = blockIdx.y * IN_CT + threadIdx.x * 4;
    double s[4] = {0, 0, 0, 0}, ss[4] = {0, 0, 0, 0};
    if (c < C) {
        for (int r = r0 + threadIdx.y; r < r1; r += IN_TY * 4) {
            float4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int rr = r + u * IN_TY;
                v[u] = rr < r1 ? __ldg(reinterpret_cast<const float4*>(x + (size_t)rr * C + c))
                               : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const double a0 = v[u].x, a1 = v[u].y, a2 = v[u].z, a3 = v[u].w;
                s[0] += a0; s[1] += a1; s[2] += a2; s[3] += a3;
                ss[0] += a0 * a0; ss[1] += a1 * a1; ss[2] += a2 * a2; ss[3] += a3 * a3;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[threadIdx.y][threadIdx.x][j] = s[j]; red[threadIdx.y][threadIdx.x][4 + j] = ss[j]; }
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        for (int t = 1; t < IN_TY; ++t)
#pragma unroll
            for (int j = 0; j < 4; ++j) { s[j] += red[t][threadIdx.x][j]; ss[j] += red[t][threadIdx.x][4 + j]; }
#pragma unroll
        for (int j = 0; j < 4; ++j) partial[(size_t)blockIdx.x * C + c + j] = make_double2(s[j], ss[j]);
    }
    if (!counters) return;
    __threadfence();                              // this block's partials are visible before it is counted
    __syncthreads();
    if (threadIdx.x == 0 && threadIdx.y == 0) {
        int32_t* cnt = counters + cloud * gridDim.y + blockIdx.y;
        s_last = atomicAdd(cnt, 1) == count - 1;
        if (s_last) *cnt = 0;                     // nobody else touches it any more: restored for the next call
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    double fs[4] = {0, 0, 0, 0}, fss[4] = {0, 0, 0, 0};
    if (c < C) {
        for (int t = threadIdx.y; t < count; t += IN_TY)
#pragma unroll
            for (int j = 0; j < 4; ++j) {         // L2 reads: the partials come from other SMs
                const double2 p = __ldcg(partial + (size_t)(first + t) * C + c + j);
                fs[j] += p.x; fss[j] += p.y;
            }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { red[threadIdx.y][threadIdx.x][j] = fs[j]; red[threadIdx.y][threadIdx.x][4 + j] = fss[j]; }
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        for (int t = 1; t < IN_TY; ++t)
#pragma unroll
            for (int j = 0; j < 4; ++j) { fs[j] += red[t][threadIdx.x][j]; fss[j] += red[t][threadIdx.x][4 + j]; }
        const int n = offs[cloud + 1] - offs[cloud];
        const double dn = n > 0 ? (double)n : 1.0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double mean = fs[j] / dn;
            double var = fss[j] / dn - mean * mean;          // biased variance (InstanceNorm)
            var = var > 0.0 ? var : 0.0;
            stats[(size_t)cloud * C + c + j] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
        }
    }
}

// stats[cloud][c] = (mean, 1/sqrt(var+eps)); the cloud's chunk partials are summed by 8 row lanes
// (fixed assignment) and combined in a fixed order: deterministic, no atomics.
__global__ void __launch_bounds__(32 * IN_TY)
k_in_finalize(const int32_t* __restrict__ offs, int n_clouds, int C, float eps, const double2* __restrict__ partial,
              float2* __restrict__ stats) {
    __shared__ double2 red[IN_TY][32];
    const int cloud = blockIdx.x;
    const int c = blockIdx.y * 32 + threadIdx.x;
    int first = 0;
    for (int k = 0; k < cloud; ++k) first += (offs[k + 1] - offs[k] + IN_CH - 1) / IN_CH;
    const int n = offs[cloud + 1] - offs[cloud];
    const int nc = (n + IN_CH - 1) / IN_CH;
    double s = 0.0, ss = 0.0;
    if (c < C) {
        for (int t = threadIdx.y; t < nc; t += IN_TY) {
            const double2 p = partial[(size_t)(first + t) * C + c];
            s += p.x; ss += p.y;
        }
    }
    red[threadIdx.y][threadIdx.x] = make_double2(s, ss);
    __syncthreads();
    if (threadIdx.y == 0 && c < C) {
        for (int t = 1; t < IN_TY; ++t) { s += red[t][threadIdx.x].x; ss += red[t][threadIdx.x].y; }
        const double dn = n > 0 ? (double)n : 1.0;
        const double mean = s / dn;
        double var = ss / dn - mean * mean;          // biased variance (InstanceNorm)
        var = var > 0.0 ? var : 0.0;
        stats[(size_t)cloud * C + c] = make_float2((float)mean, (float)(1.0 / sqrt(var + (double)eps)));
    }
}

// out = act((x - mean) * rstd + res), float4 per thread; rows beyond offs[n_clouds] are padding (see below).
// FLAGS: additionally emit flags[r] = (sum_c out[r,c] > 0), the "neighbour counts" predicate of the KPConv
// that consumes `out` (kpconv_blocks.py:409-412), summed in fp64 across the C/4 <= 32 lanes of the row.
template <bool FLAGS>
__global__ void k_in_apply(const float* x, const int32_t* __restrict__ offs, int n_clouds, int n_cap, int C,
                           const float2* __restrict__ stats, const float* res, float slope, float* out,
                           uint8_t* __restrict__ flags) {
    const int c4n = C >> 2;
    // grid-stride over float4 items (a few thousand long-lived CTAs instead of one item per thread: the offsets
    // chain is paid once per thread and the CTA launch cost once per ~10 items).  Only rows below the 128-row tile
    // that straddles the real count are touched: zeros in its padding part (the only padding a consumer -- a
    // tiled GEMM -- can read), nothing beyond.
    const int n_real = offs[n_clouds];
    const unsigned total = (unsigned)min(n_cap, (n_real + 127) & ~127) * (unsigned)c4n;
    const unsigned stride = gridDim.x * blockDim.x;
    for (unsigned t0 = blockIdx.x * blockDim.x; t0 < total; t0 += stride) {        // block-uniform trip count
        const unsigned t = t0 + threadIdx.x;
        const bool in_range = t < total;
        int r = 0, c = 0;
        if (in_range) { regtr_row_col(t, (unsigned)c4n, r, c); c *= 4; }
        const size_t o = (size_t)r * C + c;
        const bool live = in_range && r < n_real;
        float y[4] = {0.f, 0.f, 0.f, 0.f};
        if (live) {
            const float4 v = *reinterpret_cast<const float4*>(x + o);
            float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (res) rv = *reinterpret_cast<const float4*>(res + o);
            const int cloud = regtr_cloud_of(offs, n_clouds, r);
            const float4 st01 = *reinterpret_cast<const float4*>(stats + (size_t)cloud * C + c);
            const float4 st23 = *reinterpret_cast<const float4*>(stats + (size_t)cloud * C + c + 2);
            y[0] = (v.x - st01.x) * st01.y + rv.x; y[1] = (v.y - st01.z) * st01.w + rv.y;
            y[2] = (v.z - st23.x) * st23.y + rv.z; y[3] = (v.w - st23.z) * st23.w + rv.w;
            if (slope >= 0.f) {
#pragma unroll
                for (int j = 0; j < 4; ++j) y[j] = y[j] > 0.f ? y[j] : y[j] * slope;
            }
        }
        if (in_range) *reinterpret_cast<float4*>(out + o) = make_float4(y[0], y[1], y[2], y[3]);
        if (FLAGS) {                                           // single convergent shuffle site for the whole warp
            double acc = ((double)y[0] + (double)y[1]) + ((double)y[2] + (double)y[3]);
            for (int d = 1; d < c4n; d <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
            if (in_range && (threadIdx.x & (c4n - 1)) == 0) flags[r] = live && acc > 0.0;
        }
    }
}

// One warp per row; E = 32 * per <= 32 * PER (PER = 8: the model width 256; PER = 32: anything up to 1024).
// DROP (regtr_layernorm_pos with a dropout key): the row is first x + m * scale * z (the residual add of a dropped
// branch), written to x_out, and normalised from there.
template <int PER, bool DROP = false>
__global__ void k_layernorm_pos(const float* __restrict__ x, const float* __restrict__ gamma,
                                const float* __restrict__ beta, const float* __restrict__ pos, int n,
                                const int32_t* __restrict__ n_dev, int E, float eps, float* __restrict__ y,
                                float* __restrict__ y_pos, const float* __restrict__ z = nullptr,
                                float* __restrict__ x_out = nullptr, DropKey drop = DropKey{}) {
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (!DROP && n_dev) n = min(n, *n_dev);               // capacity-shaped launch: rows beyond the real count are skipped
    if (row >= n) return;
    const float* xr = x + (size_t)row * E;
    const int per = E / 32;
    // every operand is requested before the first reduction: one memory round trip instead of three dependent ones
    float v[PER], gm[PER], bt[PER], ps[PER];
#pragma unroll
    for (int j = 0; j < PER; ++j)
        if (j < per) {
            const int c = j * 32 + lane;
            v[j] = xr[c]; gm[j] = __ldg(gamma + c); bt[j] = __ldg(beta + c);
            ps[j] = (y_pos && pos) ? pos[(size_t)row * E + c] : 0.f;
        }
    if constexpr (DROP) {               // n_dev carries the cloud offsets here
        const int cl = regtr_cloud_of(n_dev, 2 * drop.n_pairs, row);
        const unsigned w1 = drop_word1(drop, cl, 0), rr = (unsigned)(row - n_dev[cl]);
#pragma unroll
        for (int j = 0; j < PER; ++j)
            if (j < per) {
                const int c = j * 32 + lane;
                const float zv = z[(size_t)row * E + c];
                v[j] = __fadd_rn(v[j], drop_keep(drop, w1, rr, (unsigned)c) ? __fmul_rn(zv, drop.scale) : 0.f);
                x_out[(size_t)row * E + c] = v[j];
            }
    }
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j) if (j < per) s += v[j];
    const float mean = warp_sum(s) / (float)E;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < PER; ++j) if (j < per) { const float d = v[j] - mean; ss += d * d; }
    const float rstd = 1.f / sqrtf(warp_sum(ss) / (float)E + eps);
#pragma unroll
    for (int j = 0; j < PER; ++j) {
        if (j >= per) break;
        const int c = j * 32 + lane;
        const float o = (v[j] - mean) * rstd * gm[j] + bt[j];
        if (y) y[(size_t)row * E + c] = o;
        if (y_pos) y_pos[(size_t)row * E + c] = o + ps[j];
    }
}

// out[i, a*n_freq + f] = f even ? sin(v) : cos(v),  v = (xyz[i,a]*scale) / dim_t[f]; zero pad.
__global__ void k_pos_embed_sine(const float* __restrict__ xyz, int n, const float* __restrict__ dim_t, int n_freq,
                                 int d_model, float scale, float* __restrict__ out) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * d_model) return;
    int i, c;
    regtr_row_col((unsigned)t, (unsigned)d_model, i, c);
    float o = 0.f;
    if (c < 3 * n_freq) {
        const int a = c / n_freq, f = c % n_freq;
        const float v = __fdiv_rn(__fmul_rn(xyz[3 * i + a], scale), dim_t[f]);
        o = (f & 1) ? cosf(v) : sinf(v);
    }
    out[t] = o;
}

static inline int in_apply_grid(long long items) {
    const long long b = (items + 255) / 256;
    return (int)(b < 8 * REGTR_NUM_SMS ? (b > 0 ? b : 1) : 8 * REGTR_NUM_SMS);
}

}  // namespace

extern "C" {

static inline int in_chunks(int n_cap, int n_clouds) { return regtr_cdiv(n_cap > 0 ? n_cap : 1, IN_CH) + n_clouds; }

size_t regtr_instnorm_ws_bytes(int n_cap, int n_clouds, int C) {
    const size_t c = (size_t)(C > 0 ? C : 1), nc = (size_t)(n_clouds > 0 ? n_clouds : 1);
    return regtr_align((size_t)in_chunks(n_cap, (int)nc) * c * sizeof(double2)) + regtr_align(nc * c * sizeof(float2));
}

size_t regtr_instnorm_counter_bytes(int n_clouds, int C) {
    return sizeof(int32_t) * (size_t)(n_clouds > 0 ? n_clouds : 1) * (size_t)regtr_cdiv(C > 0 ? C : 1, IN_CT);
}

int regtr_instnorm_act(const float* x, const int32_t* offs, int n_clouds, int n_cap, int C, float eps,
                       const float* res, float slope, float* out, uint8_t* rowflag_out, void* ws, size_t ws_bytes,
                       int32_t* counters, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || n_clouds <= 0 || n_cap < 0 || C <= 0) return REGTR_ERR_ARG;
    if (C % 4 != 0 || (long long)n_cap * (C / 4) >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;   // 32-bit work-item index
    if (n_cap == 0) return REGTR_OK;
    if (!x || !out || !ws) return REGTR_ERR_ARG;
    if (ws_bytes < regtr_instnorm_ws_bytes(n_cap, n_clouds, C)) return REGTR_ERR_WORKSPACE;
    const int chunks = in_chunks(n_cap, n_clouds);
    double2* partial = (double2*)ws;
    float2* stats = (float2*)((char*)ws + regtr_align((size_t)chunks * C * sizeof(double2)));
    dim3 block(32, IN_TY);
    k_in_stats<<<dim3(chunks, regtr_cdiv(C, IN_CT)), block, 0, st>>>(x, offs, n_clouds, C, partial, counters, eps, stats);
    REGTR_CHECK_LAUNCH();
    if (!counters) {                              // no persistent counters: separate finalize launch
        k_in_finalize<<<dim3(n_clouds, regtr_cdiv(C, 32)), block, 0, st>>>(offs, n_clouds, C, eps, partial, stats);
        REGTR_CHECK_LAUNCH();
    }
    if (rowflag_out) {
        const int c4n = C / 4;
        if (c4n > 32 || (c4n & (c4n - 1))) return REGTR_ERR_UNSUPPORTED;   // the row must sit inside one warp
        k_in_apply<true><<<in_apply_grid((long long)n_cap * c4n), 256, 0, st>>>(x, offs, n_clouds, n_cap, C, stats,
                                                                                  res, slope, out, rowflag_out);
    } else {
        k_in_apply<false><<<in_apply_grid((long long)n_cap * (C / 4)), 256, 0, st>>>(x, offs, n_clouds, n_cap, C,
                                                                                      stats, res, slope, out, nullptr);
    }
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

// Apply pass alone, with statistics produced elsewhere (the GEMM epilogue, regtr_gemm_tf32x3_instats).
int regtr_instnorm_apply(const float* x, const int32_t* offs, int n_clouds, int n_cap, int C, const float* stats,
                         const float* res, float slope, float* out, uint8_t* rowflag_out, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || n_clouds <= 0 || n_cap < 0 || C <= 0) return REGTR_ERR_ARG;
    if (C % 4 != 0 || (long long)n_cap * (C / 4) >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;   // 32-bit work-item index
    if (n_cap == 0) return REGTR_OK;
    if (!x || !out || !stats) return REGTR_ERR_ARG;
    const float2* stp = reinterpret_cast<const float2*>(stats);
    if (rowflag_out) {
        const int c4n = C / 4;
        if (c4n > 32 || (c4n & (c4n - 1))) return REGTR_ERR_UNSUPPORTED;   // the row must sit inside one warp
        k_in_apply<true><<<in_apply_grid((long long)n_cap * c4n), 256, 0, st>>>(x, offs, n_clouds, n_cap, C, stp, res, slope,
                                                                                  out, rowflag_out);
    } else {
        k_in_apply<false><<<in_apply_grid((long long)n_cap * (C / 4)), 256, 0, st>>>(x, offs, n_clouds, n_cap, C, stp, res,
                                                                                      slope, out, nullptr);
    }
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_layernorm_pos(const float* x, const float* z, const float* gamma, const float* beta, const float* pos, int n,
                        const int32_t* n_dev, const int32_t* offs, int E, float eps, float* y, float* y_pos,
                        float* x_out, const regtr_dropout_args* drop, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    // z, offs, x_out and drop come together; the dropout launch uses the kernel's n_dev slot for offs
    if (!z != !drop || !offs != !drop || !x_out != !drop || (drop && n_dev)) return REGTR_ERR_ARG;
    DropKey dk;
    if (drop && (drop_key_of(drop, dk) != REGTR_OK || x_out == x || x_out == z)) return REGTR_ERR_ARG;
    if (n < 0 || E <= 0 || E % 32 != 0 || E > 1024) return REGTR_ERR_ARG;
    if (n == 0) return REGTR_OK;
    if (!x || !gamma || !beta || (!y && !y_pos)) return REGTR_ERR_ARG;
    if (drop && E <= 256)
        k_layernorm_pos<8, true><<<regtr_cdiv((long long)n * 32, 256), 256, 0, st>>>(x, gamma, beta, pos, n, offs, E, eps,
                                                                                     y, y_pos, z, x_out, dk);
    else if (drop)
        k_layernorm_pos<32, true><<<regtr_cdiv((long long)n * 32, 256), 256, 0, st>>>(x, gamma, beta, pos, n, offs, E,
                                                                                      eps, y, y_pos, z, x_out, dk);
    else if (E <= 256)
        k_layernorm_pos<8><<<regtr_cdiv((long long)n * 32, 256), 256, 0, st>>>(x, gamma, beta, pos, n, n_dev, E, eps, y, y_pos);
    else
        k_layernorm_pos<32><<<regtr_cdiv((long long)n * 32, 256), 256, 0, st>>>(x, gamma, beta, pos, n, n_dev, E, eps, y, y_pos);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_pos_embed_sine(const float* xyz, int n, const float* dim_t, int n_freq, int d_model, float scale,
                         float* out, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n < 0 || n_freq <= 0 || d_model < 3 * n_freq) return REGTR_ERR_ARG;
    if ((long long)n * d_model >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;
    if (n == 0) return REGTR_OK;
    if (!xyz || !dim_t || !out) return REGTR_ERR_ARG;
    k_pos_embed_sine<<<regtr_cdiv((long long)n * d_model, 256), 256, 0, st>>>(xyz, n, dim_t, n_freq, d_model, scale, out);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
