// Backward kernels of the KPConv encoder (training with train_encoder=True):
//   neighbour-list transpose (incoming-edge CSR per support row)
//   KPConv input gradient                     -- kpconv_blocks.py:388-412 (gather, influence-weighted sum, count)
//   max-pool backward                         -- kpconv_blocks.py:127-143
//   per-cloud InstanceNorm (+ residual) (+ LeakyReLU) backward -- kpconv_blocks.py:497-519, 546-561, 646, 741
// (paths relative to /root/reference/src).  The weight gradients reuse regtr_kpconv_aggregate and regtr_linear_wgrad.
// Every floating-point reduction runs in a fixed order with no atomics (integer atomics only count edges, and the
// order inside each CSR row is restored by a sort): two backward passes over the same inputs are bit-identical.
#include "common.cuh"

namespace {

constexpr int KP = 15;              // kernel points
constexpr int KPP = 16;             // padded
constexpr int EW = 4;               // warps per block of the per-query edge kernel
constexpr int NB_CH = 128;          // rows per InstanceNorm-backward statistics chunk (chunks never straddle clouds)
constexpr int NB_TY = 8;            // row lanes per statistics block (32 x 8 threads, 4 channels per thread)

// ---- neighbour-list transpose ---------------------------------------------------------------------------------
__global__ void k_csr_zero(int32_t* __restrict__ cnt, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) cnt[i] = 0;
}

__global__ void k_csr_count(const int32_t* __restrict__ idx, long long n_edges, int Ns, int32_t* __restrict__ cnt) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int s = idx[e];
    if (s >= 0 && s < Ns) atomicAdd(cnt + s, 1);
}

// row_start = exclusive prefix of cnt (one block, fixed order); cnt is reset to 0 for use as the fill cursor.
constexpr int SCAN_T = 1024;
__global__ void __launch_bounds__(SCAN_T) k_csr_scan(int32_t* __restrict__ cnt, int Ns, int32_t* __restrict__ row_start) {
    __shared__ int32_t wsum[SCAN_T / 32];
    const int per = (Ns + SCAN_T - 1) / SCAN_T;
    const int a = threadIdx.x * per, b = min(a + per, Ns);
    int local = 0;
    for (int i = a; i < b; ++i) local += cnt[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = wsum[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += v;
        }
        wsum[lane] = wi - w;                      // exclusive prefix of the warp totals
    }
    __syncthreads();
    int run = wsum[warp] + incl - local;
    for (int i = a; i < b; ++i) {
        row_start[i] = run;
        run += cnt[i];
        cnt[i] = 0;
    }
    if (threadIdx.x == SCAN_T - 1) row_start[Ns] = run;      // the last thread's range ends at Ns (or is empty)
}

__global__ void k_csr_fill(const int32_t* __restrict__ idx, long long n_edges, int Ns, const int32_t* __restrict__ row_start,
                           int32_t* __restrict__ cursor, int32_t* __restrict__ edges) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const int s = idx[e];
    if (s >= 0 && s < Ns) edges[row_start[s] + atomicAdd(cursor + s, 1)] = (int32_t)e;
}

// the slots were taken in scheduling order: sort every (short) row by edge id
__global__ void k_csr_sort(const int32_t* __restrict__ row_start, int Ns, int32_t* __restrict__ edges) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= Ns) return;
    const int a = row_start[s], b = row_start[s + 1];
    for (int i = a + 1; i < b; ++i) {
        const int v = edges[i];
        int j = i - 1;
        while (j >= a && edges[j] > v) { edges[j + 1] = edges[j]; --j; }
        edges[j + 1] = v;
    }
}

// ---- KPConv input gradient --------------------------------------------------------------------------------------
// Same linear influence as the forward aggregation kernels (kpconv.cu: influence()), bit for bit.
__device__ __forceinline__ float influence(const float4 r, float kx, float ky, float kz, float inv_extent) {
    const float dx = r.x - kx, dy = r.y - ky, dz = r.z - kz;
    const float d2 = dx * dx + dy * dy + dz * dz;
    float d;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(d) : "f"(d2));
    return fmaxf(0.f, fmaf(-d, inv_extent, 1.f));
}

// Phase (a): one warp per query.  For every valid neighbour slot k of query q the edge row
//   E[q K + k, c] = (1 / cnt_q) sum_p h(q, k, p) dwf[q, p, c]          (p ascending)
// cnt_q counts the valid neighbours whose feature row sums to > 0: from `flags` (the forward's flags), or -- flags
// NULL -- recomputed from x exactly as k_row_flags does (fp64, lane-strided, butterfly).  Shadow slots write nothing.
// NV: channels per lane and pass (the warp covers 32 NV channels per pass over the neighbours).
template <int NV>
__global__ void __launch_bounds__(EW * 32)
k_kpconv_bwd_edges(const float* __restrict__ q, const float* __restrict__ s, const int32_t* __restrict__ idx,
                   const float* __restrict__ x, const uint8_t* __restrict__ flags, const float* __restrict__ kp,
                   int Nq, int Ns, int K, int Cin, float inv_extent, const float* __restrict__ dwf,
                   float* __restrict__ E) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qi = blockIdx.x * EW + warp;
    if (qi >= Nq) return;
    // per warp: w[K][16] | rel[K] (float4) | slot[K] | id[K], 16-byte aligned
    float* w_s = reinterpret_cast<float*>(smem_raw) + (size_t)warp * ((K * (KPP + 4 + 2) + 3) & ~3);
    float4* rel_s = reinterpret_cast<float4*>(w_s + K * KPP);
    int* slot_s = reinterpret_cast<int*>(w_s + K * (KPP + 4));
    int* id_s = slot_s + K;
    const float qx = q[3 * qi], qy = q[3 * qi + 1], qz = q[3 * qi + 2];
    int base = 0, counted = 0;
    for (int k0 = 0; k0 < K; k0 += 32) {
        const int kk = k0 + lane;
        const int id = kk < K ? idx[(size_t)qi * K + kk] : Ns;
        const bool valid = id >= 0 && id < Ns;
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        if (valid) {
            const int pos = base + __popc(m & ((1u << lane) - 1u));
            rel_s[pos] = make_float4(s[3 * id + 0] - qx, s[3 * id + 1] - qy, s[3 * id + 2] - qz, 0.f);
            slot_s[pos] = kk;
            id_s[pos] = id;
            if (flags) counted += flags[id];
        }
        base += __popc(m);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) counted += __shfl_xor_sync(0xffffffffu, counted, o);
    __syncwarp();
    if (!flags) {
        counted = 0;
        for (int n = 0; n < base; ++n) {
            double acc = 0.0;
            for (int c = lane; c < Cin; c += 32) acc += (double)x[(size_t)id_s[n] * Cin + c];
            counted += warp_sum(acc) > 0.0;
        }
    }
    const int p = lane & 15;
    const bool real = p < KP;
    const float kx = real ? __ldg(kp + 3 * p) : 0.f, ky = real ? __ldg(kp + 3 * p + 1) : 0.f,
                kz = real ? __ldg(kp + 3 * p + 2) : 0.f;
    for (int n = lane >> 4; n < base; n += 2) w_s[n * KPP + p] = real ? influence(rel_s[n], kx, ky, kz, inv_extent) : 0.f;
    __syncwarp();
    float inv;                                    // the forward's 1 / max(count, 1)
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"((float)max(counted, 1)));
    const float* drow = dwf + (size_t)qi * KP * Cin;
    for (int c0 = 0; c0 < Cin; c0 += 32 * NV) {
        float d[KP][NV];
#pragma unroll
        for (int pp = 0; pp < KP; ++pp)
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                const int c = c0 + 32 * j + lane;
                d[pp][j] = c < Cin ? __ldg(drow + pp * Cin + c) : 0.f;
            }
        for (int n = 0; n < base; ++n) {
            const float4* wr = reinterpret_cast<const float4*>(w_s + n * KPP);
            const float4 wa = wr[0], wb = wr[1], wc = wr[2], wd = wr[3];
            const float w[KP] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w, wc.x, wc.y, wc.z, wc.w, wd.x, wd.y, wd.z};
            float* erow = E + ((size_t)qi * K + slot_s[n]) * Cin;
#pragma unroll
            for (int j = 0; j < NV; ++j) {
                float acc = 0.f;
#pragma unroll
                for (int pp = 0; pp < KP; ++pp) acc = fmaf(w[pp], d[pp][j], acc);
                const int c = c0 + 32 * j + lane;
                if (c < Cin) erow[c] = acc * inv;
            }
        }
    }
}

// Phase (b): one warp per support row, its incoming edge rows summed in CSR (ascending edge id) order.
__global__ void __launch_bounds__(256)
k_csr_rowsum(const int32_t* __restrict__ row_start, const int32_t* __restrict__ edges, const float* __restrict__ E,
             int Ns, int C, float* __restrict__ dx) {
    const int sr = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (sr >= Ns) return;
    const int a = row_start[sr], b = row_start[sr + 1];
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
        for (int i = a; i < b; ++i) acc += __ldg(E + (size_t)__ldg(edges + i) * C + c);
        dx[(size_t)sr * C + c] = acc;
    }
}

// ---- max-pool backward ------------------------------------------------------------------------------------------
// arg[q, c] = first k (neighbour order) whose value is maximal; the shadow slots take part with value 0 (their
// gradient is dropped: shadow slots have no CSR entry) -- torch.max(dim)'s tie rule on the zero-padded gather.
__global__ void k_maxpool_arg(const float* __restrict__ x, const int32_t* __restrict__ idx, int Nq, int Ns, int K, int C,
                              uint8_t* __restrict__ arg) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)Nq * C) return;
    int qi, c;
    regtr_row_col((unsigned)t, (unsigned)C, qi, c);
    float best = -INFINITY;
    int bk = 0;
    for (int k = 0; k < K; ++k) {
        const int id = idx[(size_t)qi * K + k];
        const float v = (id >= 0 && id < Ns) ? __ldg(x + (size_t)id * C + c) : 0.f;
        if (v > best) { best = v; bk = k; }
    }
    arg[t] = (uint8_t)bk;
}

// dx[s, c] = sum over incoming edges e = (q, k) of s, in CSR order, of dout[q, c] where arg[q, c] == k
__global__ void __launch_bounds__(256)
k_maxpool_gather(const int32_t* __restrict__ row_start, const int32_t* __restrict__ edges, const uint8_t* __restrict__ arg,
                 const float* __restrict__ dout, int Ns, int K, int C, float* __restrict__ dx) {
    const int sr = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (sr >= Ns) return;
    const int a = row_start[sr], b = row_start[sr + 1];
    for (int c = lane; c < C; c += 32) {
        float acc = 0.f;
        for (int i = a; i < b; ++i) {
            const int e = __ldg(edges + i), qi = e / K, k = e - qi * K;
            if (__ldg(arg + (size_t)qi * C + c) == k) acc += __ldg(dout + (size_t)qi * C + c);
        }
        dx[(size_t)sr * C + c] = acc;
    }
}

// ---- per-cloud InstanceNorm backward ------------------------------------------------------------------------------
// y = act((x - mean) rstd + res), act = LeakyReLU(slope) (slope < 0: none).  g' = g * (out > 0 ? 1 : slope) as torch
// masks at 0;  dres = g';  dx = rstd (g' - mean_cloud(g') - xh mean_cloud(g' xh)),  xh = (x - mean) rstd.
// mean / rstd are recomputed from x: fp64 column sums over fixed 128-row chunks (a chunk never straddles two clouds),
// chunk partials added in ascending order per (cloud, channel).  sum(g' xh) = rstd (sum(g' x) - mean sum(g')).
__device__ __forceinline__ bool nb_chunk_of(const int32_t* __restrict__ offs, int n_clouds, int chunk, int& cloud,
                                            int& r0, int& r1) {
    int acc = 0;
    for (int c = 0; c < n_clouds; ++c) {
        const int a = offs[c], b = offs[c + 1];
        const int nc = (b - a + NB_CH - 1) / NB_CH;
        if (chunk < acc + nc) {
            cloud = c;
            r0 = a + (chunk - acc) * NB_CH;
            r1 = min(r0 + NB_CH, b);
            return true;
        }
        acc += nc;
    }
    return false;
}

__device__ __forceinline__ float lrelu_mask(float g, float out, float slope) {
    return slope >= 0.f ? (out > 0.f ? g : g * slope) : g;
}

// part[chunk][c] = (sum x, sum x^2, sum g', sum g' x) in fp64
__global__ void __launch_bounds__(32 * NB_TY)
k_inb_partial(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ out,
              const int32_t* __restrict__ offs, int n_clouds, int C, float slope, double4* __restrict__ part) {
    __shared__ double4 red[NB_TY][32][4];
    int cloud, r0, r1;
    if (!nb_chunk_of(offs, n_clouds, blockIdx.x, cloud, r0, r1)) return;
    const int c = blockIdx.y * 128 + threadIdx.x * 4;
    double4 a[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) a[j] = make_double4(0.0, 0.0, 0.0, 0.0);
    if (c < C) {
        for (int r = r0 + threadIdx.y; r < r1; r += NB_TY) {
            const size_t o = (size_t)r * C + c;
            const float4 xv = __ldg(reinterpret_cast<const float4*>(x + o));
            const float4 gv = __ldg(reinterpret_cast<const float4*>(g + o));
            float4 ov = make_float4(1.f, 1.f, 1.f, 1.f);
            if (slope >= 0.f) ov = __ldg(reinterpret_cast<const float4*>(out + o));
            const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
            const float gs[4] = {lrelu_mask(gv.x, ov.x, slope), lrelu_mask(gv.y, ov.y, slope),
                                 lrelu_mask(gv.z, ov.z, slope), lrelu_mask(gv.w, ov.w, slope)};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const double xd = xs[j], gd = gs[j];
                a[j].x += xd; a[j].y += xd * xd; a[j].z += gd; a[j].w += gd * xd;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) red[threadIdx.y][threadIdx.x][j] = a[j];
    __syncthreads();
    if (threadIdx.y != 0 || c >= C) return;
    for (int t = 1; t < NB_TY; ++t)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double4 v = red[t][threadIdx.x][j];
            a[j].x += v.x; a[j].y += v.y; a[j].z += v.z; a[j].w += v.w;
        }
#pragma unroll
    for (int j = 0; j < 4; ++j) part[(size_t)blockIdx.x * C + c + j] = a[j];
}

// coef[cloud][c] = (mean, rstd, mean(g'), mean(g' xh)) as fp32, from the cloud's chunk partials in ascending order
__global__ void k_inb_finalize(const int32_t* __restrict__ offs, int n_clouds, int C, float eps,
                               const double4* __restrict__ part, float4* __restrict__ coef) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x, cloud = blockIdx.y;
    if (c >= C) return;
    int first = 0;
    for (int k = 0; k < cloud; ++k) first += (offs[k + 1] - offs[k] + NB_CH - 1) / NB_CH;
    const int n = offs[cloud + 1] - offs[cloud];
    const int nc = (n + NB_CH - 1) / NB_CH;
    double sx = 0.0, sxx = 0.0, sg = 0.0, sgx = 0.0;
    for (int t = 0; t < nc; ++t) {
        const double4 v = part[(size_t)(first + t) * C + c];
        sx += v.x; sxx += v.y; sg += v.z; sgx += v.w;
    }
    const double dn = n > 0 ? (double)n : 1.0;
    const double mean = sx / dn;
    double var = sxx / dn - mean * mean;          // biased variance (InstanceNorm)
    var = var > 0.0 ? var : 0.0;
    const double rstd = 1.0 / sqrt(var + (double)eps);
    const double mg = sg / dn;
    const double mgx = rstd * (sgx / dn - mean * mg);
    coef[(size_t)cloud * C + c] = make_float4((float)mean, (float)rstd, (float)mg, (float)mgx);
}

// rows beyond offs[n_clouds] get zero gradients
__global__ void k_inb_apply(const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ out,
                            const int32_t* __restrict__ offs, int n_clouds, int n, int C, float slope,
                            const float4* __restrict__ coef, float* __restrict__ dx, float* __restrict__ dres) {
    const int c4n = C >> 2;
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long long)n * c4n) return;
    int r, c;
    regtr_row_col((unsigned)t, (unsigned)c4n, r, c);
    c *= 4;
    const size_t o = (size_t)r * C + c;
    float dxv[4] = {0.f, 0.f, 0.f, 0.f}, gp[4] = {0.f, 0.f, 0.f, 0.f};
    if (r < offs[n_clouds]) {
        const int cloud = regtr_cloud_of(offs, n_clouds, r);
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + o));
        const float4 gv = __ldg(reinterpret_cast<const float4*>(g + o));
        float4 ov = make_float4(1.f, 1.f, 1.f, 1.f);
        if (slope >= 0.f) ov = __ldg(reinterpret_cast<const float4*>(out + o));
        const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs[4] = {gv.x, gv.y, gv.z, gv.w}, os[4] = {ov.x, ov.y, ov.z, ov.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float4 k = coef[(size_t)cloud * C + c + j];
            gp[j] = lrelu_mask(gs[j], os[j], slope);
            const float xh = (xs[j] - k.x) * k.y;
            dxv[j] = k.y * ((gp[j] - k.z) - xh * k.w);
        }
    }
    *reinterpret_cast<float4*>(dx + o) = make_float4(dxv[0], dxv[1], dxv[2], dxv[3]);
    if (dres) *reinterpret_cast<float4*>(dres + o) = make_float4(gp[0], gp[1], gp[2], gp[3]);
}

int nb_chunks(int n, int n_clouds) { return regtr_cdiv(n > 0 ? n : 1, NB_CH) + n_clouds; }

size_t edge_smem_bytes(int K) { return (size_t)EW * ((K * (KPP + 4 + 2) + 3) & ~3) * sizeof(float); }

}  // namespace

extern "C" {

size_t regtr_neighbor_csr_ws_bytes(int Ns) {
    return regtr_align(sizeof(int32_t) * (size_t)(Ns > 0 ? Ns : 1));
}

int regtr_neighbor_csr(const int32_t* idx, int Nq, int K, int Ns, int32_t* row_start, int32_t* edges, void* ws,
                       size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Nq < 0 || K <= 0 || Ns < 0 || (long long)Nq * K >= (1ll << 31)) return REGTR_ERR_ARG;
    if (!row_start || (Nq > 0 && (!idx || !edges))) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_neighbor_csr_ws_bytes(Ns)) return REGTR_ERR_WORKSPACE;
    int32_t* cnt = (int32_t*)ws;
    const long long ne = (long long)Nq * K;
    if (Ns > 0) {
        k_csr_zero<<<regtr_cdiv(Ns, 256), 256, 0, st>>>(cnt, Ns);
        REGTR_CHECK_LAUNCH();
    }
    if (ne > 0 && Ns > 0) {
        k_csr_count<<<regtr_cdiv(ne, 256), 256, 0, st>>>(idx, ne, Ns, cnt);
        REGTR_CHECK_LAUNCH();
    }
    k_csr_scan<<<1, SCAN_T, 0, st>>>(cnt, Ns, row_start);
    REGTR_CHECK_LAUNCH();
    if (ne > 0 && Ns > 0) {
        k_csr_fill<<<regtr_cdiv(ne, 256), 256, 0, st>>>(idx, ne, Ns, row_start, cnt, edges);
        REGTR_CHECK_LAUNCH();
        k_csr_sort<<<regtr_cdiv(Ns, 128), 128, 0, st>>>(row_start, Ns, edges);
        REGTR_CHECK_LAUNCH();
    }
    return REGTR_OK;
}

size_t regtr_kpconv_bwd_input_ws_bytes(int Nq, int K, int Cin) {
    return regtr_align(sizeof(float) * (size_t)(Nq > 0 ? Nq : 1) * (size_t)(K > 0 ? K : 1) * (size_t)(Cin > 0 ? Cin : 1));
}

int regtr_kpconv_bwd_input(const float* q, const float* s, const int32_t* idx, const float* x, const uint8_t* flags,
                           const float* kp, int Nq, int Ns, int K, int Cin, float extent, const float* dwf,
                           const int32_t* row_start, const int32_t* edges, float* dx, void* ws, size_t ws_bytes,
                           void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Nq < 0 || Ns < 0 || K <= 0 || K > 128 || Cin <= 0 || Cin > 256 || !(extent > 0.f)) return REGTR_ERR_ARG;
    if (Ns == 0) return REGTR_OK;
    if (!x || !dx || !row_start || (Nq > 0 && (!q || !s || !idx || !kp || !dwf || !edges))) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_kpconv_bwd_input_ws_bytes(Nq, K, Cin)) return REGTR_ERR_WORKSPACE;
    float* E = (float*)ws;
    if (Nq > 0) {
        const size_t smem = edge_smem_bytes(K);
        const dim3 grid(regtr_cdiv(Nq, EW));
        const float inv_extent = 1.f / extent;
        if (Cin <= 32)
            k_kpconv_bwd_edges<1><<<grid, EW * 32, smem, st>>>(q, s, idx, x, flags, kp, Nq, Ns, K, Cin, inv_extent, dwf, E);
        else if (Cin <= 64)
            k_kpconv_bwd_edges<2><<<grid, EW * 32, smem, st>>>(q, s, idx, x, flags, kp, Nq, Ns, K, Cin, inv_extent, dwf, E);
        else
            k_kpconv_bwd_edges<4><<<grid, EW * 32, smem, st>>>(q, s, idx, x, flags, kp, Nq, Ns, K, Cin, inv_extent, dwf, E);
        REGTR_CHECK_LAUNCH();
    }
    k_csr_rowsum<<<regtr_cdiv((long long)Ns * 32, 256), 256, 0, st>>>(row_start, edges, E, Ns, Cin, dx);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_max_pool_bwd_ws_bytes(int Nq, int C) {
    return regtr_align((size_t)(Nq > 0 ? Nq : 1) * (size_t)(C > 0 ? C : 1));
}

int regtr_max_pool_bwd(const float* x, const int32_t* idx, int Nq, int Ns, int K, int C, const float* dout,
                       const int32_t* row_start, const int32_t* edges, float* dx, void* ws, size_t ws_bytes,
                       void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (Nq < 0 || Ns < 0 || K <= 0 || K > 255 || C <= 0) return REGTR_ERR_ARG;
    if ((long long)Nq * C >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;               // 32-bit work-item index
    if (Ns == 0) return REGTR_OK;
    if (!x || !dx || !row_start || (Nq > 0 && (!idx || !dout || !edges))) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_max_pool_bwd_ws_bytes(Nq, C)) return REGTR_ERR_WORKSPACE;
    uint8_t* arg = (uint8_t*)ws;
    if (Nq > 0) {
        k_maxpool_arg<<<regtr_cdiv((long long)Nq * C, 256), 256, 0, st>>>(x, idx, Nq, Ns, K, C, arg);
        REGTR_CHECK_LAUNCH();
    }
    k_maxpool_gather<<<regtr_cdiv((long long)Ns * 32, 256), 256, 0, st>>>(row_start, edges, arg, dout, Ns, K, C, dx);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

size_t regtr_instnorm_bwd_ws_bytes(int n, int n_clouds, int C) {
    const size_t c = (size_t)(C > 0 ? C : 1), nc = (size_t)(n_clouds > 0 ? n_clouds : 1);
    return regtr_align((size_t)nb_chunks(n, (int)nc) * c * sizeof(double4)) + regtr_align(nc * c * sizeof(float4));
}

int regtr_instnorm_bwd(const float* g, const float* x, const float* out, const int32_t* offs, int n_clouds, int n,
                       int C, float eps, float slope, float* dx, float* dres, void* ws, size_t ws_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || n_clouds <= 0 || n < 0 || C <= 0) return REGTR_ERR_ARG;
    if (C % 4 != 0 || (long long)n * (C / 4) >= (1ll << 31)) return REGTR_ERR_UNSUPPORTED;
    if (n == 0) return REGTR_OK;
    if (!g || !x || !dx || (slope >= 0.f && !out)) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_instnorm_bwd_ws_bytes(n, n_clouds, C)) return REGTR_ERR_WORKSPACE;
    const int chunks = nb_chunks(n, n_clouds);
    double4* part = (double4*)ws;
    float4* coef = (float4*)((char*)ws + regtr_align((size_t)chunks * C * sizeof(double4)));
    k_inb_partial<<<dim3(chunks, regtr_cdiv(C, 128)), dim3(32, NB_TY), 0, st>>>(g, x, out, offs, n_clouds, C, slope, part);
    REGTR_CHECK_LAUNCH();
    k_inb_finalize<<<dim3(regtr_cdiv(C, 128), n_clouds), 128, 0, st>>>(offs, n_clouds, C, eps, part, coef);
    REGTR_CHECK_LAUNCH();
    k_inb_apply<<<regtr_cdiv((long long)n * (C / 4), 256), 256, 0, st>>>(g, x, out, offs, n_clouds, n, C, slope, coef,
                                                                       dx, dres);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
