// Optimizer step on multi-tensor launches: gradient-norm clipping (torch.nn.utils.clip_grad_norm_, 2-norm) and the
// Adam / AdamW update (torch.optim.Adam / AdamW, single-tensor arithmetic), plus the in-place refresh of the TF32
// (hi, lo) weight splits the GEMMs read, so that an updated weight keeps its split buffers.
//
// Every kernel walks a device table of tensor descriptors: the launch count does not depend on the number of tensors.
// Work is cut into fixed chunks (REGTR_OPTIM_CHUNK elements) or 32 x 32 tiles; a CTA finds its tensor by binary search
// over the exclusive chunk / tile prefixes stored in the table.  No floating-point atomics: the squared norm is summed
// in fp64 per chunk in a fixed order, and the chunk partials are added in a fixed order by one CTA.
#include <math.h>

#include "common.cuh"

static_assert(sizeof(regtr_grad_ref) == 24, "regtr_grad_ref layout");
static_assert(sizeof(regtr_adam_tensor) == 88, "regtr_adam_tensor layout");
static_assert(sizeof(regtr_split_view) == 56, "regtr_split_view layout");
static_assert(sizeof(regtr_bucket_ref) == 32, "regtr_bucket_ref layout");

namespace {

constexpr int CHUNK = REGTR_OPTIM_CHUNK;
constexpr int NORM_THREADS = 256;
constexpr int FIN_THREADS = 1024;
constexpr int UPD_THREADS = 256;
static_assert(CHUNK % (NORM_THREADS * 4) == 0, "chunk must split evenly over the threads");

// index of the table entry that owns work item t: largest i with first(i) <= t (entries sorted by their prefix)
template <class T>
__device__ __forceinline__ int owner_of(const T* __restrict__ tab, int n, long long t) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (tab[mid].first <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// ---- gradient bucket -------------------------------------------------------------------------------------------
// One CTA per chunk of one tensor: pack copies the tensor into bucket[off, off + n) (zeros for a null tensor), unpack
// copies it back (nothing for a null tensor).  Plain copies: the values are bit-identical after a round trip.
__global__ void __launch_bounds__(UPD_THREADS)
k_bucket_chunks(const regtr_bucket_ref* __restrict__ tab, int n_tensors, float* __restrict__ bucket, bool unpack) {
    const long long c = blockIdx.x;
    const int i = owner_of(tab, n_tensors, c);
    float* __restrict__ t = tab[i].t;
    const long long base = (c - tab[i].first) * CHUNK;
    const int len = (int)min((long long)CHUNK, tab[i].n - base);
    float* __restrict__ b = bucket + tab[i].off + base;
    if (unpack) {
        if (t)
            for (int k = threadIdx.x; k < len; k += UPD_THREADS) t[base + k] = b[k];
    } else {
        for (int k = threadIdx.x; k < len; k += UPD_THREADS) b[k] = t ? t[base + k] : 0.f;
    }
}

// ---- gradient norm ----------------------------------------------------------------------------------------------
// One CTA per chunk: thread t adds x^2 (exact in fp64) of elements t, t + 256, ... of the chunk in order, then a fixed
// shuffle tree and the 8 warp sums in order.  The order does not depend on the data's alignment.
__global__ void __launch_bounds__(NORM_THREADS)
k_sumsq_chunks(const regtr_grad_ref* __restrict__ tab, int n_tensors, double* __restrict__ partial) {
    __shared__ double s_warp[NORM_THREADS / 32];
    const long long c = blockIdx.x;
    const int i = owner_of(tab, n_tensors, c);
    const float* __restrict__ g = tab[i].g;
    const long long n = tab[i].n;
    const long long base = (c - tab[i].first) * CHUNK;
    const int len = (int)min((long long)CHUNK, n - base);
    double s = 0.0;
#pragma unroll 8
    for (int k = threadIdx.x; k < len; k += NORM_THREADS) {
        const double x = (double)g[base + k];
        s += x * x;
    }
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < NORM_THREADS / 32; ++w) t += s_warp[w];
        partial[c] = t;
    }
}

// out[0] = fp32 total norm; out[1] = clip coefficient min(1, max_norm / (total + 1e-6)) with torch's fp32 roundings
// (reciprocal, then the product; NaN propagates as in torch.clamp).
__global__ void __launch_bounds__(FIN_THREADS)
k_norm_finalize(const double* __restrict__ partial, int n_chunks, float max_norm, float* __restrict__ out) {
    __shared__ double s_warp[FIN_THREADS / 32];
    double s = 0.0;
    for (int k = threadIdx.x; k < n_chunks; k += FIN_THREADS) s += partial[k];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < FIN_THREADS / 32; ++w) t += s_warp[w];
        const float total = (float)sqrt(t);
        const float r = __fdiv_rn(1.0f, __fadd_rn(total, 1e-6f));
        float coef = __fmul_rn(r, max_norm);
        coef = coef > 1.0f ? 1.0f : coef;
        out[0] = total;
        out[1] = coef;
    }
}

__global__ void __launch_bounds__(UPD_THREADS)
k_scale_chunks(const regtr_grad_ref* __restrict__ tab, int n_tensors, const float* __restrict__ coef_dev) {
    const long long c = blockIdx.x;
    const int i = owner_of(tab, n_tensors, c);
    float* __restrict__ g = tab[i].g;
    const long long base = (c - tab[i].first) * CHUNK;
    const int len = (int)min((long long)CHUNK, tab[i].n - base);
    const float coef = *coef_dev;
    float* gc = g + base;
    if ((reinterpret_cast<uintptr_t>(gc) & 15) == 0) {
        const int n4 = len >> 2;
        for (int k = threadIdx.x; k < n4; k += UPD_THREADS) {
            float4 v = reinterpret_cast<float4*>(gc)[k];
            v.x = __fmul_rn(v.x, coef); v.y = __fmul_rn(v.y, coef); v.z = __fmul_rn(v.z, coef); v.w = __fmul_rn(v.w, coef);
            reinterpret_cast<float4*>(gc)[k] = v;
        }
        for (int k = (n4 << 2) + threadIdx.x; k < len; k += UPD_THREADS) gc[k] = __fmul_rn(gc[k], coef);
    } else {
        for (int k = threadIdx.x; k < len; k += UPD_THREADS) gc[k] = __fmul_rn(gc[k], coef);
    }
}

// ---- Adam / AdamW -----------------------------------------------------------------------------------------------
// torch 2.11 _single_tensor_adam, one ATen kernel per line there; the roundings follow those kernels (a scalar
// operand is cast to fp32, `a + alpha * b` forms are fused multiply-adds, a division by a host scalar is a product
// with its fp32 reciprocal):
//   decoupled: p = p * decay                     coupled: g = fma(wd, p, g)
//   m = lerp(m, g, w)  (w < 0.5: fma(w, g - m, m), else g - (g - m) * (1 - w))
//   v = fma(1 - b2, g * g, v * b2)
//   p = fma(-step_size, m / (sqrt(v) * rcp_bc2_sqrt + eps), p)
__device__ __forceinline__ void adam_elem(float& p, float g, float& m, float& v, const regtr_adam_tensor& T, bool fresh) {
    if (T.flags & REGTR_ADAM_DECOUPLED) p = __fmul_rn(p, T.decay);
    if (T.flags & REGTR_ADAM_COUPLED) g = __fmaf_rn(T.wd, p, g);
    const float m0 = fresh ? 0.0f : m, v0 = fresh ? 0.0f : v;
    const float d = __fsub_rn(g, m0);
    m = T.b1w < 0.5f ? __fmaf_rn(T.b1w, d, m0) : __fmaf_rn(-d, __fsub_rn(1.0f, T.b1w), g);
    v = __fmaf_rn(T.one_m_b2, __fmul_rn(g, g), __fmul_rn(v0, T.b2));
    const float denom = __fadd_rn(__fmul_rn(__fsqrt_rn(v), T.rcp_bc2_sqrt), T.eps);
    p = __fmaf_rn(T.neg_step_size, __fdiv_rn(m, denom), p);
}

__global__ void __launch_bounds__(UPD_THREADS)
k_adam_chunks(const regtr_adam_tensor* __restrict__ tab, int n_tensors) {
    const long long c = blockIdx.x;
    const int i = owner_of(tab, n_tensors, c);
    const regtr_adam_tensor T = tab[i];
    const long long base = (c - T.first) * CHUNK;
    const int len = (int)min((long long)CHUNK, T.n - base);
    const bool fresh = (T.flags & REGTR_ADAM_FRESH) != 0;
    float* p = T.p + base; const float* g = T.g + base; float* m = T.m + base; float* v = T.v + base;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                       reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    int done = 0;
    if (vec) {
        const int n4 = len >> 2;
        for (int k = threadIdx.x; k < n4; k += UPD_THREADS) {
            float4 P = reinterpret_cast<float4*>(p)[k];
            const float4 G = reinterpret_cast<const float4*>(g)[k];
            float4 M = make_float4(0.f, 0.f, 0.f, 0.f), V = M;
            if (!fresh) { M = reinterpret_cast<float4*>(m)[k]; V = reinterpret_cast<float4*>(v)[k]; }
            adam_elem(P.x, G.x, M.x, V.x, T, fresh);
            adam_elem(P.y, G.y, M.y, V.y, T, fresh);
            adam_elem(P.z, G.z, M.z, V.z, T, fresh);
            adam_elem(P.w, G.w, M.w, V.w, T, fresh);
            reinterpret_cast<float4*>(p)[k] = P;
            reinterpret_cast<float4*>(m)[k] = M;
            reinterpret_cast<float4*>(v)[k] = V;
        }
        done = n4 << 2;
    }
    for (int k = done + threadIdx.x; k < len; k += UPD_THREADS) {
        float P = p[k], M = fresh ? 0.f : m[k], V = fresh ? 0.f : v[k];
        adam_elem(P, g[k], M, V, T, fresh);
        p[k] = P; m[k] = M; v[k] = V;
    }
}

// ---- split refresh ----------------------------------------------------------------------------------------------
// One CTA per 32 x 32 tile of a view: out[a, b] = src[a * s0 + b * s1] goes through shared memory, read along
// whichever stride is 1 and written along the rows of the contiguous (hi, lo) buffers, so both sides coalesce.
__global__ void __launch_bounds__(256)
k_split_refresh(const regtr_split_view* __restrict__ tab, int n_views) {
    __shared__ float tile[32][33];
    const long long t = blockIdx.x;
    const int i = owner_of(tab, n_views, t);
    const regtr_split_view V = tab[i];
    const int tcols = (V.cols + 31) >> 5;
    const int local = (int)(t - V.first);
    const int r0 = (local / tcols) << 5, c0 = (local % tcols) << 5;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    if (V.s0 == 1 && V.s1 != 1) {           // columns of the view are contiguous (a transposed matrix)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int a = r0 + tx, b = c0 + ty + 8 * k;
            if (a < V.rows && b < V.cols) tile[tx][ty + 8 * k] = V.src[(long long)a + (long long)b * V.s1];
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int a = r0 + ty + 8 * k, b = c0 + tx;
            if (a < V.rows && b < V.cols) tile[ty + 8 * k][tx] = V.src[(long long)a * V.s0 + (long long)b * V.s1];
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int a = r0 + ty + 8 * k, b = c0 + tx;
        if (a < V.rows && b < V.cols) {
            const float x = tile[ty + 8 * k][tx], h = regtr_tf32_rne(x);
            const long long o = (long long)a * V.cols + b;
            V.hi[o] = h;
            V.lo[o] = regtr_tf32_rne(x - h);
        }
    }
}

}  // namespace

extern "C" {

size_t regtr_grad_norm_ws_bytes(int n_chunks) { return regtr_align((size_t)(n_chunks > 0 ? n_chunks : 1) * sizeof(double)); }

int regtr_grad_norm(const regtr_grad_ref* table, int n_tensors, int n_chunks, float max_norm, float* out,
                    void* ws, size_t ws_bytes, void* stream_) {
    if (n_tensors < 0 || n_chunks < 0 || !out || (n_chunks > 0 && (!table || n_tensors == 0))) return REGTR_ERR_ARG;
    if (!ws || ws_bytes < regtr_grad_norm_ws_bytes(n_chunks)) return REGTR_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream_;
    double* partial = static_cast<double*>(ws);
    if (n_chunks > 0) k_sumsq_chunks<<<n_chunks, NORM_THREADS, 0, st>>>(table, n_tensors, partial);
    k_norm_finalize<<<1, FIN_THREADS, 0, st>>>(partial, n_chunks, max_norm, out);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_bucket_copy(const regtr_bucket_ref* table, int n_tensors, int n_chunks, float* bucket, int unpack,
                      void* stream_) {
    if (n_tensors < 0 || n_chunks < 0 || !bucket || (n_chunks > 0 && (!table || n_tensors == 0))) return REGTR_ERR_ARG;
    if (n_chunks == 0) return REGTR_OK;
    k_bucket_chunks<<<n_chunks, UPD_THREADS, 0, (cudaStream_t)stream_>>>(table, n_tensors, bucket, unpack != 0);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_grad_scale(const regtr_grad_ref* table, int n_tensors, int n_chunks, const float* coef, void* stream_) {
    if (n_tensors < 0 || n_chunks < 0 || !coef || (n_chunks > 0 && (!table || n_tensors == 0))) return REGTR_ERR_ARG;
    if (n_chunks == 0) return REGTR_OK;
    k_scale_chunks<<<n_chunks, UPD_THREADS, 0, (cudaStream_t)stream_>>>(table, n_tensors, coef);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_adam_step(const regtr_adam_tensor* table, int n_tensors, int n_chunks, void* stream_) {
    if (n_tensors < 0 || n_chunks < 0 || (n_chunks > 0 && (!table || n_tensors == 0))) return REGTR_ERR_ARG;
    if (n_chunks == 0) return REGTR_OK;
    k_adam_chunks<<<n_chunks, UPD_THREADS, 0, (cudaStream_t)stream_>>>(table, n_tensors);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_split_refresh(const regtr_split_view* table, int n_views, int n_tiles, void* stream_) {
    if (n_views < 0 || n_tiles < 0 || (n_tiles > 0 && (!table || n_views == 0))) return REGTR_ERR_ARG;
    if (n_tiles == 0) return REGTR_OK;
    k_split_refresh<<<n_tiles, 256, 0, (cudaStream_t)stream_>>>(table, n_views);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
