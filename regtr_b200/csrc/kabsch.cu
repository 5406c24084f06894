// Weighted Kabsch / 3x3 SVD pose solve, one warp per problem.
//
// Replaces compute_rigid_transform (/root/reference/src/utils/se3_torch.py:108-154) and the
// correspondence assembly of RegTR.forward (/root/reference/src/models/regtr.py:185-203).
// Accumulation in fp64 by warp-shuffle reduction; the 3x3 SVD is a one-sided (Hestenes)
// Jacobi in fp64 on lane 0, which works on cov directly (no cov^T cov squaring of the
// condition number); singular values are sorted descending so that the reflection fix
// flips the direction of the smallest one, exactly as `v_neg[..., 2] *= -1` does on
// torch.svd's descending output (se3_torch.py:143-148).
#include "rigid.cuh"

namespace {

struct Mat3 { double m[3][3]; };

// Loader abstraction: point i of a problem -> (a, b, w).
struct PlainLoader {
    const float *a, *b, *w;
    int base;
    __device__ __forceinline__ void get(int i, float3& pa, float3& pb, float& pw) const {
        const size_t r = (size_t)(base + i);
        pa = make_float3(a[3 * r], a[3 * r + 1], a[3 * r + 2]);
        pb = make_float3(b[3 * r], b[3 * r + 1], b[3 * r + 2]);
        pw = w[r];
    }
};

struct CorrLoader {   // regtr.py:185-194 for one (layer, pair)
    const float *kp, *corr, *logit;   // corr/logit already offset to the layer
    int s0, S, t0;                    // src rows [s0, s0+S), tgt rows [t0, ...)
    __device__ __forceinline__ void get(int i, float3& pa, float3& pb, float& pw) const {
        const bool is_src = i < S;
        const size_t r = is_src ? (size_t)(s0 + i) : (size_t)(t0 + i - S);
        const float3 k = make_float3(kp[3 * r], kp[3 * r + 1], kp[3 * r + 2]);
        const float3 c = make_float3(corr[3 * r], corr[3 * r + 1], corr[3 * r + 2]);
        pa = is_src ? k : c;
        pb = is_src ? c : k;
        pw = 1.f / (1.f + expf(-logit[r]));
    }
};

template <class Loader>
__device__ void kabsch_warp(const Loader& ld, int n, float* __restrict__ T, int lane) {
    double sw = 0.0, sa[3] = {0, 0, 0}, sb[3] = {0, 0, 0};
    for (int i = lane; i < n; i += 32) {
        float3 a, b; float w;
        ld.get(i, a, b, w);
        const double dw = (double)w;
        sw += dw;
        sa[0] += dw * a.x; sa[1] += dw * a.y; sa[2] += dw * a.z;
        sb[0] += dw * b.x; sb[1] += dw * b.y; sb[2] += dw * b.z;
    }
    sw = warp_sum(sw);
    for (int d = 0; d < 3; ++d) { sa[d] = warp_sum(sa[d]); sb[d] = warp_sum(sb[d]); }
    const double W = fmax(sw, 1e-6);                 // clamp_min(sum w, _EPS), se3_torch.py:127-128
    double ca[3], cb[3];
    for (int d = 0; d < 3; ++d) { ca[d] = sa[d] / W; cb[d] = sb[d] / W; }
    double cov[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = lane; i < n; i += 32) {
        float3 a, b; float w;
        ld.get(i, a, b, w);
        const double wn = (double)w / W;
        const double da[3] = {a.x - ca[0], a.y - ca[1], a.z - ca[2]};
        const double db[3] = {(b.x - cb[0]) * wn, (b.y - cb[1]) * wn, (b.z - cb[2]) * wn};
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) cov[r][c] += da[r] * db[c];
    }
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) cov[r][c] = warp_sum(cov[r][c]);
    if (lane != 0) return;
    double U[3][3], S[3], V[3][3];
    svd3_jacobi(cov, U, S, V);
    double R[3][3];
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) R[r][c] = V[r][0] * U[c][0] + V[r][1] * U[c][1] + V[r][2] * U[c][2];
    if (!(det3(R) > 0.0)) {
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) R[r][c] = V[r][0] * U[c][0] + V[r][1] * U[c][1] - V[r][2] * U[c][2];
    }
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) T[4 * r + c] = (float)R[r][c];
        T[4 * r + 3] = (float)(cb[r] - (R[r][0] * ca[0] + R[r][1] * ca[1] + R[r][2] * ca[2]));
    }
}

__global__ void k_kabsch(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ w,
                         const int32_t* __restrict__ offs, int n_problems, float* __restrict__ T) {
    const int prob = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (prob >= n_problems) return;
    PlainLoader ld{a, b, w, offs[prob]};
    kabsch_warp(ld, offs[prob + 1] - offs[prob], T + 12 * (size_t)prob, lane);
}

__global__ void k_pose_from_corr(const float* __restrict__ kp, const float* __restrict__ corr,
                                 const float* __restrict__ logit, const int32_t* __restrict__ offs, int n, int B, int L,
                                 float* __restrict__ pose) {
    const int prob = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (prob >= L * B) return;
    const int l = prob / B, b = prob % B;
    const int s0 = offs[b], S = offs[b + 1] - offs[b], t0 = offs[B + b], Tn = offs[B + b + 1] - offs[B + b];
    CorrLoader ld{kp, corr + (size_t)l * n * 3, logit + (size_t)l * n, s0, S, t0};
    kabsch_warp(ld, S + Tn, pose + 12 * (size_t)prob, lane);
}

}  // namespace

extern "C" {

int regtr_kabsch_fwd(const float* a, const float* b, const float* w, const int32_t* offs, int n_problems, float* T,
                     void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n_problems < 0) return REGTR_ERR_ARG;
    if (n_problems == 0) return REGTR_OK;
    if (!a || !b || !w || !offs || !T) return REGTR_ERR_ARG;
    k_kabsch<<<regtr_cdiv((long long)n_problems * 32, 128), 128, 0, st>>>(a, b, w, offs, n_problems, T);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_pose_from_corr(const float* kp, const float* corr, const float* logit, const int32_t* offs, int n, int B,
                         int L, float* pose, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (n < 0 || B < 0 || L < 0) return REGTR_ERR_ARG;
    if (B == 0 || L == 0) return REGTR_OK;
    if (!kp || !corr || !logit || !offs || !pose) return REGTR_ERR_ARG;
    k_pose_from_corr<<<regtr_cdiv((long long)L * B * 32, 128), 128, 0, st>>>(kp, corr, logit, offs, n, B, L, pose);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

int regtr_status_clear(uint32_t* status, void* stream_) {
    if (!status) return REGTR_ERR_ARG;
    return cudaMemsetAsync(status, 0, sizeof(uint32_t), (cudaStream_t)stream_) == cudaSuccess ? REGTR_OK : REGTR_ERR_ARG;
}

int regtr_version(void) { return 1; }

const char* regtr_build_info(void) {
    return "regtr_b200 ABI 1; nvcc " __DATE__ "; -gencode arch=compute_90a,code=sm_90a -lineinfo";
}

}  // extern "C"
