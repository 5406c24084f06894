// Weighted Kabsch / 3x3 SVD pose solve, one warp per problem.
//
// Replaces compute_rigid_transform (/root/reference/src/utils/se3_torch.py:108-154) and the
// correspondence assembly of RegTR.forward (/root/reference/src/models/regtr.py:185-203).
// Accumulation in fp64 by warp-shuffle reduction; the 3x3 SVD is a one-sided (Hestenes)
// Jacobi in fp64 on lane 0, which works on cov directly (no cov^T cov squaring of the
// condition number); singular values are sorted descending so that the reflection fix
// flips the direction of the smallest one, exactly as `v_neg[..., 2] *= -1` does on
// torch.svd's descending output (se3_torch.py:143-148).
#include "common.cuh"

namespace {

struct Mat3 { double m[3][3]; };

__device__ void svd3_jacobi(const double A_in[3][3], double U[3][3], double S[3], double V[3][3]) {
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { A[i][j] = A_in[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0;
        for (int p = 0; p < 2; ++p) {
            for (int q = p + 1; q < 3; ++q) {
                double alpha = 0.0, beta = 0.0, gamma = 0.0;
                for (int i = 0; i < 3; ++i) {
                    alpha += A[i][p] * A[i][p];
                    beta += A[i][q] * A[i][q];
                    gamma += A[i][p] * A[i][q];
                }
                if (gamma == 0.0) continue;
                const double lim = sqrt(alpha * beta);
                if (fabs(gamma) <= 1e-300 || fabs(gamma) <= 1e-17 * lim) continue;
                off = fmax(off, fabs(gamma) / (lim > 0.0 ? lim : 1.0));
                const double zeta = (beta - alpha) / (2.0 * gamma);
                const double t = (zeta >= 0.0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
                const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
                for (int i = 0; i < 3; ++i) {
                    const double ap = A[i][p], aq = A[i][q];
                    A[i][p] = c * ap - s * aq;
                    A[i][q] = s * ap + c * aq;
                    const double vp = V[i][p], vq = V[i][q];
                    V[i][p] = c * vp - s * vq;
                    V[i][q] = s * vp + c * vq;
                }
            }
        }
        if (off < 1e-15) break;
    }
    for (int j = 0; j < 3; ++j) S[j] = sqrt(A[0][j] * A[0][j] + A[1][j] * A[1][j] + A[2][j] * A[2][j]);
    // sort columns by descending singular value
    int ord[3] = {0, 1, 2};
    for (int a = 0; a < 2; ++a)
        for (int b = a + 1; b < 3; ++b)
            if (S[ord[b]] > S[ord[a]]) { int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
    double As[3][3], Vs[3][3], Ss[3];
    for (int j = 0; j < 3; ++j) {
        Ss[j] = S[ord[j]];
        for (int i = 0; i < 3; ++i) { As[i][j] = A[i][ord[j]]; Vs[i][j] = V[i][ord[j]]; }
    }
    for (int j = 0; j < 3; ++j) {
        S[j] = Ss[j];
        for (int i = 0; i < 3; ++i) V[i][j] = Vs[i][j];
    }
    // U columns = A columns / sigma; complete degenerate directions by cross products
    const double tiny = 1e-200 + 1e-14 * S[0];
    for (int j = 0; j < 3; ++j) {
        if (S[j] > tiny) {
            for (int i = 0; i < 3; ++i) U[i][j] = As[i][j] / S[j];
        } else if (j == 0) {
            U[0][0] = 1.0; U[1][0] = 0.0; U[2][0] = 0.0;
        } else if (j == 1) {
            // any unit vector orthogonal to u0
            const double ax = fabs(U[0][0]), ay = fabs(U[1][0]), az = fabs(U[2][0]);
            double e[3] = {0.0, 0.0, 0.0};
            if (ax <= ay && ax <= az) e[0] = 1.0; else if (ay <= az) e[1] = 1.0; else e[2] = 1.0;
            double d = e[0] * U[0][0] + e[1] * U[1][0] + e[2] * U[2][0];
            double w[3] = {e[0] - d * U[0][0], e[1] - d * U[1][0], e[2] - d * U[2][0]};
            const double n = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
            for (int i = 0; i < 3; ++i) U[i][1] = w[i] / n;
        } else {
            U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
            U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
            U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
        }
    }
}

__device__ __forceinline__ double det3(const double M[3][3]) {
    return M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
           M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
}

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
