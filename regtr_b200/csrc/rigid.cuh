// Internal to the library: float64 rigid-transform helpers shared by the pose solve (kabsch.cu), the training-data
// preparation (traindata.cu), ICP (icp.cu), the pose-graph optimiser (posegraph.cu) and Fast Global Registration
// (fgr.cu).
#pragma once

#include "common.cuh"

namespace {

// ((m0 x + m1 y) + m2 z) + m3 in float64, no contraction: the fixed operation order of every rigid transform here
__device__ __forceinline__ double rt_row(const double* m, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), __dmul_rn(m[2], z)), m[3]);
}

// x = (rx, ry, rz, tx, ty, tz) -> R = Rz(rz) Ry(ry) Rx(rx), t = (tx, ty, tz) (Open3D's TransformVector6dToMatrix4d):
// the update of point-to-plane ICP (icp.cu), of the pose-graph optimiser (posegraph.cu) and of FGR (fgr.cu)
__device__ __forceinline__ void rigid_from_vec6(const double x[6], double R[3][3], double t[3]) {
    double sa, ca, sb, cb, sc, cc;
    sincos(x[0], &sa, &ca);
    sincos(x[1], &sb, &cb);
    sincos(x[2], &sc, &cc);
    R[0][0] = cc * cb; R[0][1] = cc * sb * sa - sc * ca; R[0][2] = cc * sb * ca + sc * sa;
    R[1][0] = sc * cb; R[1][1] = sc * sb * sa + cc * ca; R[1][2] = sc * sb * ca - cc * sa;
    R[2][0] = -sb;     R[2][1] = cb * sa;                R[2][2] = cb * ca;
    for (int r = 0; r < 3; ++r) t[r] = x[3 + r];
}

// Solve A x = -v for the symmetric 6x6 A given by its upper triangle H (row-major) by LDL^T without pivoting, in a
// fixed order.  False, x untouched, when |det A| = |prod D| < 1e-6 or det is not finite (Open3D's
// SolveLinearSystemPSD check).
__device__ __forceinline__ bool solve6_ldlt(const double H[21], const double v[6], double x[6]) {
    double A[6][6], L[6][6], D[6];
#pragma unroll
    for (int a = 0, e = 0; a < 6; ++a)
#pragma unroll
        for (int c = a; c < 6; ++c, ++e) { A[a][c] = H[e]; A[c][a] = H[e]; }
    double det = 1.0;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double d = A[j][j];
#pragma unroll
        for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k] * D[k];
        D[j] = d;
        det *= d;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double a = A[i][j];
#pragma unroll
            for (int k = 0; k < j; ++k) a -= L[i][k] * L[j][k] * D[k];
            L[i][j] = a / d;
        }
    }
    if (!(fabs(det) >= 1e-6) || isinf(det)) return false;
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {                      // L y = -v
        double a = -v[i];
#pragma unroll
        for (int k = 0; k < i; ++k) a -= L[i][k] * y[k];
        y[i] = a;
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {                     // L^T x = D^-1 y
        double a = y[i] / D[i];
#pragma unroll
        for (int k = i + 1; k < 6; ++k) a -= L[k][i] * x[k];
        x[i] = a;
    }
    return true;
}

// The sweeps of svd3_jacobi: one-sided (Hestenes) Jacobi rotations of A's column pairs, accumulated in V, until the
// columns of A (now A_in V) are orthogonal; column j's norm is then the singular value of V's column j (unsorted).
__device__ __forceinline__ void jacobi3_sweeps(double A[3][3], double V[3][3]) {
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
}

// 3x3 SVD A = U diag(S) V^T in fp64: one-sided (Hestenes) Jacobi on A directly (no A^T A squaring of the condition
// number); singular values sorted descending, so that a reflection fix flips the direction of the smallest one.
__device__ void svd3_jacobi(const double A_in[3][3], double U[3][3], double S[3], double V[3][3]) {
    double A[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) { A[i][j] = A_in[i][j]; V[i][j] = (i == j) ? 1.0 : 0.0; }
    jacobi3_sweeps(A, V);
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

}  // namespace
