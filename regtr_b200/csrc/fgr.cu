// Fast Global Registration for B pairs at once: Open3D's registration_fgr_based_on_correspondence and the solve of
// registration_fgr_based_on_feature_matching (Zhou, Park and Koltun, ECCV 2016) with FastGlobalRegistrationOption,
// restated as one deterministic rule (DESIGN.md section 8, "Fast Global Registration"; include/regtr_b200.h,
// regtr_fgr).
//
// Two launches whatever the data.  k_fgr_prepare (one CTA per pair): the clouds' means and scale, the valid
// correspondences compacted and normalised in their original order, then the tuple test (one trial per thread, an
// in-order block scan appends the passes and stops at the cap) or a plain copy; the result is the correspondence list
// of the solve.  k_fgr_solve (one CTA per pair): the graduated non-convexity iterations, each a fixed-order block
// reduction of the 27 normal-equation sums, thread 0's LDL^T solve and update, and the moved target points kept in the
// workspace.  Every sum has a fixed order, nothing uses value atomics and nothing waits on the host, so a pair gets the
// same bits alone or in a batch with the same pair_base + b.
#include <cfloat>
#include <climits>

#include "philox.cuh"
#include "rigid.cuh"

namespace {

constexpr int PREP_THREADS = 512;
constexpr int PREP_WARPS = PREP_THREADS / 32;
constexpr int SOLVE_THREADS = 256;
constexpr int SOLVE_WARPS = SOLVE_THREADS / 32;
constexpr unsigned FGR_WORD3 = 0x46475254u;      // "FGRT": counter word 3 of every tuple draw

// Per-pair state handed from k_fgr_prepare to k_fgr_solve.
struct FgrPair {
    double mu_s[3], mu_t[3];
    double sg, par0;                               // sigma_g and the initial par
    int n_corr;                                    // correspondences of the solve
    int tuples, trials;
};

__device__ __forceinline__ double norm3_rn(double dx, double dy, double dz) {
    return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// Fixed-order block sum of N per-thread values: each warp's lanes by the xor butterfly (lane 0's value is the halving
// tree of the 32 lanes), then thread e < N adds the W warp sums of value e by a halving tree into tot[e].  Ends with a
// barrier, so every thread may read tot; s and tot are free again after the caller's next barrier.
template <int N, int W>
__device__ __forceinline__ void block_sum(double (&v)[N], double (*s)[W], double* tot, int t, int lane, int warp) {
#pragma unroll
    for (int e = 0; e < N; ++e) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[e] = __dadd_rn(v[e], __shfl_xor_sync(0xffffffffu, v[e], o));
    }
    if (lane == 0) {
#pragma unroll
        for (int e = 0; e < N; ++e) s[e][warp] = v[e];
    }
    __syncthreads();
    if (t < N) {
        double w[W];
#pragma unroll
        for (int i = 0; i < W; ++i) w[i] = s[t][i];
#pragma unroll
        for (int h = W / 2; h > 0; h >>= 1)
#pragma unroll
            for (int i = 0; i < W / 2; ++i)
                if (i < h) w[i] = __dadd_rn(w[i], w[i + h]);
        tot[t] = w[0];
    }
    __syncthreads();
}

// One CTA per pair.
// 1. mu_s, mu_t: thread t adds points t, t + 512, ... of the cloud in order, then block_sum; / n (0 without points).
//    sigma = the largest |p - mu| over both clouds (1 when that is 0); sigma_g, par0 by use_absolute_scale.
// 2. The valid correspondences (mask[i] != 0, every one without a mask) in their original order, normalised as
//    (a - mu_s) / sigma_g, (c - mu_t) / sigma_g into ka / kc from coffs[b]: n of them.
// 3. With the tuple test and n > 0: rounds of 512 trials k (k < 100 n), trial k drawing mulhi32(w_e, n) from
//    Philox4x32-10 at (k, pair_base + b, 0, "FGRT"); the passes of a round are appended in k order (three
//    correspondences each) until maximum_tuple_count, and the walk ends right after the pass that reaches it.
//    Otherwise the n correspondences are copied.  The solve's list goes to gp / gq from goffs = coffs[b] + 3 cap b.
__global__ void __launch_bounds__(PREP_THREADS)
k_fgr_prepare(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
              const double* __restrict__ ca, const double* __restrict__ cc, const int32_t* __restrict__ coffs,
              const uint8_t* __restrict__ mask, int use_abs, int tuple_test, double tuple_scale, int cap, unsigned k0,
              unsigned k1, int pair_base, double* __restrict__ ka, double* __restrict__ kc, double* __restrict__ gp,
              double* __restrict__ gq, FgrPair* __restrict__ pst) {
    __shared__ double s_red[3][PREP_WARPS];
    __shared__ double s_tot[3];
    __shared__ int s_cnt[PREP_WARPS];
    __shared__ int s_last;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    double mu[2][3];
#pragma unroll
    for (int side = 0; side < 2; ++side) {
        const int c = side * B + b, i0 = offs[c], i1 = offs[c + 1];
        double acc[3] = {0.0, 0.0, 0.0};
        for (int i = i0 + t; i < i1; i += PREP_THREADS)
#pragma unroll
            for (int a = 0; a < 3; ++a) acc[a] = __dadd_rn(acc[a], xyz[3 * (size_t)i + a]);
        block_sum<3, PREP_WARPS>(acc, s_red, s_tot, t, lane, warp);
#pragma unroll
        for (int a = 0; a < 3; ++a) mu[side][a] = i1 > i0 ? __ddiv_rn(s_tot[a], (double)(i1 - i0)) : 0.0;
        __syncthreads();
    }
    double mx = 0.0;
#pragma unroll
    for (int side = 0; side < 2; ++side) {
        const int c = side * B + b;
        for (int i = offs[c] + t; i < offs[c + 1]; i += PREP_THREADS) {
            const double* p = xyz + 3 * (size_t)i;
            mx = fmax(mx, norm3_rn(__dsub_rn(p[0], mu[side][0]), __dsub_rn(p[1], mu[side][1]),
                                   __dsub_rn(p[2], mu[side][2])));
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) s_red[0][warp] = mx;
    __syncthreads();
    for (int w = 0; w < PREP_WARPS; ++w) mx = fmax(mx, s_red[0][w]);
    const double sigma = mx > 0.0 ? mx : 1.0;
    const double sg = use_abs ? 1.0 : sigma, par0 = use_abs ? sigma : 1.0;

    const int m0 = coffs[b], m1 = coffs[b + 1];
    int n = 0;                                                  // valid correspondences before this round
    for (int r = m0; r < m1; r += PREP_THREADS) {
        const int i = r + t;
        const int f = i < m1 && (!mask || mask[i] != 0);
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_cnt[warp] = __popc(bal);
        __syncthreads();
        int before = n, total = n;
        for (int w = 0; w < PREP_WARPS; ++w) {
            if (w < warp) before += s_cnt[w];
            total += s_cnt[w];
        }
        if (f) {
            const size_t o = 3 * (size_t)(m0 + before + __popc(bal & ((1u << lane) - 1u)));
#pragma unroll
            for (int a = 0; a < 3; ++a) {
                ka[o + a] = __ddiv_rn(__dsub_rn(ca[3 * (size_t)i + a], mu[0][a]), sg);
                kc[o + a] = __ddiv_rn(__dsub_rn(cc[3 * (size_t)i + a], mu[1][a]), sg);
            }
        }
        n = total;
        __syncthreads();                                        // s_cnt is reused; ka / kc are complete after the loop
    }

    const double* A = ka + 3 * (size_t)m0;
    const double* C = kc + 3 * (size_t)m0;
    const size_t g0 = 3 * ((size_t)m0 + 3 * (size_t)cap * b);
    int tuples = 0, trials = 0;
    if (tuple_test && n > 0) {
        const long long total = 100ll * n;
        for (long long r = 0; r < total && tuples < cap; r += PREP_THREADS) {
            const long long k = r + t;
            int idx[3] = {0, 0, 0};
            bool pass = false;
            if (k < total) {
                const U4 v = philox(U4{(unsigned)k, (unsigned)(pair_base + b), 0u, FGR_WORD3}, k0, k1);
                idx[0] = (int)__umulhi(v.x, (unsigned)n);
                idx[1] = (int)__umulhi(v.y, (unsigned)n);
                idx[2] = (int)__umulhi(v.z, (unsigned)n);
                pass = true;
#pragma unroll
                for (int e = 0; e < 3; ++e) {
                    const double* a0 = A + 3 * idx[e]; const double* a1 = A + 3 * idx[e == 2 ? 0 : e + 1];
                    const double* c0 = C + 3 * idx[e]; const double* c1 = C + 3 * idx[e == 2 ? 0 : e + 1];
                    const double ls = norm3_rn(__dsub_rn(a0[0], a1[0]), __dsub_rn(a0[1], a1[1]), __dsub_rn(a0[2], a1[2]));
                    const double lt = norm3_rn(__dsub_rn(c0[0], c1[0]), __dsub_rn(c0[1], c1[1]), __dsub_rn(c0[2], c1[2]));
                    pass = pass && __dmul_rn(ls, tuple_scale) < lt && lt < __ddiv_rn(ls, tuple_scale);
                }
            }
            const unsigned bal = __ballot_sync(0xffffffffu, pass);
            if (lane == 0) s_cnt[warp] = __popc(bal);
            __syncthreads();
            int before = tuples, passes = 0;
            for (int w = 0; w < PREP_WARPS; ++w) {
                if (w < warp) before += s_cnt[w];
                passes += s_cnt[w];
            }
            const int slot = before + __popc(bal & ((1u << lane) - 1u));
            if (pass && slot < cap) {
#pragma unroll
                for (int e = 0; e < 3; ++e)
#pragma unroll
                    for (int a = 0; a < 3; ++a) {
                        gp[g0 + 9 * (size_t)slot + 3 * e + a] = A[3 * idx[e] + a];
                        gq[g0 + 9 * (size_t)slot + 3 * e + a] = C[3 * idx[e] + a];
                    }
                if (slot == cap - 1) s_last = (int)k;
            }
            __syncthreads();
            if (tuples + passes >= cap) {
                trials = s_last + 1;
                tuples = cap;
            } else {
                trials = (int)(r + PREP_THREADS < total ? r + PREP_THREADS : total);
                tuples += passes;
            }
            __syncthreads();                                    // s_cnt / s_last are reused
        }
    } else {
        for (int i = t; i < 3 * n; i += PREP_THREADS) { gp[g0 + i] = A[i]; gq[g0 + i] = C[i]; }
    }
    if (t == 0) {
        FgrPair s;
#pragma unroll
        for (int a = 0; a < 3; ++a) { s.mu_s[a] = mu[0][a]; s.mu_t[a] = mu[1][a]; }
        s.sg = sg; s.par0 = par0;
        s.n_corr = tuple_test && n > 0 ? 3 * tuples : n;
        s.tuples = tuples; s.trials = trials;
        pst[b] = s;
    }
}

// One CTA per pair: the graduated non-convexity solve of OptimizePairwiseRegistration on the list of k_fgr_prepare.
// Fewer than 10 correspondences: the identity.  Otherwise T = I, par = par0 and per iteration: correspondence c
// (thread c % 256, in ascending order) moves its q by the previous update (kept in gq), r = p - q,
// s = (par / (r.r + par))^2, and rows x, y, z add (J_a J_b) s to the 21 upper J^T J sums and (J_a r) s to the 6
// J^T r sums; block_sum; thread 0 solves J^T J x = -J^T r by solve6_ldlt, and on success delta = rigid_from_vec6(x),
// T = delta T (a failed solve leaves T and the points alone); then par /= division_factor when decrease_mu,
// itr % 4 == 0 and par > max_dist.  pose_out = R^T, -R^T (-R mu_t + sigma_g t + mu_s); result = (correspondences,
// tuples, trials, par).
__global__ void __launch_bounds__(SOLVE_THREADS)
k_fgr_solve(const int32_t* __restrict__ coffs, const FgrPair* __restrict__ pst, int iters, double max_dist,
            double division, int decrease_mu, int cap, const double* __restrict__ gp, double* __restrict__ gq,
            double* __restrict__ pose_out, double* __restrict__ result) {
    __shared__ double s_red[27][SOLVE_WARPS];
    __shared__ double s_tot[27];
    __shared__ double s_delta[12], s_T[12];
    __shared__ int s_ok;
    const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const FgrPair st = pst[b];
    const int n = st.n_corr;
    const size_t g0 = 3 * ((size_t)coffs[b] + 3 * (size_t)cap * b);
    const double* P = gp + g0;
    double* Q = gq + g0;
    double par = st.par0;
    double* T = s_T;                                            // thread 0's pose, normalised target -> source
    if (t < 12) T[t] = (t % 5 == 0) ? 1.0 : 0.0;
    if (t == 0) s_ok = 0;
    __syncthreads();
    for (int itr = 0; n >= 10 && itr < iters; ++itr) {
        double acc[27];
#pragma unroll
        for (int e = 0; e < 27; ++e) acc[e] = 0.0;
        const bool move = s_ok != 0;
        for (int c = t; c < n; c += SOLVE_THREADS) {
            double q[3] = {Q[3 * c], Q[3 * c + 1], Q[3 * c + 2]};
            if (move) {
                const double x = q[0], y = q[1], z = q[2];
                q[0] = rt_row(s_delta, x, y, z); q[1] = rt_row(s_delta + 4, x, y, z); q[2] = rt_row(s_delta + 8, x, y, z);
                Q[3 * c] = q[0]; Q[3 * c + 1] = q[1]; Q[3 * c + 2] = q[2];
            }
            const double r[3] = {__dsub_rn(P[3 * c], q[0]), __dsub_rn(P[3 * c + 1], q[1]), __dsub_rn(P[3 * c + 2], q[2])};
            const double rr = __dadd_rn(__dadd_rn(__dmul_rn(r[0], r[0]), __dmul_rn(r[1], r[1])), __dmul_rn(r[2], r[2]));
            const double tmp = __ddiv_rn(par, __dadd_rn(rr, par));
            const double s = __dmul_rn(tmp, tmp);
#pragma unroll
            for (int row = 0; row < 3; ++row) {
                double J[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
                if (row == 0) { J[1] = -q[2]; J[2] = q[1]; J[3] = -1.0; }
                if (row == 1) { J[0] = q[2]; J[2] = -q[0]; J[4] = -1.0; }
                if (row == 2) { J[0] = -q[1]; J[1] = q[0]; J[5] = -1.0; }
#pragma unroll
                for (int a = 0, e = 0; a < 6; ++a)
#pragma unroll
                    for (int bb = a; bb < 6; ++bb, ++e) acc[e] = __dadd_rn(acc[e], __dmul_rn(__dmul_rn(J[a], J[bb]), s));
#pragma unroll
                for (int a = 0; a < 6; ++a) acc[21 + a] = __dadd_rn(acc[21 + a], __dmul_rn(__dmul_rn(J[a], r[row]), s));
            }
        }
        block_sum<27, SOLVE_WARPS>(acc, s_red, s_tot, t, lane, warp);
        if (t == 0) {
            double H[21], v[6], x[6];
#pragma unroll
            for (int e = 0; e < 21; ++e) H[e] = s_tot[e];
#pragma unroll
            for (int e = 0; e < 6; ++e) v[e] = s_tot[21 + e];
            const bool ok = solve6_ldlt(H, v, x);
            if (ok) {
                double R[3][3], tr[3];
                rigid_from_vec6(x, R, tr);
                double D[12], N[12];
                for (int rw = 0; rw < 3; ++rw) {
                    for (int c = 0; c < 3; ++c) D[4 * rw + c] = R[rw][c];
                    D[4 * rw + 3] = tr[rw];
                }
                for (int rw = 0; rw < 3; ++rw)
                    for (int c = 0; c < 4; ++c)
                        N[4 * rw + c] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(D[4 * rw], T[c]), __dmul_rn(D[4 * rw + 1], T[4 + c])),
                                                            __dmul_rn(D[4 * rw + 2], T[8 + c])),
                                                  c == 3 ? D[4 * rw + 3] : 0.0);
                for (int e = 0; e < 12; ++e) { T[e] = N[e]; s_delta[e] = D[e]; }
            }
            s_ok = ok ? 1 : 0;
        }
        if (decrease_mu && itr % 4 == 0 && par > max_dist) par = __ddiv_rn(par, division);
        __syncthreads();                                        // s_delta / s_ok published, s_red free again
    }
    if (t != 0) return;
    double* o = pose_out + 12 * b;
    if (n < 10) {
        for (int e = 0; e < 12; ++e) o[e] = (e % 5 == 0) ? 1.0 : 0.0;
    } else {
        double u[3];
        for (int rw = 0; rw < 3; ++rw)
            u[rw] = __dadd_rn(__dadd_rn(-(T[4 * rw] * st.mu_t[0] + T[4 * rw + 1] * st.mu_t[1] + T[4 * rw + 2] * st.mu_t[2]),
                                        __dmul_rn(T[4 * rw + 3], st.sg)),
                              st.mu_s[rw]);
        for (int rw = 0; rw < 3; ++rw) {
            for (int c = 0; c < 3; ++c) o[4 * rw + c] = T[4 * c + rw];
            o[4 * rw + 3] = -(T[rw] * u[0] + T[4 + rw] * u[1] + T[8 + rw] * u[2]);
        }
    }
    double* res = result + 4 * b;
    res[0] = (double)n; res[1] = (double)st.tuples; res[2] = (double)st.trials; res[3] = par;
}

struct FgrWs {
    double *ka, *kc, *gp, *gq;
    FgrPair* pst;
    size_t total;
};

FgrWs carve_fgr(void* ws, int m_cap, int B, int cap) {
    FgrWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t m = (size_t)m_cap, g = m + 3 * (size_t)cap * (size_t)B;
    w.ka = (double*)take(sizeof(double) * 3 * m);
    w.kc = (double*)take(sizeof(double) * 3 * m);
    w.gp = (double*)take(sizeof(double) * 3 * g);
    w.gq = (double*)take(sizeof(double) * 3 * g);
    w.pst = (FgrPair*)take(sizeof(FgrPair) * (size_t)B);
    w.total = off;
    return w;
}

}  // namespace

extern "C" {

size_t regtr_fgr_ws_bytes(int m_cap, int B, int maximum_tuple_count) {
    const int cap = maximum_tuple_count >= 1 && maximum_tuple_count <= REGTR_FGR_MAX_TUPLES ? maximum_tuple_count : 1;
    return carve_fgr(nullptr, m_cap > 0 ? m_cap : 1, B > 0 ? B : 1, cap).total;
}

int regtr_fgr(const double* xyz, const int32_t* offs, int B, int n_cap, const double* corr_src,
              const double* corr_tgt, const int32_t* coffs, const uint8_t* corr_mask, int m_cap,
              const regtr_fgr_options* opt, double* pose_out, double* result, void* ws, size_t ws_bytes,
              void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !coffs || !opt || !pose_out || !result || !ws || B <= 0 || n_cap < 0 || m_cap < 0 ||
        m_cap > REGTR_FGR_MAX_CORR || (n_cap > 0 && !xyz) || (m_cap > 0 && (!corr_src || !corr_tgt)))
        return REGTR_ERR_ARG;
    const regtr_fgr_options o = *opt;
    if (!(o.division_factor > 0.0 && o.division_factor <= DBL_MAX) ||
        !(o.maximum_correspondence_distance > 0.0 && o.maximum_correspondence_distance <= DBL_MAX) ||
        o.iteration_number < 0 || !(o.tuple_scale > 0.0 && o.tuple_scale <= 1.0) || o.maximum_tuple_count < 1 ||
        o.maximum_tuple_count > REGTR_FGR_MAX_TUPLES || o.pair_base < 0 || o.pair_base > INT_MAX - B)
        return REGTR_ERR_ARG;
    const int mc = m_cap > 0 ? m_cap : 1;
    FgrWs w = carve_fgr(ws, mc, B, o.maximum_tuple_count);
    if (ws_bytes < w.total) return REGTR_ERR_WORKSPACE;
    k_fgr_prepare<<<B, PREP_THREADS, 0, st>>>(xyz, offs, B, corr_src, corr_tgt, coffs, corr_mask,
                                              o.use_absolute_scale != 0, o.tuple_test != 0, o.tuple_scale,
                                              o.maximum_tuple_count, (unsigned)o.seed, (unsigned)(o.seed >> 32),
                                              o.pair_base, w.ka, w.kc, w.gp, w.gq, w.pst);
    REGTR_CHECK_LAUNCH();
    k_fgr_solve<<<B, SOLVE_THREADS, 0, st>>>(coffs, w.pst, o.iteration_number, o.maximum_correspondence_distance,
                                             o.division_factor, o.decrease_mu != 0, o.maximum_tuple_count, w.gp,
                                             w.gq, pose_out, result);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
