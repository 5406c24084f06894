// ICP of B pairs at once: Open3D's registration_icp with TransformationEstimationPointToPoint (no scaling),
// TransformationEstimationPointToPlane(kernel), or registration_generalized_icp with
// TransformationEstimationForGeneralizedICP(epsilon, kernel), or registration_colored_icp with
// TransformationEstimationForColoredICP(lambda_geometric, kernel), and ICPConvergenceCriteria, restated with this
// library's determinism rules (DESIGN.md section 8, "ICP").  Point-to-point has its own two-pass reduction.  The
// point-to-plane family (L2, a robust kernel, generalized ICP, colored ICP) shares one reduction body (icp.cuh) and one
// record.  Its mode is a template argument, so L2 compiles without the weight and keeps two CTAs per SM (a runtime
// loss would cost it 30 registers); the colored mode is instantiated in color.cu.
// Both methods share the update kernel, with the method as a template argument.
//
// Stacked clouds as in the registration fit: src_0..src_{B-1}, tgt_0..tgt_{B-1} (float64) with int32 device offsets.
// One cell list over the targets is built once; then every round is a fixed sequence of three launches (nearest
// neighbours, per-chunk sums, per-pair update) enqueued without a host synchronisation.  A pair that has converged
// reads its `done` flag on the device and skips its work, so the launch count depends on max_iter alone.
#include "icp.cuh"

extern "C" int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                                    void* grid, int32_t* order, uint32_t* status, void* ws, size_t ws_bytes,
                                    void* state, size_t state_bytes, void* stream);
extern "C" size_t regtr_cellgrid_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_ws_bytes(int n_cap);
extern "C" size_t regtr_cellgrid_state_bytes(int n_cap);
extern "C" double regtr_overlap_coord_bound(double radius, float cell);

namespace {

constexpr int NN_WARPS = 8;
constexpr int PART_POINT = 17;         // k, sum d2, mean_src[3], mean_tgt[3], C[9] per chunk
constexpr int UPD_THREADS = 64;

// P = init . source (rt_row order), the fp32 copy of the targets for their cell list, the targets' own offsets
// (tofs[c] = offs[B + c] - offs[B]), the chunk prefix of the reduction (pair b owns chunks [cpre[b], cpre[b+1]),
// ceil(n_b / CHUNK) of them) and the initial per-pair state.  |coordinate| of a moved source or a target beyond
// `bound`, or not finite, raises REGTR_STATUS_RANGE.
__global__ void k_icp_init(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, int n_cap,
                           const double* __restrict__ init, double bound, double* __restrict__ P,
                           float* __restrict__ x32, int32_t* __restrict__ tofs, int32_t* __restrict__ cpre,
                           IcpPair* __restrict__ pst, double* __restrict__ pose_out, double* __restrict__ result,
                           uint32_t* status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i <= B) tofs[i] = offs[B + i] - offs[B];
    if (i < B) {
        IcpPair s;
        for (int k = 0; k < 12; ++k) { s.upd[k] = (k % 5 == 0) ? 1.0 : 0.0; pose_out[12 * i + k] = init[12 * i + k]; }
        s.fit = 0.0; s.rmse = 0.0; s.k = 0; s.iters = 0; s.done = 0; s.pad = 0;
        pst[i] = s;
        for (int k = 0; k < 4; ++k) result[4 * i + k] = 0.0;
    }
    if (i == 0) {
        int acc = 0;
        cpre[0] = 0;
        for (int b = 0; b < B; ++b) { acc += (offs[b + 1] - offs[b] + CHUNK - 1) / CHUNK; cpre[b + 1] = acc; }
    }
    if (i >= n_cap || i >= offs[2 * B]) return;
    const int c = regtr_cloud_of(offs, 2 * B, i);
    double x = xyz[3 * i + 0], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (c < B) {
        const double* m = init + 12 * c;
        const double ax = rt_row(m, x, y, z), ay = rt_row(m + 4, x, y, z), az = rt_row(m + 8, x, y, z);
        x = ax; y = ay; z = az;
        P[3 * i + 0] = x; P[3 * i + 1] = y; P[3 * i + 2] = z;
    } else {
        const int j = i - offs[B];
        x32[3 * j + 0] = (float)x; x32[3 * j + 1] = (float)y; x32[3 * j + 2] = (float)z;
    }
    if (!(fabs(x) <= bound && fabs(y) <= bound && fabs(z) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
}

// One warp per source point, in index order.  After round 0 the point is first moved in place by its pair's update
// (rt_row), and range-checked.  Then k_overlap_nn's search against the targets' cell list: lanes 0..26 look up one
// stencil cell each, candidates are flattened 32 wide, d2 = (dx dx + dy dy) + dz dz in float64 without contraction,
// the nearest target with d2 < r2 wins and equal distances go to the lowest index.  nn[i] = the stacked index of
// that target point or -1, d2[i] its squared distance.  Pairs that are done are skipped.
__global__ void __launch_bounds__(NN_WARPS * 32, 8)     // 8 CTAs per SM, as the grid is sized
k_icp_nn(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B, int n_cap, double* __restrict__ P,
         const IcpPair* __restrict__ pst, int apply, const CellSlot* __restrict__ table, int log2t,
         const float4* __restrict__ sxyzi, float cell, double r2, double bound, int32_t* __restrict__ nn,
         double* __restrict__ d2o, uint32_t* status) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int n_src = offs[B], t0 = offs[B];
    for (int qi = blockIdx.x * NN_WARPS + warp; qi < n_cap && qi < n_src; qi += gridDim.x * NN_WARPS) {
        const int b = regtr_cloud_of(offs, B, qi);
        if (pst[b].done) continue;
        double qx = P[3 * qi + 0], qy = P[3 * qi + 1], qz = P[3 * qi + 2];
        if (apply) {
            const double* m = pst[b].upd;
            const double ax = rt_row(m, qx, qy, qz), ay = rt_row(m + 4, qx, qy, qz), az = rt_row(m + 8, qx, qy, qz);
            qx = ax; qy = ay; qz = az;
            __syncwarp();
            if (lane == 0) {
                P[3 * qi + 0] = qx; P[3 * qi + 1] = qy; P[3 * qi + 2] = qz;
                if (!(fabs(qx) <= bound && fabs(qy) <= bound && fabs(qz) <= bound)) atomicOr(status, REGTR_STATUS_RANGE);
            }
        }
        const int cx = regtr_cell_of((float)qx, cell), cy = regtr_cell_of((float)qy, cell),
                  cz = regtr_cell_of((float)qz, cell);
        int c_start = 0, c_cnt = 0;
        if (lane < 27) {
            const int x = cx + lane / 9 - 1, y = cy + (lane / 3) % 3 - 1, z = cz + lane % 3 - 1;
            if (x >= -32767 && x <= 32767 && y >= -32767 && y <= 32767 && z >= -32767 && z <= 32767)
                cell_lookup(table, log2t, regtr_pack_key(b, x, y, z), c_start, c_cnt);
        }
        int pre = c_cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, pre, o);
            if (lane >= o) pre += v;
        }
        const int total = __shfl_sync(0xffffffffu, pre, 31);
        double best = r2;
        int bi = -1;
        for (int base = 0; base < total; base += 32) {
            const int t = base + lane;
            int cellid = 0;
#pragma unroll
            for (int step = 16; step > 0; step >>= 1) {
                const int pv = __shfl_sync(0xffffffffu, pre, cellid + step - 1);
                if (pv <= t) cellid += step;
            }
            const int cell_pre = __shfl_sync(0xffffffffu, pre, cellid);
            const int cell_cnt = __shfl_sync(0xffffffffu, c_cnt, cellid);
            const int cell_start = __shfl_sync(0xffffffffu, c_start, cellid);
            if (t < total) {
                const int j = t0 + __float_as_int(sxyzi[cell_start + (t - (cell_pre - cell_cnt))].w);
                const double dx = __dsub_rn(qx, xyz[3 * j + 0]), dy = __dsub_rn(qy, xyz[3 * j + 1]),
                             dz = __dsub_rn(qz, xyz[3 * j + 2]);
                const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
                if (d2 < best || (d2 == best && bi >= 0 && j < bi)) { best = d2; bi = j; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (bi < 0 || ob < best || (ob == best && oi < bi))) { best = ob; bi = oi; }
        }
        if (lane == 0) { nn[qi] = bi; d2o[qi] = best; }
    }
}

// One CTA per chunk of CHUNK consecutive source points of one pair (chunks never straddle pairs, so the sums do not
// depend on the batch).  Over the chunk's correspondences: count, sum of d2 and the two means, then, in a second pass
// over the same points, C = sum (q - mean_q)(p - mean_p)^T (target rows, source columns).  part[g] = (k, sum d2,
// mean_p, mean_q, C).  Fixed per-thread strides and a fixed tree: deterministic, no atomics.
__global__ void __launch_bounds__(RED_THREADS)
k_icp_reduce_point(const double* __restrict__ xyz, const int32_t* __restrict__ offs, int B,
                   const int32_t* __restrict__ cpre, const double* __restrict__ P, const int32_t* __restrict__ nn,
                   const double* __restrict__ d2, const IcpPair* __restrict__ pst, double* __restrict__ part) {
    __shared__ double s_warp[RED_WARPS];
    const int g = blockIdx.x, t = threadIdx.x;
    if (g >= cpre[B]) return;
    const int b = regtr_cloud_of(cpre, B, g);
    if (pst[b].done) return;
    const int i0 = offs[b] + (g - cpre[b]) * CHUNK, i1 = min(i0 + CHUNK, offs[b + 1]);
    double k = 0.0, sd = 0.0, sp[3] = {0.0, 0.0, 0.0}, sq[3] = {0.0, 0.0, 0.0};
    for (int i = i0 + t; i < i1; i += RED_THREADS) {
        const int j = nn[i];
        if (j < 0) continue;
        k += 1.0;
        sd += d2[i];
        for (int a = 0; a < 3; ++a) { sp[a] += P[3 * i + a]; sq[a] += xyz[3 * j + a]; }
    }
    double out[PART_POINT];
    out[0] = block_sum(k, s_warp);
    out[1] = block_sum(sd, s_warp);
    for (int a = 0; a < 3; ++a) out[2 + a] = block_sum(sp[a], s_warp);
    for (int a = 0; a < 3; ++a) out[5 + a] = block_sum(sq[a], s_warp);
    const double inv = out[0] > 0.0 ? 1.0 / out[0] : 0.0;
    double mp[3], mq[3];
    for (int a = 0; a < 3; ++a) { mp[a] = out[2 + a] * inv; mq[a] = out[5 + a] * inv; }
    double C[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = i0 + t; i < i1; i += RED_THREADS) {
        const int j = nn[i];
        if (j < 0) continue;
        double dp[3], dq[3];
        for (int a = 0; a < 3; ++a) { dp[a] = P[3 * i + a] - mp[a]; dq[a] = xyz[3 * j + a] - mq[a]; }
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) C[3 * r + c] += dq[r] * dp[c];
    }
    for (int e = 0; e < 9; ++e) out[8 + e] = block_sum(C[e], s_warp);
    if (t != 0) return;
    double* o = part + (size_t)PART_POINT * g;
    o[0] = out[0]; o[1] = out[1];
    for (int a = 0; a < 3; ++a) { o[2 + a] = mp[a]; o[5 + a] = mq[a]; }
    for (int e = 0; e < 9; ++e) o[8 + e] = out[8 + e];
}

// One thread per pair.  The pair's chunks are combined in chunk order, giving k, fitness = k / n and inlier
// RMSE = sqrt(sum d2 / k) of the current correspondences.  After round 0 the stop test |d fitness| < rel_fitness and
// |d rmse| < rel_rmse ends the pair; so does round max_iter.  Otherwise the update, composed as T = update . T.
//
// Point-to-point: the chunks' means and co-moments are combined by the pairwise update, then Umeyama without scaling:
// Sigma = C / k, SVD, reflection fix when det(U) det(V) < 0, R = U S V^T, t = mean_q - R mean_p (the identity with
// k = 0).
//
// Point-to-plane family (PLANE): the chunks' J^T J and J^T r are summed, and J^T J x = -J^T r is solved by LDL^T in
// float64 (Open3D's SolveLinearSystemPSD: the identity when k = 0 or |det J^T J| < 1e-6 or det is not finite); the
// update is R = Rz(x2) Ry(x1) Rx(x0), t = (x3, x4, x5) (TransformVector6dToMatrix4d).
template <bool PLANE>
__global__ void __launch_bounds__(UPD_THREADS)
k_icp_update(const int32_t* __restrict__ offs, int B, const int32_t* __restrict__ cpre,
             const double* __restrict__ part, IcpPair* __restrict__ pst, int round, int max_iter, double rel_fitness,
             double rel_rmse, double* __restrict__ pose_out, double* __restrict__ result) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B || pst[b].done) return;
    IcpPair s = pst[b];
    double K = 0.0, sd = 0.0, H[21], v[6], mp[3] = {0.0, 0.0, 0.0}, mq[3] = {0.0, 0.0, 0.0}, C[9];
    if constexpr (PLANE) {
        for (int e = 0; e < 21; ++e) H[e] = 0.0;
        for (int e = 0; e < 6; ++e) v[e] = 0.0;
        for (int g = cpre[b]; g < cpre[b + 1]; ++g) {
            const double* o = part + (size_t)PART_PLANE * g;
            if (!(o[0] > 0.0)) continue;
            K += o[0];
            sd += o[1];
            for (int e = 0; e < 21; ++e) H[e] += o[2 + e];
            for (int e = 0; e < 6; ++e) v[e] += o[23 + e];
        }
    } else {
        for (int e = 0; e < 9; ++e) C[e] = 0.0;
        for (int g = cpre[b]; g < cpre[b + 1]; ++g) {
            const double* o = part + (size_t)PART_POINT * g;
            const double k = o[0];
            if (!(k > 0.0)) continue;
            const double n = K + k, f = k / n, w = K * f;
            double dp[3], dq[3];
            for (int a = 0; a < 3; ++a) {
                dp[a] = o[2 + a] - mp[a]; dq[a] = o[5 + a] - mq[a];
                mp[a] += dp[a] * f; mq[a] += dq[a] * f;
            }
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) C[3 * r + c] += o[8 + 3 * r + c] + dq[r] * dp[c] * w;
            sd += o[1];
            K = n;
        }
    }
    const int n_src = offs[b + 1] - offs[b];
    const double fit = n_src > 0 ? K / (double)n_src : 0.0;
    const double rmse = K > 0.0 ? sqrt(sd / K) : 0.0;
    const bool conv = round > 0 && fabs(s.fit - fit) < rel_fitness && fabs(s.rmse - rmse) < rel_rmse;
    s.fit = fit; s.rmse = rmse; s.k = (int)K;
    if (conv || round >= max_iter) {
        s.done = 1;
    } else {
        double R[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}}, t[3] = {0.0, 0.0, 0.0};
        if constexpr (PLANE) {
            double x[6];
            if (K > 0.0 && solve6_ldlt(H, v, x)) rigid_from_vec6(x, R, t);
        } else if (K > 0.0) {
            const double inv = 1.0 / K;
            double A[3][3], U[3][3], S[3], V[3][3];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) A[r][c] = C[3 * r + c] * inv;
            svd3_jacobi(A, U, S, V);
            const double d = det3(U) * det3(V) < 0.0 ? -1.0 : 1.0;
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 3; ++c) R[r][c] = U[r][0] * V[c][0] + U[r][1] * V[c][1] + d * U[r][2] * V[c][2];
            for (int r = 0; r < 3; ++r) t[r] = mq[r] - (R[r][0] * mp[0] + R[r][1] * mp[1] + R[r][2] * mp[2]);
        }
        double* T = pose_out + 12 * b;
        double N[12];
        for (int r = 0; r < 3; ++r) {
            for (int c = 0; c < 3; ++c) s.upd[4 * r + c] = R[r][c];
            s.upd[4 * r + 3] = t[r];
        }
        for (int r = 0; r < 3; ++r)                       // update . T as rigid transforms
            for (int c = 0; c < 4; ++c) {
                const double u = __dadd_rn(__dadd_rn(__dmul_rn(R[r][0], T[c]), __dmul_rn(R[r][1], T[4 + c])),
                                           __dmul_rn(R[r][2], T[8 + c]));
                N[4 * r + c] = c == 3 ? __dadd_rn(u, t[r]) : u;
            }
        for (int e = 0; e < 12; ++e) T[e] = N[e];
        s.iters = round + 1;
    }
    pst[b] = s;
    double* o = result + 4 * b;
    o[0] = fit; o[1] = rmse; o[2] = K; o[3] = (double)s.iters;
}

struct IcpWs {
    double *P, *d2, *part, *snrm;
    float* x32;
    int32_t *tofs, *cpre, *nn;
    IcpPair* pst;
    void *grid, *gws;
    size_t gws_bytes, total;
};

int n_chunks_cap(int n_cap, int B) { return regtr_cdiv(n_cap, CHUNK) + B; }

IcpWs carve_icp(void* ws, int n_cap, int B) {
    IcpWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t n = (size_t)n_cap;
    w.P = (double*)take(sizeof(double) * 3 * n);
    w.d2 = (double*)take(sizeof(double) * n);
    w.part = (double*)take(sizeof(double) * PART_PLANE * (size_t)n_chunks_cap(n_cap, B));   // the larger record
    w.x32 = (float*)take(sizeof(float) * 3 * n);
    w.tofs = (int32_t*)take(sizeof(int32_t) * ((size_t)B + 1));
    w.cpre = (int32_t*)take(sizeof(int32_t) * ((size_t)B + 1));
    w.nn = (int32_t*)take(sizeof(int32_t) * n);
    w.pst = (IcpPair*)take(sizeof(IcpPair) * (size_t)B);
    w.grid = take(regtr_cellgrid_bytes(n_cap));
    w.gws_bytes = regtr_cellgrid_ws_bytes(n_cap);
    w.gws = take(w.gws_bytes);
    w.snrm = (double*)take(sizeof(double) * 3 * n);                  // generalized ICP's moved source normals
    w.total = off;
    return w;
}

}  // namespace

extern "C" {

size_t regtr_icp_ws_bytes(int n_cap, int B) {
    return carve_icp(nullptr, n_cap > 0 ? n_cap : 1, B > 0 ? B : 1).total;
}
size_t regtr_icp_state_bytes(int n_cap) { return regtr_cellgrid_state_bytes(n_cap > 0 ? n_cap : 1); }

int regtr_icp(const double* xyz, const int32_t* offs, int B, int n_cap, const double* init, double max_dist,
              float cell, int max_iter, double rel_fitness, double rel_rmse, const double* tgt_normals,
              const double* src_normals, const regtr_icp_options* opt, double* pose_out, double* result,
              uint32_t* status, void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    if (!offs || !init || !pose_out || !result || !status || !ws || !state || B <= 0 || 2 * B > 32767 || n_cap < 0 ||
        !(max_dist > 0.0) || !((double)cell > max_dist) || max_iter < 0 || !(rel_fitness >= 0.0) ||
        !(rel_rmse >= 0.0) || (n_cap > 0 && !xyz))
        return REGTR_ERR_ARG;
    const regtr_icp_options o = opt ? *opt : regtr_icp_options{REGTR_ICP_LOSS_L2, 1.0, 1e-3};
    const bool colored = o.src_colors != nullptr;
    if (o.loss < REGTR_ICP_LOSS_L2 || o.loss > REGTR_ICP_LOSS_TUKEY || !(o.epsilon > 0.0 && o.epsilon <= 1.0) ||
        (o.loss != REGTR_ICP_LOSS_L2 && !(o.loss_k > 0.0 && o.loss_k <= DBL_MAX)) ||
        ((src_normals || o.loss != REGTR_ICP_LOSS_L2 || colored) && !tgt_normals) ||
        (colored ? (src_normals || !o.tgt_colors || !o.tgt_color_gradients ||
                    !(o.lambda_geometric >= 0.0 && o.lambda_geometric <= 1.0))
                 : (o.tgt_colors || o.tgt_color_gradients)))
        return REGTR_ERR_ARG;
    const auto reduce_plane = src_normals ? k_icp_reduce_plane<PLANE_GICP>
                            : o.loss != REGTR_ICP_LOSS_L2 ? k_icp_reduce_plane<PLANE_ROBUST>
                                                          : k_icp_reduce_plane<PLANE_L2>;
    const int nc = n_cap > 0 ? n_cap : 1;      // offs[2B] = 0 without points: every kernel then reads no xyz
    IcpWs w = carve_icp(ws, nc, B);
    if (ws_bytes < w.total || state_bytes < regtr_icp_state_bytes(n_cap)) return REGTR_ERR_WORKSPACE;
    const double bound = regtr_overlap_coord_bound(max_dist, cell);
    const int T = 256;
    k_icp_init<<<regtr_cdiv((nc > B + 1 ? nc : B + 1), T), T, 0, st>>>(xyz, offs, B, nc, init, bound, w.P, w.x32,
                                                                       w.tofs, w.cpre, w.pst, pose_out, result,
                                                                       status);
    REGTR_CHECK_LAUNCH();
    const int rc = regtr_cellgrid_build(w.x32, w.tofs, B, nc, cell, w.grid, nullptr, status, w.gws, w.gws_bytes,
                                        state, state_bytes, stream_);
    if (rc != REGTR_OK) return rc;
    const int nn_blocks = regtr_cdiv(nc, NN_WARPS) < 8 * REGTR_NUM_SMS ? regtr_cdiv(nc, NN_WARPS) : 8 * REGTR_NUM_SMS;
    const CellSlot* table = grid_table(w.grid, (size_t)nc);
    const float4* sxyzi = grid_sxyzi(w.grid);
    const int log2t = cell_table_log2(nc);
    for (int round = 0; round <= max_iter; ++round) {
        k_icp_nn<<<nn_blocks, NN_WARPS * 32, 0, st>>>(xyz, offs, B, nc, w.P, w.pst, round > 0, table, log2t, sxyzi,
                                                      cell, max_dist * max_dist, bound, w.nn, w.d2, status);
        REGTR_CHECK_LAUNCH();
        const int red_blocks = n_chunks_cap(nc, B), upd_blocks = regtr_cdiv(B, UPD_THREADS);
        if (colored) {
            regtr_icp_reduce_colored(red_blocks, st, xyz, offs, B, w.cpre, w.P, w.nn, w.d2, w.pst, w.part, tgt_normals,
                                     o.loss, o.loss_k, o.src_colors, o.tgt_colors, o.tgt_color_gradients,
                                     sqrt(o.lambda_geometric), sqrt(1.0 - o.lambda_geometric));
            REGTR_CHECK_LAUNCH();
            k_icp_update<true><<<upd_blocks, UPD_THREADS, 0, st>>>(offs, B, w.cpre, w.part, w.pst, round, max_iter,
                                                                   rel_fitness, rel_rmse, pose_out, result);
        } else if (tgt_normals) {
            reduce_plane<<<red_blocks, RED_THREADS, 0, st>>>(xyz, offs, B, w.cpre, w.P, w.nn, w.d2, w.pst, w.part,
                                                             tgt_normals, src_normals, w.snrm, init, round, o.loss,
                                                             o.loss_k, 1.0 - o.epsilon, IcpColor{});
            REGTR_CHECK_LAUNCH();
            k_icp_update<true><<<upd_blocks, UPD_THREADS, 0, st>>>(offs, B, w.cpre, w.part, w.pst, round, max_iter,
                                                                   rel_fitness, rel_rmse, pose_out, result);
        } else {
            k_icp_reduce_point<<<red_blocks, RED_THREADS, 0, st>>>(xyz, offs, B, w.cpre, w.P, w.nn, w.d2, w.pst,
                                                                   w.part);
            REGTR_CHECK_LAUNCH();
            k_icp_update<false><<<upd_blocks, UPD_THREADS, 0, st>>>(offs, B, w.cpre, w.part, w.pst, round, max_iter,
                                                                    rel_fitness, rel_rmse, pose_out, result);
        }
        REGTR_CHECK_LAUNCH();
    }
    return REGTR_OK;
}

}  // extern "C"
