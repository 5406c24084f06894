/*
 * regtr_b200 -- C ABI of the H100-native (sm_90a) RegTR correspondence-prediction hot path.
 *
 * The reference (yewzijian/RegTR) has no FFI layer: its boundary for this path is
 * the nn.Module surface (src/models/regtr.py:104-235) over ATen ops plus two
 * un-vendored CUDA libraries.  Each entry point below replaces one reference
 * operation (file:line cited per function; paths relative to /root/reference/src).
 * INTEGRATION.md shows the ctypes binding a maintainer adds on the reference side.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless marked "host";
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, no
 *     call synchronises, allocates or frees (workspaces are caller-owned and sized
 *     by the matching *_ws_bytes function);
 *   - stacked clouds are described by int32 prefix offsets `offs[n_clouds + 1]`
 *     (device memory) so that data-dependent level sizes never cross to the host
 *     inside the pyramid; `*_cap` arguments are host-known capacities (upper
 *     bounds of offs[n_clouds]) used only to size grids and buffers;
 *   - return value: 0 on success, REGTR_ERR_* (<0) on a rejected argument,
 *     -(1000 + cudaError_t) when a launch fails.  Data-dependent failures
 *     (coordinates outside the +-32767-cell key range) are reported through the
 *     device status word, see regtr_status_*.
 */
#ifndef REGTR_B200_H_
#define REGTR_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define REGTR_OK 0
#define REGTR_ERR_ARG (-1)        /* null pointer / negative size / unsupported shape */
#define REGTR_ERR_WORKSPACE (-2)  /* workspace too small */
#define REGTR_ERR_UNSUPPORTED (-3)

#define REGTR_STATUS_KEY_RANGE 1u /* a voxel / cell coordinate left the 16-bit key range */
#define REGTR_STATUS_CAPACITY 2u  /* a capacity-bounded output (sub-sampled level) overflowed; results truncated */
#define REGTR_STATUS_GRID 4u      /* voxel bounding box beyond the dense-grid budget: redo with regtr_grid_subsample_sorted */
#define REGTR_STATUS_RANGE 8u     /* overlap search: |coordinate| beyond regtr_overlap_coord_bound; neighbours may be missed */

int regtr_version(void);                 /* ABI version, currently 1 */
const char* regtr_build_info(void);      /* host pointer: arch + compile flags string */

/* ---- pyramid pre-processing ------------------------------------------------------- */

/* Voxel-grid barycentre sub-sampling.
 * Replaces batch_grid_subsampling_kpconv_gpu (models/backbone_kpconv/kpconv.py:213-240,
 * i.e. MinkowskiEngine 0.5.4 SparseTensor(UNWEIGHTED_AVERAGE)) with the deterministic
 * rules of DESIGN.md: voxel = floor(p / dl) (IEEE fp32 division), output ordered by
 * ascending (cloud, vx, vy, vz), barycentre = fp32 sum in ascending input index / count.
 * xyz (n_cap,3) f32; offs (n_clouds+1) i32; out_xyz (out_cap,3); out_offs (n_clouds+1).
 * out_cap may be smaller than n_cap (static-shape pipelines): on overflow the output is
 * truncated memory-safely and REGTR_STATUS_CAPACITY is raised.
 * status: device uint32 word, OR-ed with REGTR_STATUS_* on data-dependent errors. */
size_t regtr_grid_subsample_ws_bytes(int n_cap, int n_clouds);
size_t regtr_grid_subsample_state_bytes(int n_cap);
int regtr_grid_subsample(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float dl,
                         float* out_xyz, int out_cap, int32_t* out_offs, uint32_t* status,
                         void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream);
/* regtr_grid_subsample sorts by COUNTING over a dense voxel grid spanning each cloud's bounding box (hand-written
 * kernels only; budget: 16 cells per point of capacity, at least 2^18).  `state`: regtr_grid_subsample_state_bytes
 * bytes, ZERO before the first call and owned by this op between calls (every call leaves it zero).  A box beyond
 * the budget raises REGTR_STATUS_GRID; regtr_grid_subsample_sorted (stable library radix sort of (key, index)
 * pairs, any extent) gives the same result for such inputs. */
size_t regtr_grid_subsample_sorted_ws_bytes(int n_cap);
int regtr_grid_subsample_sorted(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float dl,
                                float* out_xyz, int out_cap, int32_t* out_offs, uint32_t* status,
                                void* ws, size_t ws_bytes, void* stream);

/* Float64 voxel down-sampling with attributes (Open3D's PointCloud::VoxelDownSample), the multi-scale ICP pyramid's
 * per-level step.  xyz (n_cap,3) float64 with offs (C+1) i32, offs[0] = 0, 1 <= C <= 32767; voxel V > 0 and finite
 * (else REGTR_ERR_ARG).  attr (n_cap,3) float64, nullable (colours); out_attr is then required.
 *   Per cloud: lo = the exact per-axis minimum of its points, origin = lo - 0.5 V, and point p falls in voxel
 *   v = floor((p - origin) / V) per axis, the subtraction and the division each rounded to nearest (no contraction).
 *   One output row per occupied voxel, rows in ascending (cloud, vx, vy, vz); a row is the float64 sum of its member
 *   points in ascending point index divided by their count, and out_attr's row the same of their attributes.
 * out_xyz / out_attr (n_cap,3) float64 capacity buffers (always sufficient); out_offs (C+1) i32 the rows of each
 * cloud (an empty cloud has none).  An index above 65535 on any axis, or a non-finite coordinate, raises
 * REGTR_STATUS_KEY_RANGE (Open3D allows up to INT_MAX); the rows are then not meaningful.  5 launches plus the
 * library radix sort and scan whatever C and the data; no value atomics and no host synchronisation: a cloud's rows
 * are the same bits alone or in a stack.  ws: regtr_voxel_down_sample_ws_bytes(n_cap, C). */
size_t regtr_voxel_down_sample_ws_bytes(int n_cap, int C);
int regtr_voxel_down_sample(const double* xyz, const double* attr, const int32_t* offs, int C, int n_cap,
                            double voxel, double* out_xyz, double* out_attr, int32_t* out_offs, uint32_t* status,
                            void* ws, size_t ws_bytes, void* stream);

/* Outlier removal (Open3D's PointCloud::RemoveStatisticalOutliers and RemoveRadiusOutliers) for C stacked clouds:
 * xyz (n_cap,3) float64 with offs (C+1) i32, offs[0] = 0, 1 <= C <= 32767.  Each filter writes per-point keep flags
 * (n_cap) i32, 1 = kept, rows >= offs[C] untouched; regtr_select_points then gathers the kept rows.  No value atomics
 * and no host synchronisation: a cloud's results are the same bits alone or in a stack, and the launch counts
 * depend on neither the data nor C.  ws: regtr_outlier_ws_bytes(n_cap, C); state: regtr_outlier_state_bytes(n_cap),
 * ZERO before the first call, every call leaves it zero.
 *
 * k nearest neighbours (both in the statistical filter): the neighbours of point i are the k points of i's own cloud
 * with the smallest (d^2, index) keys, d^2 = (dx dx + dy dy) + dz dz in float64, each operation rounded on its own
 * (no contraction), i itself included, ties to the lower index, all m = min(k, n) points of a cloud of n < k points;
 * no radius.  The result is defined by this rule, not by the search (one warp per point walks rings of cells of a
 * cell list of size `cell` around the point and sweeps its whole cloud past 4 rings), so it is the same bits for any
 * cell size.
 *
 * regtr_statistical_outlier, RemoveStatisticalOutliers(nb_neighbors, std_ratio) restated:
 *   1. for each point i, its k = nb_neighbors nearest neighbours by the rule above, m = min(k, n) of them;
 *   2. avg_i = (sum of sqrt(d^2)) / m, the sum sequential in ascending (d^2, index) order (nanoflann's result order);
 *   3. valid = the number of points with m > 0, i.e. n for a non-empty cloud;
 *   4. cloud_mean = (sum of avg_i over the points with avg_i > 0) / valid: points with avg 0 are left out of the sum
 *      but counted in valid (Open3D's rule, kept);
 *   5. sq_sum = sum over the points with avg_i > 0 of (avg_i - cloud_mean)^2;
 *   6. std_dev = sqrt(sq_sum / (valid - 1)), threshold = cloud_mean + std_ratio * std_dev;
 *   7. point i is kept iff avg_i > 0 and avg_i < threshold.
 *   So exact duplicates of k or more points are dropped, a one-point cloud keeps nothing (valid - 1 = 0 makes the
 *   threshold NaN) and an empty cloud yields nothing (its statistics are NaN).
 *   Summation order (the departure from Open3D, which sums 4. and 5. sequentially over the cloud): each sum runs over
 *   chunks of 256 points anchored at the cloud's first point, past-the-end entries 0 and excluded points 0; a chunk
 *   is reduced by the fixed tree e[i] = e[i] + e[i + h] for h = 128, 64, ..., 1, and the chunk partials are added in
 *   ascending chunk order starting from 0.  Every operation is rounded on its own, including (avg_i - cloud_mean)^2,
 *   std_ratio * std_dev and its addition.  The result then differs from Open3D's sequential sums in the last bits of
 *   cloud_mean and std_dev at most.
 *   nb_neighbors in 1..64, std_ratio > 0 and finite, cell > 0 and finite (else REGTR_ERR_ARG).  avg (n_cap) f64;
 *   stats (C,3) f64: (cloud_mean, std_dev, threshold) per cloud.  A |coordinate| above 1e30 (the cell list holds fp32
 *   copies) or not finite raises REGTR_STATUS_RANGE; a cell index of floor(fp32(p) / cell) outside +-32766 raises
 *   REGTR_STATUS_KEY_RANGE, so a caller picks cell >= max |coordinate| / 32000 (ops.knn_cell does).  1 + 4 + 7
 *   launches.
 *
 * regtr_radius_outlier, RemoveRadiusOutliers(nb_points, radius): counts[i] = the number of points of i's own cloud
 *   with d^2 (as above) strictly below radius^2, i included (the library's radius rule and nanoflann's strict test),
 *   always the full count; point i is kept iff counts[i] >= nb_points.  nb_points >= 1, radius > 0 and finite, cell
 *   = radius * (1 + 1e-3) rounded to fp32 (ops.overlap_cell), cell > radius (else REGTR_ERR_ARG).  counts (n_cap)
 *   i32.  A |coordinate| beyond regtr_overlap_coord_bound(radius, cell), or not finite, raises REGTR_STATUS_RANGE,
 *   as in regtr_estimate_normals.  1 + 4 + 1 launches.
 *
 * regtr_select_points: the stable compaction of either filter's output.  keep (n_cap) i32, nonzero = kept; attr
 * (n_cap,3) f64 nullable (colours), out_attr then required.  Kept rows go to out_xyz / out_attr (n_cap,3) in their
 * original order; out_index (n_cap) i32, nullable, receives the index of each kept row inside its own cloud;
 * out_offs (C+1) i32 the kept rows of each cloud.  3 launches (flags, the single-pass scan, the scatter).
 * ws: regtr_select_points_ws_bytes(n_cap); state: regtr_select_points_state_bytes(n_cap), ZERO before the first call,
 * every call leaves it zero. */
size_t regtr_outlier_ws_bytes(int n_cap, int C);
size_t regtr_outlier_state_bytes(int n_cap);
int regtr_statistical_outlier(const double* xyz, const int32_t* offs, int C, int n_cap, int nb_neighbors,
                              double std_ratio, float cell, double* avg, int32_t* keep, double* stats,
                              uint32_t* status, void* ws, size_t ws_bytes, void* state, size_t state_bytes,
                              void* stream);
int regtr_radius_outlier(const double* xyz, const int32_t* offs, int C, int n_cap, int nb_points, double radius,
                         float cell, int32_t* counts, int32_t* keep, uint32_t* status, void* ws, size_t ws_bytes,
                         void* state, size_t state_bytes, void* stream);
size_t regtr_select_points_ws_bytes(int n_cap);
size_t regtr_select_points_state_bytes(int n_cap);
int regtr_select_points(const double* xyz, const double* attr, const int32_t* keep, const int32_t* offs, int C,
                        int n_cap, double* out_xyz, double* out_attr, int32_t* out_index, int32_t* out_offs, void* ws,
                        size_t ws_bytes, void* state, size_t state_bytes, void* stream);

/* Uniform cell list over a stacked point set (search structure for regtr_ball_query).
 * `grid` is an opaque caller-owned buffer of regtr_cellgrid_bytes(n_cap) bytes; `order`
 * (n_cap) i32, optional, receives the cell-sorted permutation of the points (a spatially
 * coherent processing order for queries drawn from the same set). */
size_t regtr_cellgrid_bytes(int n_cap);
size_t regtr_cellgrid_ws_bytes(int n_cap);
size_t regtr_cellgrid_state_bytes(int n_cap);   /* ZERO before the first call; every call leaves it zero */
int regtr_cellgrid_build(const float* xyz, const int32_t* offs, int n_clouds, int n_cap, float cell,
                         void* grid, int32_t* order, uint32_t* status,
                         void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream);

/* Fixed-radius neighbour search, first K supports in ascending index order.
 * Replaces batch_neighbors_kpconv_gpu (kpconv.py:261-288: pytorch3d 0.6.0 packed_to_padded +
 * ball_query + re-packing): per query keep support j (ascending) while
 * ((dx*dx + dy*dy) + dz*dz) < r*r in fp32 without FMA contraction; pad with the total
 * support count.  `s_grid` must have been built over (s, s_offs) with capacity s_cap and
 * cell >= radius.
 * q_order (optional, nq_cap): processing order of the queries (a permutation of [0,nq_cap)).
 * out_idx32 / out_idx64 (nq_cap,K): either may be NULL; rows of capacity padding
 * (>= q_offs[n_clouds]) are filled with the shadow index. */
int regtr_ball_query(const float* q, const int32_t* q_offs, const int32_t* q_order,
                     const float* s, const int32_t* s_offs, const void* s_grid,
                     int n_clouds, int nq_cap, int s_cap, int K, float radius,
                     int32_t* out_idx32, int64_t* out_idx64, void* stream);

/* ---- KPConv encoder --------------------------------------------------------------- */

/* Rigid KPConv, linear influence, 'sum' aggregation.
 * Replaces KPConv.forward (models/backbone_kpconv/kpconv_blocks.py:269-414):
 *   out[n] = (1/max(1,#{k: sum_c x[idx[n,k]] > 0})) * sum_p (sum_k h(n,k,p) x[idx[n,k]]) W[p]
 *   h = max(0, 1 - |s[idx[n,k]] - q[n] - kp[p]| / extent); idx == Ns is the shadow neighbour.
 * q (Nq,3) s (Ns,3) idx (Nq,K) i32, x (Ns,Cin) f32, W (P,Cin,Cout) f32, kp (P,3), out (Nq,Cout).
 * P must be 15.  Cin in {1..16} or 32/64/128/256.
 * nq_dev / ns_dev (optional, device int32): actual query / support counts when Nq / Ns are
 * capacities (static-shape pipelines); rows >= *nq_dev are padding (zeroed up to the next multiple of
 * 128, untouched beyond -- consumers work in 128-row tiles); the shadow index is *ns_dev.
 * ws: regtr_kpconv_fwd_ws_bytes(Nq, Ns, Cin, Cout) bytes (aggregated features + row flags + the split
 * transposed weights + the GEMM's workspace; the contraction runs on regtr_gemm_tf32x3 -- no library GEMM).
 * regtr_kpconv_ws_bytes(Nq, Ns, Cin) is the part regtr_kpconv_aggregate alone needs (wf + row flags). */
size_t regtr_kpconv_ws_bytes(int Nq, int Ns, int Cin);
size_t regtr_kpconv_fwd_ws_bytes(int Nq, int Ns, int Cin, int Cout);
int regtr_kpconv_fwd(const float* q, const float* s, const int32_t* idx, const float* x,
                     const float* W, const float* kp, int Nq, int Ns, const int32_t* nq_dev,
                     const int32_t* ns_dev, int K, int Cin, int Cout,
                     float extent, float* out, void* ws, size_t ws_bytes, void* stream);

/* Gather + influence + aggregation stage alone: wf (Nq, 15*Cin), already divided by the
 * neighbour count.  (The "neighbour gather" kernel of the north star.)  rowflag_ws (Ns bytes):
 * flags[r] = (sum_c x[r,c] > 0); computed here unless flags_ready != 0 (then it must already hold
 * them, e.g. from regtr_instnorm_act's rowflag_out). */
int regtr_kpconv_aggregate(const float* q, const float* s, const int32_t* idx, const float* x,
                           const float* kp, int Nq, int Ns, const int32_t* nq_dev, const int32_t* ns_dev,
                           int K, int Cin, float extent,
                           float* wf, uint8_t* rowflag_ws, int flags_ready, void* stream);

/* max over the K gathered rows with a zero shadow row.  Replaces max_pool
 * (kpconv_blocks.py:127-143).  x (Ns,C), idx (Nq,K) i32 -> out (Nq,C). */
int regtr_max_pool(const float* x, const int32_t* idx, int Nq, int Ns, const int32_t* ns_dev, int K, int C,
                   float* out, void* stream);

/* Per-cloud InstanceNorm1d(affine=False, eps) over the points of each cloud, optional
 * residual add, optional LeakyReLU.  Replaces BatchNormBlock.forward + nn.LeakyReLU
 * (kpconv_blocks.py:497-519, 546-561, 646, 741):  out = act(norm(x) + res).
 * x (n,C); offs (n_clouds+1) i32 device; n_cap >= offs[n_clouds]; res optional (n,C);
 * slope < 0 disables the activation.  In-place (out == x) is allowed.  Rows in [offs[n_clouds], n_cap)
 * are padding: zeroed up to the next multiple of 128, untouched beyond.
 * rowflag_out (optional, n_cap bytes, C/4 a power of two <= 32): flags[r] = (sum_c out[r,c] > 0),
 * the neighbour-count predicate of the KPConv that consumes `out`.
 * counters (optional): regtr_instnorm_counter_bytes(n_clouds, C) bytes of int32, ZERO before the first call
 * and owned by this op between calls (every call leaves them zero); with them the statistics are
 * finalised by the last statistics block (one launch fewer), without them by a separate kernel. */
size_t regtr_instnorm_ws_bytes(int n_cap, int n_clouds, int C);
size_t regtr_instnorm_counter_bytes(int n_clouds, int C);
int regtr_instnorm_act(const float* x, const int32_t* offs, int n_clouds, int n_cap, int C, float eps,
                       const float* res, float slope, float* out, uint8_t* rowflag_out,
                       void* ws, size_t ws_bytes, int32_t* counters, void* stream);

/* The apply pass alone: out = act((x - mean) * rstd + res) with stats (n_clouds, C, 2) = (mean, rstd) produced
 * elsewhere -- by regtr_gemm_tf32x3_instats, which accumulates them in the GEMM epilogue so that the Linear ->
 * InstanceNorm pairs of the KPConv blocks (kpconv_blocks.py:546-561, 401-406 + 497-519) never re-read their
 * output for the statistics.  rowflag_out as in regtr_instnorm_act. */
int regtr_instnorm_apply(const float* x, const int32_t* offs, int n_clouds, int n_cap, int C, const float* stats,
                         const float* res, float slope, float* out, uint8_t* rowflag_out, void* stream);

/* ---- dense layers ---------------------------------------------------------------- */

/* The two TF32 halves of x (low 13 mantissa bits zero), each rounded to nearest, ties to even:
 *   hi = tf32_rne(x),  lo = tf32_rne(x - hi)   (x - hi is exact in fp32).
 * hi + lo is not x in general: lo drops the low bits of x - hi, so |x - (hi + lo)| <= half a TF32 ulp of
 * x - hi, about 2^-22 |x|.  Used to pre-split weight matrices for regtr_gemm_tf32x3. */
int regtr_split_tf32(const float* x, long long n, float* hi, float* lo, void* stream);

/* fp32-accurate GEMM on the Hopper tensor cores (wgmma, 3xTF32):
 *   C[M,N] = act(A[M,K] @ B[N,K]^T + bias[N] + R[M,N]),  B given pre-split as B_hi / B_lo.
 * Replaces nn.Linear (kpconv_blocks.py:546, regtr.py:36/145, transformers.py:95-101,
 * regtr.py:404-411) and the KPConv weight contraction (kpconv_blocks.py:401-406).
 * Row-major fp32; lda/ldb multiples of 4 and 16-byte aligned bases (TMA); bias / R optional;
 * C, R and bias may be any views (the epilogue uses 16-byte accesses only where their bases and
 * pitches allow); m_dev (optional device int32): actual row count when M is a capacity; relu != 0
 * applies ReLU.  ws: regtr_gemm_ws_bytes(M,N,K) bytes, 16-byte aligned (deterministic split-K
 * planes for skinny long-K shapes). */
size_t regtr_gemm_ws_bytes(int M, int N, int K);
int regtr_gemm_tf32x3(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                      float* C, int ldc, const float* bias, const float* R, int ldr,
                      int M, int N, int K, const int32_t* m_dev, int relu,
                      void* ws, size_t ws_bytes, void* stream);

/* C = A @ B^T (no bias / residual / activation) PLUS the per-cloud InstanceNorm statistics of C:
 * stats (n_clouds, N, 2) = (mean, 1/sqrt(biased var + eps)) over the rows [offs[c], offs[c+1]) of each column,
 * without a second pass over C: every epilogue warp stores the column sums / sums of squares of its 32 rows
 * (fixed shuffle tree) to `part`, and a small second kernel adds the partials of each cloud in a fixed order
 * (fp64) -- no atomics, run-to-run bit-identical.  N % 32 == 0.
 * part: regtr_instnorm_part_bytes(M, N) bytes of scratch (8-byte aligned; contents irrelevant on entry). */
size_t regtr_instnorm_part_bytes(int M, int N);
int regtr_gemm_tf32x3_instats(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                              float* C, int ldc, int M, int N, int K, const int32_t* m_dev,
                              const int32_t* offs, int n_clouds, float eps, void* part, float* stats,
                              void* ws, size_t ws_bytes, void* stream);

/* ---- transformer ------------------------------------------------------------------ */

/* 3-D sine position embedding.  Replaces PositionEmbeddingCoordsSine.forward
 * (models/transformer/position_embedding.py:29-50).  dim_t (n_freq) f32 is the reference's
 * `temperature ** (2*(i//2)/n_freq)` table; out (n, d_model), zero padded. */
int regtr_pos_embed_sine(const float* xyz, int n, const float* dim_t, int n_freq, int d_model,
                         float scale, float* out, void* stream);

/* The six dropouts of TransformerCrossEncoderLayer.forward_pre in train mode (transformers.py:85-110, 183-244), all
 * with the same p: site 1 the self-attention probabilities, 2 the self-attention output (dropout1), 3 the cross-
 * attention probabilities, 4 the cross-attention output (dropout2), 5 relu(linear1) (dropout), 6 the linear2 output
 * (dropout3).  Masks are regenerated, never stored: the keep decision of (row, column) of a site is a Philox4x32-10
 * draw keyed by (seed, step, global cloud 2 (pair_base + b) + side, layer, site, head, row, column) -- independent of
 * the batch size, packing, rank and launch configuration (counter layout: regtr_b200/csrc/philox.cuh).  Row: token
 * within the (query) cloud; column: key index within the key cloud (sites 1, 3) or feature index (head 0).  Local
 * cloud c of the (src x B, tgt x B) stack is pair c % B, side c / B (B = n_pairs).  A value is dropped when its 16-bit
 * draw is below `threshold` = round(p 65536); kept values are multiplied by `scale` = fp32(1 / (1 - p)).  Limits:
 * 2 (pair_base + n_pairs) <= 2^20, layer < 16, head < 16, clouds shorter than 2^16 tokens.  Passed by host pointer. */
typedef struct regtr_dropout_args {
    unsigned long long seed, step;
    int32_t pair_base;      /* global index of the batch's first pair */
    int32_t layer;          /* 0..15 */
    int32_t site;           /* 1..6 */
    uint32_t threshold;     /* round(p * 65536), <= 65536 */
    float scale;            /* fp32(1 / (1 - p)) */
    int32_t n_pairs;        /* B */
} regtr_dropout_args;

/* LayerNorm over the last dim with optional position add:  y = LN(x)*g + b ;
 * y_pos = y + pos.  Replaces nn.LayerNorm + with_pos_embed (transformers.py:117-119,
 * 194-196, 213-215, 232).  Any of y / y_pos may be NULL.  n_dev (optional, device): the real row count
 * when n is a capacity; rows beyond it are left untouched.
 * drop (optional): the residual dropout fused into the LayerNorm that follows it (sites 2, 4, 6):  x' = x + m scale z
 * (z: the out-projection / linear2 output), x_out = x', and the LayerNorm is that of x'.  offs (2B + 1, device): cloud
 * offsets of the packed rows (n = offs[2B]).  z, offs, x_out and drop are all NULL or all set, and n_dev is NULL with
 * drop; x_out must not alias x or z. */
int regtr_layernorm_pos(const float* x, const float* z, const float* gamma, const float* beta, const float* pos, int n,
                        const int32_t* n_dev, const int32_t* offs, int E, float eps, float* y, float* y_pos,
                        float* x_out, const regtr_dropout_args* drop, void* stream);

/* Device-side attention problem table for a (src x B, tgt x B) token stack with cloud offsets
 * offs (2B+1): plan (6, 2B+1) i32 rows = q_start, q_len, cross k_start, cross k_len (the cross
 * partner of src_b is tgt_b and vice versa; regtr.py:156-166's key-padding masks made explicit), then the
 * exclusive prefix of the number of 64-query / 128-query tiles per problem (entry 2B = total): the `tile_base`
 * tables of the attention kernels below. */
int regtr_attention_plan(const int32_t* offs, int B, int32_t* plan, void* stream);

/* Variable-length multi-head attention core, fp32:  O = softmax(Q K^T * scale) V per head.
 * Replaces the attention core of nn.MultiheadAttention as called at
 * transformers.py:197-226 (key-padding masks become explicit (start,len) ranges).
 * Problem i attends queries rows [q_start[i], q_start[i]+q_len[i]) of Q to key rows
 * [k_start[i], k_start[i]+k_len[i]) of K/V.  Q/K/V/O are row-major with leading
 * dimensions ldq/ldk/ldv/ldo (floats); head h uses columns [h*head_dim, (h+1)*head_dim).
 * head_dim must be 32; ldo must be even (REGTR_ERR_UNSUPPORTED otherwise).  max_q_len: host upper bound of
 * q_len[].
 * tile_base (optional, n_problems + 1, device): exclusive prefix of ceil(q_len / 64) with the total last; the launch
 * then covers max_tiles (a host bound of that total, e.g. capacity / 64 + n_problems) linear tiles instead of
 * ceil(max_q_len / 64) tiles per problem -- capacity-shaped launches know the per-problem lengths on the device only.
 * lse (optional, training): also writes lse [n_tokens, n_heads] = log2(sum_k exp2(s_qk)) of the base-2 scores
 * s = (q * scale * log2 e) . k -- what regtr_mha_varlen_bwd recomputes the softmax from (-inf for a query whose key
 * range is empty); O is the same, bit for bit.
 * drop (optional, training; needs lse): the attention-probability dropout (site 1 or 3; the problem tables of
 * regtr_attention_plan, problem c = query cloud c, n_heads <= 16): O = scale * sum_k m_qk P_qk V_k, the mask applied to
 * the probabilities in registers before the P V product; lse is that of the undropped probabilities.
 * tile_base together with lse or drop is REGTR_ERR_UNSUPPORTED. */
int regtr_mha_varlen_fwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                         float* O, int ldo, float* lse, const int32_t* q_start, const int32_t* q_len,
                         const int32_t* k_start, const int32_t* k_len, int n_problems, int max_q_len,
                         const int32_t* tile_base, int max_tiles, int n_heads, int head_dim, float scale,
                         const regtr_dropout_args* drop, void* stream);

/* CorrespondenceDecoder.simple_attention (regtr.py:316-351, the `direct_regress_coor: False` branch):
 * single-head attention whose values are the key coordinates,
 *   out[l, q] = sum_k softmax_k(Qp[l, q] . Kp[l, k] * scale) xyz[k]          (fp32)
 * for all n_layers decoder inputs at once.  Qp/Kp: (n_layers * n_rows, D) row-major with leading
 * dimension ld -- the q_proj / k_proj outputs; row l*n_rows + t belongs to token t of layer l.
 * xyz (n_rows, 3): token coordinates; out (n_layers * n_rows, 3).  Problem tables as for
 * regtr_mha_varlen_fwd (token ranges, shared by all layers).  D % 4 == 0. */
int regtr_corr_decode_fwd(const float* Qp, const float* Kp, int ld, const float* xyz, float* out,
                          const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                          const int32_t* k_len, int n_problems, int max_q_len, int n_layers, int n_rows,
                          int D, float scale, void* stream);

/* Tensor-core attention core (bf16 operands, fp32 register accumulation, fp32 softmax): the "fast"
 * precision mode of the same nn.MultiheadAttention core (transformers.py:197-226), head_dim 32.
 * Inputs are produced by regtr_gemm_tf32x3_qkv_bf16 (the packed in-projection with a bf16
 * epilogue): QK [n_tokens, 2E] bf16 row-major (q | k), Vt [E, ld_vt] bf16 (v transposed, columns
 * >= n_tokens zero).  O [n_tokens, E] fp32.  Problem tables as for regtr_mha_varlen_fwd. */
int regtr_gemm_tf32x3_qkv_bf16(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                               const float* bias, int M, int N, int K, int split, void* qk_out, int ld_qk,
                               void* vt_out, int ld_vt, const int32_t* m_dev, void* stream);
int regtr_mha_bf16_tc_fwd(const void* QK, int ld_qk, const void* Vt, int ld_vt, int n_tokens, float* O,
                          int ldo, const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                          const int32_t* k_len, int n_problems, int max_q_len, int n_heads, int head_dim,
                          float scale, void* stream);

/* fp32-accurate attention core on the Hopper tensor cores (the parity mode of the same nn.MultiheadAttention core,
 * transformers.py:197-226): S = Q K^T and O = P V as 3xTF32 wgmma with TMA-fed operands, P kept in registers,
 * fp32 softmax.  Inputs from regtr_gemm_tf32x3_qkv_split, the packed in-projection (N = 3E: q | k | v) whose
 * epilogue writes every value as its two TF32 halves: qk4 [n_tokens, 4E] fp32 = [Q_hi | Q_lo | K_hi | K_lo] with q
 * pre-multiplied by qscale (pass softmax_scale * log2(e)); vt2 [2E, ld_vt] fp32 = v transposed, hi rows then lo rows
 * (columns >= the real token count must be finite, e.g. zero; the epilogue leaves them untouched).  Both halves are
 * rounded to nearest with ties away from zero: hi = rna(x), lo = rna(x - hi).  The in-projection's bias is read
 * 16 bytes at a time: its base must be 16-byte aligned.  O [n_tokens, E] fp32.  head_dim must be 32.
 * Problem tables as for regtr_mha_varlen_fwd. */
int regtr_gemm_tf32x3_qkv_split(const float* A, int lda, const float* B_hi, const float* B_lo, int ldb,
                                const float* bias, int M, int N, int K, int E, float qscale, float* qk4, int ld4,
                                float* vt2, int ld_vt, const int32_t* m_dev, void* stream);
int regtr_mha_tf32_tc_fwd(const float* qk4, int ld4, const float* vt2, int ld_vt, int n_tokens, float* O, int ldo,
                          const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                          const int32_t* k_len, int n_problems, int max_q_len, const int32_t* tile_base,
                          int max_tiles, int n_heads, int head_dim, void* stream);
/* (tile_base / max_tiles as for regtr_mha_varlen_fwd, with 128-query tiles.) */

/* Head-averaged attention probabilities (analysis; TransformerCrossEncoder.get_attentions):
 *   P[q, k] = (1/H) sum_h softmax_k(Q_h[q] . K_h[k] * scale)
 * for every (query range, key range) problem of the tables above -- nn.MultiheadAttention's weights with
 * average_attn_weights=True.  Q / K are row-major with leading dims ldq / ldk (column slices allowed, 16-byte
 * aligned, ld % 4 == 0).  Problem p writes its q_len[p] x k_len[p] block at P + p_offset[p] with row pitch p_pitch[p]
 * (>= k_len[p]), so one launch fills e.g. a padded (B, Lq_max, Lk_max) layout directly; every other element of P is
 * left untouched (the caller zero-fills padding), and a problem with an empty query or key range writes nothing.
 * Scores on 3xTF32 mma.sync (fp32-accurate); base-2 softmax from a per-(row, head) maximum and sum computed by the
 * kernel itself in a first sweep (no workspace).  No atomics: reruns are bit-identical.  head_dim 32, n_heads <= 16. */
int regtr_mha_probs_avg(const float* Q, int ldq, const float* K, int ldk, float* P, const int64_t* p_offset,
                        const int32_t* p_pitch, const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                        const int32_t* k_len, int n_problems, int max_q_len, int n_heads, int head_dim, float scale,
                        void* stream);

/* ---- backward (training) ---------------------------------------------------------- */

/* Backward of the attention core over the same problem tables: given O and lse from regtr_mha_varlen_fwd and
 * dO, writes dQ (rows of every query range), dK and dV (rows of every key range; 0 for a key range whose problem
 * has no queries).  Each key row must belong to the key range of exactly one problem (true of the self and of the
 * cross table of regtr_attention_plan); dQ / dK / dV may be column slices of one packed [n_rows, 3E] buffer.
 * n_rows: rows of Q / lse (an upper bound of every query row index + 1); max_k_len: host bound of k_len[].
 * Deterministic (no atomics): one pass owns the query rows, a second one the key rows.  The softmax is renormalised
 * from the backward's own recomputed scores, and delta = sum_k P dP is formed from them too, so O is checked for
 * NULL but its values are not read.
 * drop (optional): the forward's dropout key; dP_qk becomes g_qk = m_qk scale (dO_q . V_k), delta = sum_k P g,
 * dV_k = sum_q P_qk m_qk scale dO_q.
 * ws: regtr_mha_varlen_bwd_ws_bytes(n_rows, n_heads) bytes (delta and 1 / sum_k exp2(s - lse) per query and head). */
size_t regtr_mha_varlen_bwd_ws_bytes(int n_rows, int n_heads);
int regtr_mha_varlen_bwd(const float* Q, int ldq, const float* K, int ldk, const float* V, int ldv,
                         const float* O, int ldo, const float* dO, int lddo, const float* lse,
                         float* dQ, int lddq, float* dK, int lddk, float* dV, int lddv,
                         const int32_t* q_start, const int32_t* q_len, const int32_t* k_start,
                         const int32_t* k_len, int n_problems, int n_rows, int max_q_len, int max_k_len,
                         int n_heads, int head_dim, float scale, const regtr_dropout_args* drop, void* ws,
                         size_t ws_bytes, void* stream);

/* Backward of regtr_layernorm_pos: dy and dy_pos (either may be NULL; they add) are the gradients of y and y_pos,
 * dres (optional) a gradient of x arriving through a residual connection, added to dx.  Mean and rstd are
 * recomputed from x.  dgamma / dbeta (E) from per-block column partials summed in a fixed order.  E % 32 == 0,
 * E <= 256.  ws: regtr_layernorm_bwd_ws_bytes(n, E) bytes.  n = 0 writes dgamma = dbeta = 0 (x and dx may be NULL).
 * drop (optional; offs, dz and drop are all NULL or all set): the backward of the residual dropout, with x = the
 * forward's x_out: dx is the gradient of x' (dres included), plus dz = dx m scale. */
size_t regtr_layernorm_bwd_ws_bytes(int n, int E);
int regtr_layernorm_bwd(const float* x, const float* gamma, const float* dy, const float* dy_pos, const float* dres,
                        int n, const int32_t* offs, int E, float eps, float* dx, float* dz, float* dgamma, float* dbeta,
                        const regtr_dropout_args* drop, void* ws, size_t ws_bytes, void* stream);

/* ReLU backward: out = dh * scale where h > 0, else 0 (n elements; out may alias dh).  h is the ReLU's output and
 * scale = 1, or, with the feed-forward dropout, h is the dropped ReLU output of regtr_dropout_rows (positive exactly
 * where the ReLU passed and the mask kept) and scale the dropout's. */
int regtr_relu_bwd(const float* dh, const float* h, long long n, float scale, float* out, void* stream);

/* Weight gradient of a dense layer Y = X W^T + b:  dW[N,K] = dY^T X,  db[N] = sum_rows dY (db optional),
 * 3xTF32 on regtr_gemm_tf32x3 (the reduction over the M rows uses its deterministic split-K).  X (M,K) and
 * dY (M,N) row-major with leading dimensions ldx / ldy; M = 0 writes dW = 0 and db = 0 (X, dY and their
 * leading dimensions are then not read: an empty tensor's data pointer is null and its strides arbitrary).  ws: regtr_linear_wgrad_ws_bytes(M, N, K) bytes,
 * 256-byte aligned (transposed, TF32-split operands and the product). */
size_t regtr_linear_wgrad_ws_bytes(int M, int N, int K);
int regtr_linear_wgrad(const float* X, int ldx, const float* dY, int ldy, int M, int N, int K,
                       float* dW, float* db, void* ws, size_t ws_bytes, void* stream);

/* ---- backward of the KPConv encoder (training with the encoder) --------------------- */

/* Transpose of a neighbour list: the incoming edges of every support row as CSR.  idx (Nq,K) i32 with shadow
 * index Ns (any entry outside [0, Ns) is a shadow slot and is left out) -> row_start (Ns+1) i32 and
 * edges (Nq*K capacity) i32 = edge ids q*K + k, ascending inside each row (rows in support order).  The edge
 * order does not depend on scheduling.  The gather-scatter of the KPConv (kpconv_blocks.py:388-391) and of
 * max_pool (kpconv_blocks.py:138-141) read their lists through it in the backward, so that every support row
 * sums its gradient contributions itself: no floating-point atomics.
 * ws: regtr_neighbor_csr_ws_bytes(Ns) bytes (per-row counters, contents irrelevant on entry). */
size_t regtr_neighbor_csr_ws_bytes(int Ns);
int regtr_neighbor_csr(const int32_t* idx, int Nq, int K, int Ns, int32_t* row_start, int32_t* edges,
                       void* ws, size_t ws_bytes, void* stream);

/* Input gradient of the rigid KPConv (kpconv_blocks.py:388-412) given dwf = dOut W^T (Nq, 15*Cin), the
 * gradient of the aggregated features (compute it with regtr_gemm_tf32x3 and W viewed as (15*Cin, Cout)):
 *   dx[s] = sum_{(q,k): idx[q,k]=s} (1/cnt_q) sum_p h(q,k,p) dwf[q,p,:]
 * h is recomputed exactly as regtr_kpconv_aggregate computes it; cnt_q = max(1, #valid neighbours whose
 * feature row sums to > 0) carries no gradient.  flags (Ns bytes, optional): the forward's row flags (as
 * regtr_kpconv_aggregate's rowflag_ws); NULL recomputes them from x.  row_start / edges: regtr_neighbor_csr of
 * idx.  dx (Ns, Cin), every row written (0 for supports no query references).  Cin <= 256, K <= 128.
 * ws: regtr_kpconv_bwd_input_ws_bytes(Nq, K, Cin) bytes: one (1/cnt_q) h^T dwf[q] row per edge, then summed
 * per support in CSR order (2 * nnz * Cin * 4 bytes of traffic). */
size_t regtr_kpconv_bwd_input_ws_bytes(int Nq, int K, int Cin);
int regtr_kpconv_bwd_input(const float* q, const float* s, const int32_t* idx, const float* x,
                           const uint8_t* flags, const float* kp, int Nq, int Ns, int K, int Cin, float extent,
                           const float* dwf, const int32_t* row_start, const int32_t* edges, float* dx,
                           void* ws, size_t ws_bytes, void* stream);

/* Backward of regtr_max_pool (kpconv_blocks.py:127-143): the gradient of out[q,c] goes to the first maximal
 * entry in neighbour order (torch.max(dim)'s tie rule); the zero shadow row is a candidate and gradient routed
 * to it is dropped.  x (Ns,C) the pooled input, idx (Nq,K) i32, dout (Nq,C), row_start / edges its
 * regtr_neighbor_csr -> dx (Ns,C), every row written.  K <= 255.
 * ws: regtr_max_pool_bwd_ws_bytes(Nq, C) bytes (the arg-max slot per output entry). */
size_t regtr_max_pool_bwd_ws_bytes(int Nq, int C);
int regtr_max_pool_bwd(const float* x, const int32_t* idx, int Nq, int Ns, int K, int C, const float* dout,
                       const int32_t* row_start, const int32_t* edges, float* dx, void* ws, size_t ws_bytes,
                       void* stream);

/* Backward of regtr_instnorm_act / regtr_instnorm_apply, out = act(norm(x) + res)
 * (kpconv_blocks.py:497-519, 546-561, 646, 741).  g (n,C) the gradient of out; out is read for the LeakyReLU
 * mask (g' = g * (out > 0 ? 1 : slope)) and may be NULL when slope < 0 (no activation).
 *   dx = rstd (g' - mean_cloud(g') - xh mean_cloud(g' xh)),  xh = (x - mean) rstd;   dres = g' (optional).
 * mean / rstd are recomputed from x in fp64 (fixed 128-row chunks inside each cloud, added in order), so the
 * result does not depend on which forward entry produced the statistics.  A one-point cloud gets dx = 0; rows
 * beyond offs[n_clouds] get zeros.  C % 4 == 0.  ws: regtr_instnorm_bwd_ws_bytes(n, n_clouds, C) bytes. */
size_t regtr_instnorm_bwd_ws_bytes(int n, int n_clouds, int C);
int regtr_instnorm_bwd(const float* g, const float* x, const float* out, const int32_t* offs, int n_clouds,
                       int n, int C, float eps, float slope, float* dx, float* dres,
                       void* ws, size_t ws_bytes, void* stream);

/* ---- optimizer step (training) ---------------------------------------------------- */

/* Multi-tensor launches over a DEVICE table of descriptors: the number of launches does not depend on the number of
 * tensors.  Each tensor is cut into chunks of REGTR_OPTIM_CHUNK elements; `first` is the exclusive prefix of the
 * chunk counts ceil(n / REGTR_OPTIM_CHUNK) over the table (the table is sorted by it) and n_chunks the total.
 * Tensors are contiguous fp32; entries with n == 0 own no chunk. */
#define REGTR_OPTIM_CHUNK 8192

typedef struct {
    float* g;             /* gradient (scaled in place by regtr_grad_scale) */
    long long n;          /* elements */
    long long first;      /* first chunk */
} regtr_grad_ref;

/* Total 2-norm of all gradients, as torch.nn.utils.clip_grad_norm_(max_norm, norm_type=2) computes it:
 * out[0] = sqrt(sum g^2) (sum of squares in fp64: fixed per-chunk order, then the chunk partials in a fixed order;
 * no atomics), out[1] = min(1, max_norm / (out[0] + 1e-6)) in fp32 with torch's roundings (NaN propagates).
 * Two launches.  ws: regtr_grad_norm_ws_bytes(n_chunks) bytes (one fp64 partial per chunk). */
size_t regtr_grad_norm_ws_bytes(int n_chunks);
int regtr_grad_norm(const regtr_grad_ref* table, int n_tensors, int n_chunks, float max_norm, float* out,
                    void* ws, size_t ws_bytes, void* stream);
/* g *= *coef for every gradient of the table (coef: device fp32, e.g. out + 1 of regtr_grad_norm).  One launch. */
int regtr_grad_scale(const regtr_grad_ref* table, int n_tensors, int n_chunks, const float* coef, void* stream);

/* One tensor of a flat fp32 bucket (data-parallel gradient exchange: one collective for every gradient). */
typedef struct {
    float* t;             /* fp32 tensor; NULL: packs zeros, unpacks nothing */
    long long n;          /* elements */
    long long first;      /* first chunk (REGTR_OPTIM_CHUNK elements) */
    long long off;        /* first element in the bucket */
} regtr_bucket_ref;

/* unpack == 0: bucket[off, off + n) = t for every entry; unpack != 0: t = bucket[off, off + n).  One launch, plain
 * copies (a pack and an unpack round-trip bit for bit). */
int regtr_bucket_copy(const regtr_bucket_ref* table, int n_tensors, int n_chunks, float* bucket, int unpack,
                      void* stream);

#define REGTR_ADAM_FRESH 1u      /* state just created: exp_avg / exp_avg_sq are read as zero (and written) */
#define REGTR_ADAM_COUPLED 2u    /* Adam weight decay: g += wd * p */
#define REGTR_ADAM_DECOUPLED 4u  /* AdamW weight decay: p *= decay */

/* One tensor of an Adam / AdamW step.  The host scalars are torch's for this tensor's step t (already incremented),
 * rounded to fp32 as torch's kernels round them:  decay = 1 - lr * wd,  b1w = 1 - beta1 (the lerp weight),
 * one_m_b2 = 1 - beta2,  rcp_bc2_sqrt = 1 / fp32(sqrt(1 - beta2^t)) (fp32 division),
 * neg_step_size = -lr / (1 - beta1^t)  (the bias corrections in double). */
typedef struct {
    float* p;             /* parameter */
    const float* g;       /* gradient */
    float* m;             /* exp_avg */
    float* v;             /* exp_avg_sq */
    long long n;
    long long first;      /* first chunk */
    float decay, wd, b1w, b2, one_m_b2, rcp_bc2_sqrt, neg_step_size, eps;
    uint32_t flags;       /* REGTR_ADAM_* */
    uint32_t pad;
} regtr_adam_tensor;

/* Replaces torch.optim.Adam / AdamW.step (foreach=False arithmetic, torch 2.11 _single_tensor_adam):
 *   p = p * decay (decoupled) or g = g + wd * p (coupled);  m = lerp(m, g, b1w);  v = v * b2 + one_m_b2 * g * g;
 *   p = p - step_size * m / (sqrt(v) / sqrt(1 - beta2^t) + eps).   One launch. */
int regtr_adam_step(const regtr_adam_tensor* table, int n_tensors, int n_chunks, void* stream);

/* A 2-D view of a weight whose TF32 halves are cached: out[a, b] = src[a * s0 + b * s1] for a < rows, b < cols,
 * hi / lo contiguous (rows, cols).  `first`: exclusive prefix of the 32 x 32 tile counts
 * ceil(rows / 32) * ceil(cols / 32) over the table. */
typedef struct {
    const float* src;
    float* hi;
    float* lo;
    long long s0, s1;     /* element strides of the view (a transposed weight has s0 == 1) */
    long long first;      /* first tile */
    int rows, cols;
} regtr_split_view;

/* Re-split updated weights into their existing (hi, lo) buffers with the rounding of regtr_split_tf32 (the result
 * is bit-identical to a fresh split of the view); transposed views go through a shared-memory tile so that reads
 * and writes coalesce.  One launch. */
int regtr_split_refresh(const regtr_split_view* table, int n_views, int n_tiles, void* stream);

/* ---- pose ------------------------------------------------------------------------- */

/* Weighted Kabsch.  Replaces compute_rigid_transform (utils/se3_torch.py:108-154):
 * problem i uses rows [offs[i], offs[i+1]) of a,b (n,3) and w (n); T (n_problems,3,4),
 * T*a = b.  One warp per problem, fp64 accumulation, one-sided Jacobi 3x3 SVD. */
int regtr_kabsch_fwd(const float* a, const float* b, const float* w, const int32_t* offs,
                     int n_problems, float* T, void* stream);

/* Fused correspondence assembly + sigmoid + Kabsch for RegTR.forward (models/regtr.py:185-203):
 * kp (n,3) coarse key points, packed src clouds first then tgt clouds; corr (L,n,3) predicted
 * correspondences; logit (L,n) overlap logits; offs (2B+1) i32 cloud offsets.
 * pose (L,B,3,4): for pair b, a=[src_kp ; tgt_corr], b=[src_corr ; tgt_kp],
 * w=[sigmoid(src_logit) ; sigmoid(tgt_logit)]. */
int regtr_pose_from_corr(const float* kp, const float* corr, const float* logit,
                         const int32_t* offs, int n, int B, int L, float* pose, void* stream);

/* ---- training data (3DMatch) ------------------------------------------------------ */

/* Overlap ground truth of B pairs.  Replaces compute_overlap (utils/pointcloud.py:8-65) on the aligned clouds
 * (data_loaders/threedmatch.py:79-86).  xyz (n_cap,3) float64 stacked src_0..src_{B-1}, tgt_0..tgt_{B-1} with
 * offs (2B+1) i32; pose (B,3,4) float64 maps source to target.  The sources are moved by the pose in float64
 * (((r0 x + r1 y) + r2 z) + t, no contraction); one cell list over the fp32 copy of all 2B clouds (cell `cell`, use
 * radius * (1 + 1e-3)); per point the NEAREST point of the partner cloud with float64 squared distance strictly below
 * radius^2, equal distances to the lowest index: nn (n_cap) i32 = its index inside the partner cloud, or -1.
 * A |coordinate| of an aligned point beyond regtr_overlap_coord_bound(radius, cell) raises REGTR_STATUS_RANGE: past
 * it the fp32 cell assignment could hide a neighbour.  ws / state: the *_bytes functions below (state ZERO before the
 * first call; every call leaves it zero). */
double regtr_overlap_coord_bound(double radius, float cell);
size_t regtr_overlap_ws_bytes(int n_cap);
size_t regtr_overlap_state_bytes(int n_cap);
int regtr_overlap_nn(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose, double radius,
                     float cell, int32_t* nn, uint32_t* status, void* ws, size_t ws_bytes, void* state,
                     size_t state_bytes, void* stream);

/* Fitness and inlier RMSE of B registered pairs (the definitions of Open3D's evaluate_registration, which the
 * reference's demo.py leaves to a viewer), from the matches of regtr_overlap_nn: xyz, offs, pose and radius as given
 * to it, nn its output.  out (B,4) float64 per pair = (fitness_src, rmse_src, fitness_tgt, rmse_tgt):
 *   fitness = |{i : nn_i >= 0}| / n (0 for an empty cloud), rmse = sqrt(sum d_i^2 / n_inliers) (0 without inliers),
 * d_i^2 the float64 squared distance of regtr_overlap_nn (the source moved by ((r0 x + r1 y) + r2 z) + t, no
 * contraction), so every summed distance is one that passed "strictly below radius".  Sums in a fixed order, one CTA
 * per (pair, direction): the result is bit-reproducible.  A match index outside the partner cloud, or a distance not
 * below radius, is not counted and raises REGTR_STATUS_INPUT.  n_cap >= offs[2B].  One launch. */
int regtr_registration_fit(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose,
                           double radius, const int32_t* nn, double* out, uint32_t* status, void* stream);

/* Information matrices of B registered pairs (Open3D's get_information_matrix_from_point_clouds on this library's
 * match rule), from the matches of regtr_overlap_nn: xyz, offs, pose and radius as given to it, nn its output.
 * out (B,6,6) float64 per pair = sum over the source points i with nn_i >= 0, in ascending i, of G^T G with q the
 * matched TARGET point in the target's own frame and
 *   G = [[0, q_z, -q_y, 1, 0, 0], [-q_z, 0, q_x, 0, 1, 0], [q_y, -q_x, 0, 0, 0, 1]],
 * so out[5][5] is the match count.  Its 21 unique entries are ten float64 sums (y^2 + z^2, x^2 + z^2, x^2 + y^2, xy,
 * xz, yz, x, y, z, 1), each in a fixed order, one CTA per pair: the result is bit-reproducible and independent of
 * the batch.  A match index outside the target, or a distance not below radius, is not counted and raises
 * REGTR_STATUS_INPUT, as in regtr_registration_fit.  n_cap >= offs[2B].  One launch. */
int regtr_registration_information(const double* xyz, const int32_t* offs, int B, int n_cap, const double* pose,
                                   double radius, const int32_t* nn, double* out, uint32_t* status, void* stream);

/* C stacked clouds moved by one pose each: xyz (n_cap,3) float64 with offs (C+1) i32, pose (C,3,4) float64;
 * out (n_cap,3) fp32 = fp32(((r0 x + r1 y) + r2 z) + t) in float64, no contraction; rows >= offs[C] untouched.
 * C <= 32767.  One launch. */
int regtr_transform_clouds(const double* xyz, const int32_t* offs, int C, int n_cap, const double* pose, float* out,
                           void* stream);

/* ICP of B pairs (Open3D's registration_icp with TransformationEstimationPointToPoint, no scaling, or with
 * TransformationEstimationPointToPlane, or registration_generalized_icp, and ICPConvergenceCriteria(rel_fitness,
 * rel_rmse, max_iter)).
 * xyz (n_cap,3) float64 stacked src_0..src_{B-1},
 * tgt_0..tgt_{B-1} with offs (2B+1) i32; init (B,3,4) float64 source -> target.  Per pair: P = init . source
 * (((r0 x + r1 y) + r2 z) + t, no contraction), T = init; correspondences are regtr_overlap_nn's (the nearest target
 * point with float64 d^2 strictly below max_dist^2, ties to the lowest index), fitness = k / n_src,
 * rmse = sqrt(sum d^2 / k) (both 0 without inliers).  Then up to max_iter times: the Umeyama update without scaling
 * on the correspondences (the identity when k = 0), T = update . T, P moved by the update in place, re-match; stop
 * when |d fitness| < rel_fitness and |d rmse| < rel_rmse.  pose_out (B,3,4) float64 = T; result (B,4) float64 =
 * (fitness, rmse, k, iterations run).  One cell list over the targets (cell `cell`, use max_dist * (1 + 1e-3)), then
 * 3 launches per round for max_iter + 1 rounds whatever B and convergence; no host synchronisation; sums in a fixed
 * order, so the result is bit-reproducible and independent of the batch.  A coordinate of a moved source or of a
 * target beyond regtr_overlap_coord_bound(max_dist, cell), or not finite, raises REGTR_STATUS_RANGE.  ws / state:
 * the *_bytes functions below (state ZERO before the first call; every call leaves it zero).
 * tgt_normals NULL: point-to-point, as above.  Non-NULL: (offs[2B] - offs[B], 3) float64, row j - offs[B] the normal of
 * target row j (regtr_estimate_normals); point-to-plane with the same correspondences, fitness, RMSE (point distances)
 * and stop test.  Per correspondence (p moved source, q target, n its normal) r = (p - q) . n, J = [p x n ; n]; J^T J
 * (21 unique entries) and J^T r summed per chunk in the fixed order; per pair J^T J x = -J^T r solved by LDL^T in
 * float64; the update is the identity when k = 0, |det J^T J| < 1e-6 or det is not finite (Open3D's
 * SolveLinearSystemPSD), else R = Rz(x2) Ry(x1) Rx(x0), t = (x3, x4, x5) (TransformVector6dToMatrix4d).  A zero
 * normal drops its correspondence out of the update, not out of k.  Same launches as point-to-point.
 * src_normals NULL with opt NULL: the above, unchanged.  src_normals non-NULL (needs tgt_normals): generalized ICP
 * (Open3D's registration_generalized_icp with TransformationEstimationForGeneralizedICP(epsilon, kernel)),
 * (offs[B], 3) float64 stacked like the sources; every round they are rotated with the sources (first by init, then
 * by each update) in a workspace copy.  Per correspondence (a moved source normal, b target normal, c = 1 - epsilon)
 * M = (I - c a a^T) + (I - c b b^T) (a zero normal gives I), (U, S, V) its float64 Jacobi SVD,
 * W = V diag(1 / sqrt(S)) V^T; the rows w_i of W give r_i = w_i . (p - q), J_i = [p x w_i ; w_i], each into J^T J and
 * J^T r with weight loss(r_i); a correspondence whose M has an eigenvalue that is not > 0 or not finite leaves the
 * update, not k.  opt (host memory, nullable: L2 and epsilon 1e-3): a loss other than REGTR_ICP_LOSS_L2 weights every
 * residual row of point-to-plane (r = (p - q) . n) or generalized ICP by Open3D's RobustKernel::Weight(r):
 * huber 1 if |r| <= k else k / |r|; cauchy 1 / (1 + (r/k)^2); gm k / (k + r^2)^2; tukey (1 - (r/k)^2)^2 if |r| <= k
 * else 0.  REGTR_ERR_ARG: src_normals without tgt_normals, a loss other than L2 without tgt_normals, an unknown loss,
 * loss_k not > 0 or not finite with a loss other than L2, epsilon outside (0, 1].  Same launches in every mode.
 * opt->src_colors non-NULL (needs tgt_normals, opt->tgt_colors and opt->tgt_color_gradients, and no src_normals):
 * colored ICP (Open3D's registration_colored_icp with TransformationEstimationForColoredICP(lambda_geometric, kernel)),
 * with the correspondences, fitness, RMSE (point distances), stop test and update of point-to-plane.  src_colors
 * (offs[B], 3) and tgt_colors (offs[2B] - offs[B], 3) float64 rgb stacked like their clouds, intensity
 * ((r + g) + b) / 3; tgt_color_gradients (offs[2B] - offs[B], 3) float64 (regtr_color_gradients).  Per correspondence
 * (p moved source, q target, n its normal, d its gradient, l = lambda_geometric), two residual rows, each into J^T J
 * and J^T r with weight loss(r) of its own r: geometric r = sqrt(l) (p - q) . n, J = [p x sqrt(l) n ; sqrt(l) n];
 * photometric, with p' = p - ((p - q) . n) n, is0 = d . (p' - q) + it_q and m = (d . n) n - d (= -(I - n n^T) d):
 * r = sqrt(1 - l) (is_p - is0), J = [p x sqrt(1 - l) m ; sqrt(1 - l) m].  A zero target normal drops its
 * correspondence out of the update, not out of k.  REGTR_ERR_ARG: lambda_geometric outside [0, 1], tgt_colors or
 * tgt_color_gradients without src_colors, or src_colors without tgt_normals, tgt_colors or tgt_color_gradients, or
 * with src_normals. */
#define REGTR_ICP_LOSS_L2 0
#define REGTR_ICP_LOSS_HUBER 1
#define REGTR_ICP_LOSS_CAUCHY 2
#define REGTR_ICP_LOSS_GM 3
#define REGTR_ICP_LOSS_TUKEY 4
typedef struct {
    int loss;                                /* REGTR_ICP_LOSS_* [L2] */
    double loss_k;                           /* the loss's parameter k, > 0 (ignored by L2) */
    double epsilon;                          /* generalized ICP's covariance epsilon, 0 < epsilon <= 1 [1e-3] */
    const double* src_colors;                /* colored ICP's device inputs (see above) [NULL: not colored] */
    const double* tgt_colors;
    const double* tgt_color_gradients;
    double lambda_geometric;                 /* colored ICP's weight of the geometric residual, 0 <= l <= 1 */
} regtr_icp_options;

size_t regtr_icp_ws_bytes(int n_cap, int B);
size_t regtr_icp_state_bytes(int n_cap);
int regtr_icp(const double* xyz, const int32_t* offs, int B, int n_cap, const double* init, double max_dist,
              float cell, int max_iter, double rel_fitness, double rel_rmse, const double* tgt_normals,
              const double* src_normals, const regtr_icp_options* opt, double* pose_out, double* result,
              uint32_t* status, void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream);

/* Normals of C stacked clouds (Open3D's estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) followed by
 * orient_normals_towards_camera_location() at the origin, with this library's tie and boundary rules).
 * xyz (n_cap,3) float64 with offs (C+1) i32, offs[0] = 0, C <= 32767; cell = radius * (1 + 1e-3) rounded to fp32
 * (ops.overlap_cell); 1 <= max_nn <= 64 (else REGTR_ERR_ARG).  normals (n_cap,3) float64, rows >= offs[C] untouched.
 *   Neighbours of point i: the points of i's own cloud with float64 d^2 = (dx dx + dy dy) + dz dz (no contraction)
 *   strictly below radius^2, i itself included (d^2 = 0); the max_nn smallest by (d^2, index), ties to the lower index.
 *   Found through one cell list over the fp32 copy (27-cell stencil), without a capacity limit or truncation.
 *   Covariance: over the neighbours in ascending (d^2, index) order, the mean first, then the centred sum of outer
 *   products / count, float64 sums in that fixed order.
 *   Normal: the unit eigenvector of the covariance's smallest eigenvalue (the right singular vector of the smallest
 *   singular value of a float64 one-sided Jacobi SVD), negated when ((nx px + ny py) + nz pz) > 0 (towards the origin).
 *   Fewer than 3 neighbours: (0,0,0), so that the point drops out of point-to-plane ICP (Open3D returns an arbitrary
 *   axis there).
 * counts (n_cap) i32, nullable: the number of neighbours used per point.  A |coordinate| beyond
 * regtr_overlap_coord_bound(radius, cell), or not finite, raises REGTR_STATUS_RANGE.  1 + 4 + 1 launches whatever C;
 * no value atomics, no host synchronisation: the result is bit-identical whether a cloud is passed alone or in a stack.
 * ws / state: the *_bytes functions below (state ZERO before the first call; every call leaves it zero). */
size_t regtr_estimate_normals_ws_bytes(int n_cap);
size_t regtr_estimate_normals_state_bytes(int n_cap);
int regtr_estimate_normals(const double* xyz, const int32_t* offs, int C, int n_cap, double radius, float cell,
                           int max_nn, double* normals, int32_t* counts, uint32_t* status, void* ws, size_t ws_bytes,
                           void* state, size_t state_bytes, void* stream);

/* Intensity gradients of C stacked coloured clouds for colored ICP (Open3D's InitializePointCloudForColoredICP with
 * KDTreeSearchParamHybrid(radius, max_nn), with this library's tie and order rules).  xyz / normals / colors
 * (n_cap,3) float64 with offs (C+1) i32, offs[0] = 0, C <= 32767 (normals from regtr_estimate_normals, a zero normal
 * allowed; colors rgb); cell = radius * (1 + 1e-3) rounded to fp32 (ops.overlap_cell); 1 <= max_nn <= 64 (else
 * REGTR_ERR_ARG).  grad (n_cap,3) float64, rows >= offs[C] untouched.
 *   Neighbours of point p: regtr_estimate_normals' rule (own cloud, d^2 strictly below radius^2, p included, the
 *   max_nn smallest by (d^2, index)), nn of them.  Intensity it = ((r + g) + b) / 3.
 *   Gradient 0 when nn < 4 or the normal n of p is zero.  Otherwise rows of A and b: for every entry i >= 1 in
 *   ascending (d^2, index) order, with q_i - ((q_i - p) . n) n = v_i, the row v_i - p and b = it_i - it_p; then the row
 *   (nn - 1) n with b = 0.  (A^T A) x = A^T b, both summed row by row in that order in float64, solved by LDL^T; the
 *   gradient is x, or 0 when |det A^T A| < 1e-6 or det is not finite (Open3D's SolveLinearSystemPSD, as regtr_icp).
 * A |coordinate| beyond regtr_overlap_coord_bound(radius, cell), or not finite, raises REGTR_STATUS_RANGE.
 * 1 + 4 + 1 launches whatever C; no value atomics, no host synchronisation: the result is bit-identical whether a cloud
 * is passed alone or in a stack.  ws / state: the *_bytes functions below (state ZERO before the first call; every
 * call leaves it zero). */
size_t regtr_color_gradients_ws_bytes(int n_cap);
size_t regtr_color_gradients_state_bytes(int n_cap);
int regtr_color_gradients(const double* xyz, const double* normals, const double* colors, const int32_t* offs, int C,
                          int n_cap, double radius, float cell, int max_nn, double* grad, uint32_t* status, void* ws,
                          size_t ws_bytes, void* state, size_t state_bytes, void* stream);

/* FPFH features of C stacked clouds (Open3D's ComputeFPFHFeature(KDTreeSearchParamHybrid(radius, max_nn)), with this
 * library's tie and order rules).  xyz / normals (n_cap,3) float64 with offs (C+1) i32, offs[0] = 0, C <= 32767 (the
 * normals of regtr_estimate_normals; a zero normal is allowed); cell = radius * (1 + 1e-3) rounded to fp32
 * (ops.overlap_cell); 1 <= max_nn <= REGTR_FPFH_MAX_NN (else REGTR_ERR_ARG).  feature (n_cap,33) float64, rows >= offs[C]
 * untouched.
 *   Neighbours of point i: regtr_estimate_normals' rule (own cloud, d^2 strictly below radius^2, i included, the max_nn
 *   smallest by (d^2, index)), entry 0 first.  Fewer than 2 neighbours: a zero row.
 *   Pair feature (p1, n1, p2, n2), products and sums rounded one by one, dot products (x x + y y) + z z: d = p2 - p1
 *   (zero feature when |d| = 0); a1 = n1.d / |d|, a2 = n2.d / |d|; when |a1| < |a2|, n1 <-> n2, d -> -d, f2 = -a2,
 *   else f2 = a1; v = d x n1 (zero feature when |v| = 0), v /= |v|; w = n1 x v; f1 = v.n2; f0 = atan2(w.n2, n1.n2).
 *   SPFH of i (count >= 2): entries k >= 1, in order, add 100 / (count - 1) to bins floor(11 (f0 + pi) / 2pi),
 *   11 + floor(11 (f1 + 1) 0.5) and 22 + floor(11 (f2 + 1) 0.5), each floor clamped to 0..10.
 *   FPFH of i (count >= 2): entries k >= 1 with d^2 != 0, in order, add val = spfh[j][b] / d^2 to feature[b] and to
 *   sum[b / 11]; then feature[b] = feature[b] * (sum != 0 ? 100 / sum : 0) + spfh[i][b].
 * counts (n_cap) i32, nullable: the neighbour count per point.  A |coordinate| beyond
 * regtr_overlap_coord_bound(radius, cell), or not finite, raises REGTR_STATUS_RANGE.  1 + 4 + 3 launches whatever C;
 * no value atomics, no host synchronisation: the result is bit-identical whether a cloud is passed alone or in a stack.
 * ws: regtr_fpfh_ws_bytes(n_cap, max_nn); state: regtr_fpfh_state_bytes(n_cap) (ZERO before the first call; every
 * call leaves it zero). */
#define REGTR_FPFH_DIM 33
#define REGTR_FPFH_MAX_NN 128
size_t regtr_fpfh_ws_bytes(int n_cap, int max_nn);
size_t regtr_fpfh_state_bytes(int n_cap);
int regtr_fpfh(const double* xyz, const double* normals, const int32_t* offs, int C, int n_cap, double radius,
               float cell, int max_nn, double* feature, int32_t* counts, uint32_t* status, void* ws, size_t ws_bytes,
               void* state, size_t state_bytes, void* stream);

/* Feature-space correspondences of B pairs (the matching of Open3D's registration_ransac_based_on_feature_matching).
 * src_feat (offs_s[B],33) float64 with soffs (B+1) i32; tgt_feat (nt_cap,33) float64 and tgt_xyz (nt_cap,3) float64
 * with toffs (B+1) i32; every pair has at most ns_max sources and nt_max targets.  Per pair, with
 * d^2(i, j) = sum over k = 0..32 of (a_k - b_k)^2 accumulated in that order without contraction:
 *   nn[i] (local target index) = the lowest (d^2, j) over the targets (-1 without targets), corr_tgt[i] = its point;
 *   the reverse match of target j = the lowest (d^2, i) over the sources; match i is mutual when the reverse match of
 *   nn[i] is i; n_mutual[b] = their number; mask[i] = mutual, or 1 for every match when mutual_filter = 0 or
 *   n_mutual[b] < min_mutual (Open3D's fallback below 3 ransac_n).
 * Features must be finite.  3 launches; no atomics, no host synchronisation; the result is bit-identical for a pair
 * alone or in a batch.  ws: regtr_feature_match_ws_bytes(B, ns_max, nt_max, nt_cap). */
size_t regtr_feature_match_ws_bytes(int B, int ns_max, int nt_max, int nt_cap);
int regtr_feature_match(const double* src_feat, const int32_t* soffs, const double* tgt_feat, const double* tgt_xyz,
                        const int32_t* toffs, int B, int ns_max, int nt_max, int nt_cap, int mutual_filter,
                        int min_mutual, int32_t* nn, double* corr_tgt, uint8_t* mask, int32_t* n_mutual, void* ws,
                        size_t ws_bytes, void* stream);

/* RANSAC over correspondences of B pairs (Open3D's registration_ransac_based_on_correspondence with
 * TransformationEstimationPointToPoint(false), CorrespondenceCheckerBasedOnEdgeLength(edge_length),
 * CorrespondenceCheckerBasedOnDistance(distance) and RANSACConvergenceCriteria(max_iteration, confidence)), with one
 * deterministic sequential rule in place of Open3D's OpenMP schedule.
 * xyz (n_cap,3) float64 stacked src_0..src_{B-1}, tgt_0..tgt_{B-1} with offs (2B+1) i32 (the validation clouds);
 * corr_src / corr_tgt (m_cap,3) float64, pair b's correspondences (a_i, c_i) in rows [coffs[b], coffs[b+1]) (coffs
 * (B+1) i32); corr_mask (m_cap) u8, nullable: the correspondences with a non-zero byte take part.  The valid ones,
 * in their original order, are 0..n-1.  Per pair:
 *   n < ransac_n or max_iteration = 0: Open3D's empty result.  Otherwise hypotheses k = 0, 1, ... while k < est_k
 *   (est_k = max_iteration at first).  Hypothesis k draws index j < ransac_n as mulhi32(w, n), w word j & 3 of
 *   Philox4x32-10 at counter (k, pair_base + b, j >> 2, 0x52534143) with key (seed lo, seed hi), with replacement.
 *   It is rejected by a repeated index; by the edge-length checker (edge_length > 0): for a pair i < j of the sample,
 *   |a_i - a_j| < |c_i - c_j| edge_length or |c_i - c_j| < |a_i - a_j| edge_length; by Umeyama without scaling on
 *   the sample (means, Sigma = sum (c - mc)(a - ma)^T / n, float64 Jacobi SVD, reflection fix, t = mc - R ma) having
 *   S[1] <= 1e-12 S[0]; or by the distance checker (distance > 0): |T a_i - c_i| > distance for a sample point.
 *   (Norms are sqrt((dx dx + dy dy) + dz dz) without contraction.)  Otherwise it is validated: the source moved by T
 *   (((r0 x + r1 y) + r2 z) + t), the matches of regtr_overlap_nn (nearest target with d^2 < max_dist^2, ties to the
 *   lowest index), fitness = k / n_src, rmse = sqrt(sum d^2 / k); sum d^2 in a fixed order (blocks of 1024 source
 *   points summed as regtr_registration_fit sums a cloud, the blocks by 32 strided chains and a butterfly), so a cloud
 *   of up to 1024 points gets regtr_registration_fit's bits.  It replaces the best (fitness 0, rmse 0, identity at
 *   first) when its fitness is higher, or equal with a lower rmse; then d = log(1 - confidence) / log(1 - f^ransac_n)
 *   (f^n as n - 1 products) sets est_k = ceil(d) when 0 <= d < est_k (d = -inf, a fitness too small for 1 - f^n to
 *   differ from 1, leaves est_k alone).
 * pose_out (B,3,4) float64 = the best T; result (B,5) float64 = (fitness, rmse, hypotheses walked, hypotheses
 * validated, index of the best hypothesis or -1).  A moved source coordinate of a validated hypothesis, or a target
 * coordinate, beyond regtr_overlap_coord_bound(max_dist, cell), or not finite, raises REGTR_STATUS_RANGE.
 * Launches: 2 + 4 (the targets' cell list, cell = max_dist (1 + 1e-3) in fp32) + 3 per chunk, the chunks being
 * first_chunk 2^c hypotheses, at most REGTR_RANSAC_CHUNK_MAX, the last cut at max_iteration; no host synchronisation.
 * The result is bit-identical for every first_chunk, and for a pair alone or in a batch with the same pair_base + b.
 * REGTR_ERR_ARG: ransac_n outside 3..REGTR_RANSAC_MAX_N, max_dist not > 0, confidence outside [0, 1], a negative or
 * non-finite edge_length / distance, first_chunk outside 1..REGTR_RANSAC_CHUNK_MAX, a negative max_iteration or
 * pair_base.  ws: regtr_ransac_ws_bytes(n_cap, m_cap, B, max_iteration, first_chunk); state: regtr_icp_state_bytes(n_cap)
 * (ZERO before the first call; every call leaves it zero). */
#define REGTR_RANSAC_MAX_N 16
#define REGTR_RANSAC_CHUNK_MAX 8192
typedef struct {
    int max_iteration;                       /* hypotheses at most [100000] */
    double confidence;                       /* in [0, 1] [0.999] */
    int ransac_n;                            /* sample size, 3..REGTR_RANSAC_MAX_N [3] */
    double edge_length;                      /* edge-length checker's similarity threshold, 0 = off [0.9] */
    double distance;                         /* distance checker's threshold, 0 = off [0] */
    unsigned long long seed;                 /* Philox key */
    int pair_base;                           /* global index of pair 0 in the draws */
    int first_chunk;                         /* hypotheses of the first chunk, 1..REGTR_RANSAC_CHUNK_MAX [256] */
} regtr_ransac_options;

size_t regtr_ransac_ws_bytes(int n_cap, int m_cap, int B, int max_iteration, int first_chunk);
int regtr_ransac(const double* xyz, const int32_t* offs, int B, int n_cap, const double* corr_src,
                 const double* corr_tgt, const int32_t* coffs, const uint8_t* corr_mask, int m_cap, double max_dist,
                 float cell, const regtr_ransac_options* opt, double* pose_out, double* result, uint32_t* status,
                 void* ws, size_t ws_bytes, void* state, size_t state_bytes, void* stream);

/* Fast Global Registration of B pairs (Open3D's registration_fgr_based_on_correspondence, and the solve of
 * registration_fgr_based_on_feature_matching, with FastGlobalRegistrationOption; Zhou, Park and Koltun, ECCV 2016),
 * with one deterministic rule in place of Open3D's rand() draws and OpenMP sums.
 * xyz (n_cap,3) float64 stacked src_0..src_{B-1}, tgt_0..tgt_{B-1} with offs (2B+1) i32 (the clouds whose means and
 * scale normalise the problem); corr_src / corr_tgt (m_cap,3) float64, pair b's correspondences (a_i, c_i) in rows
 * [coffs[b], coffs[b+1]) (coffs (B+1) i32); corr_mask (m_cap) u8, nullable: the correspondences with a non-zero byte
 * take part, in their original order (n of them).  Products, sums and norms are rounded one by one; norms are
 * sqrt((dx dx + dy dy) + dz dz).  Per pair:
 *   mu_s, mu_t: each cloud's mean (point i added to chain i % 512 in order; each warp's 32 chains by a halving tree,
 *   then the 16 warp sums by a halving tree; / count, 0 for an empty cloud); sigma = the largest |p - mu| over both
 *   clouds (1 when it is 0).  use_absolute_scale: sigma_g = 1, par0 = sigma; else sigma_g = sigma, par0 = 1.  Points
 *   are used as (p - mu) / sigma_g.
 *   tuple_test with n > 0: trials k = 0, 1, ... < 100 n; trial k draws indices mulhi32(w_e, n), e = 0..2, w the words
 *   of Philox4x32-10 at counter (k, pair_base + b, 0, 0x46475254) with key (seed lo, seed hi); it passes when the
 *   edges (0,1), (1,2), (2,0) of both sides have l_s tuple_scale < l_t < l_s / tuple_scale; a pass appends its three
 *   correspondences in draw order, and the walk stops right after the pass that reaches maximum_tuple_count.  The
 *   solve then runs on the 3 x tuples list; without the test on the n correspondences.
 *   Fewer than 10 correspondences: the identity.  Otherwise T = I, par = par0, and iteration_number times: with q the
 *   normalised target point moved by every earlier update, r = p - q, s = (par / (r.r + par))^2, the rows
 *   J_x = (0, -q_z, q_y, -1, 0, 0), J_y = (q_z, 0, -q_x, 0, -1, 0), J_z = (-q_y, q_x, 0, 0, 0, -1) add (J_a J_b) s
 *   to J^T J and (J_a r) s to J^T r (correspondence c to chain c % 256 in order, rows x, y, z; the chains reduced as
 *   above with 8 warps); J^T J x = -J^T r by LDL^T (|det| < 1e-6 or not finite: T and the points stay as they are);
 *   delta = Rz(x2) Ry(x1) Rx(x0) with t = (x3, x4, x5), T = delta T; then with decrease_mu, itr % 4 == 0 and
 *   par > maximum_correspondence_distance, par /= division_factor.
 * pose_out (B,3,4) float64 = R^T, -R^T (-R mu_t + sigma_g t + mu_s) (Open3D's GetInvTransformationOriginalScale);
 * result (B,4) float64 = (correspondences of the solve, tuples kept, trials walked, final par).
 * 2 launches whatever the data; no value atomics, no host synchronisation; the result is bit-identical for a pair
 * alone or in a batch with the same pair_base + b.  Coordinates must be finite.
 * REGTR_ERR_ARG: B < 1, m_cap above REGTR_FGR_MAX_CORR, division_factor or maximum_correspondence_distance not
 * > 0 and finite, a negative iteration_number, tuple_scale outside (0, 1], maximum_tuple_count outside
 * 1..REGTR_FGR_MAX_TUPLES, pair_base < 0 or pair_base + B beyond INT_MAX.
 * ws: regtr_fgr_ws_bytes(m_cap, B, maximum_tuple_count). */
#define REGTR_FGR_MAX_CORR 21474836                 /* 100 trials per correspondence stay below 2^31 */
#define REGTR_FGR_MAX_TUPLES (1 << 20)
typedef struct {
    double division_factor;                  /* par divisor of the GNC schedule, > 0 [1.4] */
    int use_absolute_scale;                  /* [0] */
    int decrease_mu;                         /* [1] */
    double maximum_correspondence_distance;  /* par's lower bound in the schedule, > 0 [0.025] */
    int iteration_number;                    /* GNC iterations [64] */
    double tuple_scale;                      /* in (0, 1] [0.95] */
    int maximum_tuple_count;                 /* 1..REGTR_FGR_MAX_TUPLES [1000] */
    int tuple_test;                          /* [0] */
    unsigned long long seed;                 /* Philox key of the tuple draws */
    int pair_base;                           /* global index of pair 0 in the draws */
} regtr_fgr_options;

size_t regtr_fgr_ws_bytes(int m_cap, int B, int maximum_tuple_count);
int regtr_fgr(const double* xyz, const int32_t* offs, int B, int n_cap, const double* corr_src,
              const double* corr_tgt, const int32_t* coffs, const uint8_t* corr_mask, int m_cap,
              const regtr_fgr_options* opt, double* pose_out, double* result, void* ws, size_t ws_bytes,
              void* stream);

/* ---- pose graph ------------------------------------------------------------------- */

#define REGTR_POSE_GRAPH_MAX_NODES 256

/* Options of regtr_pose_graph_optimize (Open3D's GlobalOptimizationOption and GlobalOptimizationConvergenceCriteria;
 * defaults in brackets). */
typedef struct {
    double max_correspondence_distance;      /* d of the line process */
    double edge_prune_threshold;             /* [0.25] */
    double preference_loop_closure;          /* [1.0] */
    double min_relative_increment;           /* [1e-6] */
    double min_relative_residual_increment;  /* [1e-6] */
    double min_right_term;                   /* [1e-6] */
    double min_residual;                     /* [1e-6] */
    double upper_scale_factor;               /* [2/3] */
    double lower_scale_factor;               /* [1/3] */
    int reference_node;                      /* [0] */
    int max_iteration;                       /* [100] */
    int max_iteration_lm;                    /* [20] */
} regtr_pose_graph_options;

/* Robust optimisation of G independent pose graphs (Open3D's global_optimization with
 * GlobalOptimizationLevenbergMarquardt; Choi, Zhou and Koltun 2015, section 5).  All arithmetic is float64.
 * Graph g owns nodes [node_offs[g], node_offs[g+1]) and edges [edge_offs[g], edge_offs[g+1]) (int32 device offsets);
 * poses (n_nodes,3,4) fragment -> world, read as the initial poses and overwritten with the result; edges (n_edges,2)
 * graph-local (s, t); X (n_edges,3,4) maps source-fragment into target-fragment coordinates (rigid: X^-1 is taken as
 * [R^T | -R^T t]); info (n_edges,6,6); uncertain (n_edges) nonzero for a loop closure.
 *   zeta_e = v(X^-1 P_t^-1 P_s), v(M) = ((M21-M12)/2, (M02-M20)/2, (M10-M01)/2, M03, M13, M23);
 *   J_s[:,k] = v(X^-1 P_t^-1 A_k P_s) (A_k the generators of rotations about x, y, z and translations), J_t = -J_s;
 *   P_n <- T(delta_n) P_n, T(delta) = [Rz(d2) Ry(d1) Rx(d0) | d3..5];
 *   mu = preference * d^2 * mean Lambda_e[5][5]; F = sum c_e zeta^T Lambda zeta + mu sum (sqrt(c_e) - 1)^2;
 *   H = sum c_e [J_s J_t]^T Lambda [J_s J_t], b = -sum c_e [J_s J_t]^T Lambda zeta (dense 6N system);
 *   confidence update (uncertain edges only): c_e = (mu / (mu + zeta^T Lambda zeta))^2, certain edges c_e = 1.
 * LM: lambda = 1e-5 max diag H, nu = 2; stop when max|b| < min_right_term.  Per outer iteration up to
 * max_iteration_lm attempts: Cholesky of H + lambda I (a failure is a rejected step); stop when |delta| <
 * min_rel_inc (|x| + min_rel_inc), x the stacked v(P_n); F' at the moved poses, rho = (F - F') / (delta . (lambda delta
 * + b) + 1e-3); rho > 0 accepts the step (stop when |F - F'| < min_rel_res_inc F; recompute zeta, H, b; stop when
 * max|b| < min_right_term; lambda *= max(lower, min(upper, 1 - (2 rho - 1)^3)), nu = 2), else lambda *= nu, nu *= 2;
 * out of attempts stops.  Then the confidences, F, H and b are updated; stop when F < min_residual or at
 * max_iteration.  A graph without edges or with H = 0 is returned unchanged.
 * Two passes: all edges, then (from pass 1's poses and confidences, mu over the kept edges) the edges left after
 * dropping every uncertain edge with c_e < edge_prune_threshold.  Gauge: P_n <- P_ref^0 P_ref^-1 P_n, the reference
 * node written back bit for bit (nothing is touched when no step was accepted).
 * confidence (n_edges) float64, kept (n_edges) uint8, result (G,4) float64 = (pass-1 iterations, pass-2 iterations,
 * final objective, edges kept).  max_nodes >= every graph's node count: above REGTR_POSE_GRAPH_MAX_NODES
 * REGTR_ERR_UNSUPPORTED.  sq_nodes = sum over the graphs of N_g^2 (graph g's dense system lives at 36 sum_{g'<g} N_g'^2
 * doubles of the workspace).  A graph with more nodes than max_nodes or beyond sq_nodes, s = t, an index out of
 * range, a reference node out of range or a non-finite pose, X or info raises REGTR_STATUS_INPUT and is left as it
 * was (confidence 0, kept 0, result (0, 0, nan, 0)).  One persistent CTA per graph: one launch whatever G, N or convergence, no host
 * synchronisation, sums in a fixed order: a graph's result is bit-identical alone or in a batch.
 * ws: regtr_pose_graph_ws_bytes (36 * sq_nodes * 16 bytes for the dense systems and their factors, plus per-node
 * and per-edge terms). */
size_t regtr_pose_graph_ws_bytes(int G, int n_nodes, int n_edges, long long sq_nodes);
int regtr_pose_graph_optimize(const int32_t* node_offs, const int32_t* edge_offs, int G, int n_nodes, int n_edges,
                              int max_nodes, long long sq_nodes, double* poses, const int32_t* edges, const double* X,
                              const double* info, const uint8_t* uncertain, const regtr_pose_graph_options* opt,
                              double* confidence, uint8_t* kept, double* result, uint32_t* status, void* ws,
                              size_t ws_bytes, void* stream);

/* Per-pair flags of regtr_train_augment */
#define REGTR_PREP_PERTURB_SRC 1  /* the perturbation moves the source (else the target) */
#define REGTR_PREP_CENTRE 2       /* rotate about the perturbed cloud's centroid ('small' mode) */
#define REGTR_PREP_SWAP 4         /* swap source and target */
#define REGTR_PREP_SHUFFLE 8      /* permute the points (and truncate to max_pts) */

/* The reference's training augmentations (data_loaders/transforms.py:15-149: RigidPerturb -> Jitter ->
 * ShufflePoints -> RandomSwap) applied to the clouds of regtr_overlap_nn, with its nn as the overlap.
 * pert (B,3,4) float64: the host-drawn perturbation P; flags (B) i32: REGTR_PREP_*.  Pose: pose P'^-1 (source
 * perturbed) or P' pose, inverted when swapped, P' = P about the centroid with REGTR_PREP_CENTRE.  Output slot s of
 * the augmented batch (src_0..src_{B-1}, tgt_0..) holds out_offs[s+1] - out_offs[s] = min(n, max_pts) points (no
 * truncation without SHUFFLE) of its input cloud: out_xyz[k] = fp32(P' x[perm(k)] + noise * N(0,1)^3) with perm a
 * keyed bijection (Feistel network, cycle walking) and the normals from Philox4x32-10 keyed by (seed, step, pair,
 * side, point index); out_mask (out_cap bytes) = nn >= 0 of that point.  out_pose (B,3,4) fp32.
 * corr (2, corr_cap >= n_src_cap) i32: mutual matches with a nonzero target index whose ends survive the truncation,
 * in ascending source index, remapped through the permutation (rows swapped for swapped pairs); pair b owns columns
 * [corr_offs[b], corr_offs[b+1]).  n_src_cap >= offs[B].  ws / state: the *_bytes functions (state ZERO before the
 * first call; every call leaves it zero).  The device draws of pair b are keyed by pair_base + b (0 <= pair_base <=
 * 2^30): a slice of a batch that starts at global pair pair_base draws exactly what those pairs draw in the whole
 * batch; a whole batch passes 0. */
size_t regtr_train_augment_ws_bytes(int n_src_cap, int B);
size_t regtr_train_augment_state_bytes(int n_src_cap);
int regtr_train_augment(const double* xyz, const int32_t* offs, int B, int n_src_cap, const double* pose,
                        const int32_t* nn, const double* pert, const int32_t* flags, unsigned long long seed,
                        unsigned long long step, int pair_base, double noise, int max_pts, const int32_t* out_offs,
                        int out_cap, float* out_xyz, uint8_t* out_mask, float* out_pose, int32_t* corr, int corr_cap,
                        int32_t* corr_offs, void* ws, size_t ws_bytes, void* state, size_t state_bytes,
                        void* stream);

/* ---- training data (ModelNet40) --------------------------------------------------- */

#define REGTR_STATUS_INPUT 16u    /* ModelNet pairs: a shape index out of range or a coordinate that is not finite;
                                     registration fit: a match that regtr_overlap_nn cannot have produced */
#define REGTR_STATUS_CROP 32u     /* ModelNet pairs: a crop kept fewer than n_out points */
#define REGTR_MODELNET_MAX_PTS 2048
#define REGTR_MODELNET_PARAMS 18  /* doubles per pair in params: dir_src[3], dir_tgt[3], transform[12] */

/* The reference's ModelNet crop chain (data_loaders/modelnet_transforms.py: SplitSourceRef -> RandomCrop ->
 * RandomTransformSE3_euler -> Resampler -> RandomJitter -> ShufflePoints) for B pairs, one CTA per pair.  Pair b
 * takes shape items[b] of shapes (n_shapes, n_pts <= REGTR_MODELNET_MAX_PTS, 3) fp32 and, per side (0 = source,
 * 1 = target) with the crop direction of params[b]:
 *   centroid c = fp32(S / n_pts), S the float64 sum of the points in a fixed order (see modelnet.cu);
 *   d_i = ((fp64(x_i - c) u0 + fp64(y_i - c) u1) + fp64(z_i - c) u2), the differences in fp32, no contraction;
 *   kept = d_i > thr, thr = numpy's linear interpolation between order statistics k and k + 1 of d with weight
 *   gamma, or thr = 0 when k < 0 (RandomCrop with p_keep == 0.5);
 *   the first n_out positions of a keyed Feistel bijection over the kept points, in ascending raw index, choose the
 *   ordered subset; a source point is moved by params' 3x4 transform in float64 and rounded once to fp32; every point
 *   gets fp32(fp64(x) + clip(noise * N(0,1), -clip, clip)), N(0,1) from Philox4x32-10 keyed by (seed, step, pair,
 *   side, raw index).
 * out_xyz (2B, n_out, 3): src_0..src_{B-1}, tgt_0..tgt_{B-1}; out_mask (2B, n_out): the raw point survives the other
 * side's crop; corr (B, 2, n_out): (source position, target position) of every raw point present in both outputs, in
 * ascending raw index, corr_n (B) of them.  A crop with fewer than n_out points raises REGTR_STATUS_CROP, a bad item
 * or a non-finite coordinate REGTR_STATUS_INPUT; such a pair gets corr_n = 0.  The struct is passed by value.
 * The device draws of pair b are keyed by pair_base + b (0 <= pair_base <= 2^30), as for regtr_train_augment.
 * One launch. */
typedef struct {
    const float* shapes;
    const double* params;     /* (B, REGTR_MODELNET_PARAMS) */
    const int32_t* items;     /* (B) */
    float* out_xyz;
    uint8_t* out_mask;
    int32_t* corr;
    int32_t* corr_n;
    uint32_t* status;
    unsigned long long seed, step;
    double gamma, noise, clip;
    int n_shapes, n_pts, n_out, k, B;
} regtr_modelnet_args;
int regtr_modelnet_augment(const regtr_modelnet_args* args, int pair_base, void* stream);

/* ---- training-loop bookkeeping ---------------------------------------------------- */

#define REGTR_METER_MAX_KEYS 16
#define REGTR_METER_MAX_BANKS 4

/* One step's loss scalars into device-resident meter banks (utils/misc.py AverageMeter.update, StatsMeter) and the
 * trainer's loss_smooth EMA (trainer.py:127-134).  The struct lives in host memory and is passed to the kernel by
 * value: no descriptor upload.  Every pointer inside is device memory.
 *   bank b, key k: banks[b][4k .. 4k+3] = (val, sum, sq_sum, count) in fp64; a NaN value is skipped (math.isnan:
 *   +-inf is accumulated), else val = v, sum += v, sq_sum += v * v, count += 1 with IEEE double roundings (no FMA),
 *   so the sums equal Python floats fed the same .item() values.  All-zero rows are cleared meters.
 *   smooth (NULL: no EMA) = [loss_smooth, 1.0 once set], fed by vals[total_key]: the first value is taken as it is;
 *   afterwards a non-finite value is skipped and its step appended to log, else s = 0.99 s + 0.01 v.
 *   log (NULL: none) = [n, step_1 .. step_log_cap]: n counts every skipped step, the first log_cap are kept.
 * One launch. */
typedef struct {
    const float* vals[REGTR_METER_MAX_KEYS];  /* 0-d fp32 loss values, one per key */
    double* banks[REGTR_METER_MAX_BANKS];     /* (n_keys, 4) fp64 each */
    double* smooth;
    long long* log;
    long long step;                           /* recorded in the log */
    int n_keys, n_banks;
    int total_key;                            /* index of 'total' in vals, or -1: no EMA */
    int log_cap;
} regtr_meter_args;
int regtr_meter_update(const regtr_meter_args* args, void* stream);

/* Pose errors of one validation batch (utils/se3_torch.py se3_compare, generic_reg_model.py _compute_metrics /
 * _aggregate_metrics): for layer l < L and pair b < B, in fp64 from the fp32 inputs, with R = Ra Rb^T,
 *   rot = acos(clamp(0.5 (trace R - 1), -1, 1)) * 180 / pi,   trans = || ta - R tb ||.
 * rot_hist / trans_hist (L, hist_cap) fp64 get them at columns [offset, offset + B); acc (L, 4) fp64 accumulates
 * (sum rot, sum trans, n_success, n) pair by pair in order; success = rot < thresh_rot && trans < thresh_trans.
 * One launch. */
typedef struct {
    const float* pred;    /* (L, B, 3, 4) predicted poses */
    const float* gt;      /* (B, 3, 4) ground truth */
    double* rot_hist;
    double* trans_hist;
    double* acc;
    double thresh_rot, thresh_trans;
    int L, B, offset, hist_cap;
} regtr_pose_err_args;
int regtr_pose_errors(const regtr_pose_err_args* args, void* stream);

/* ---- training losses --------------------------------------------------------------- */

#define REGTR_LOSS_DIM 256       /* d_embed of the InfoNCE kernels */
#define REGTR_LOSS_MAX_LEVELS 8
#define REGTR_LOSS_MAX_LAYERS 8
#define REGTR_LOSS_MAX_TERMS 8

/* Ground-truth overlap of every pyramid level (compute_overlaps, kpconv.py:540-566).  pyr[0] (n[0]) is given: the
 * stacked level-0 masks as fp32.  Level p >= 1:
 *   pyr[p][i] = clamp(sum_{valid k} pyr[p-1][pool[p][i,k]] / #valid, 0, 1),  valid: pool[p][i,k] < *n_prev[p],
 * summed over the K[p] slots in ascending order in fp32, one fp32 division; 0 / 0 stays NaN.  pool[p] is the
 * (n[p], K[p]) int32 pooling table from level p-1 to level p; n_prev[p] points at the device int32 number of points of
 * level p-1.  Index 0 of pool, K and n_prev is unused.  One launch per level. */
typedef struct {
    float* pyr[REGTR_LOSS_MAX_LEVELS];
    const int32_t* pool[REGTR_LOSS_MAX_LEVELS];
    const int32_t* n_prev[REGTR_LOSS_MAX_LEVELS];
    int n[REGTR_LOSS_MAX_LEVELS];
    int K[REGTR_LOSS_MAX_LEVELS];
    int n_levels;
} regtr_overlap_pyr_args;
int regtr_overlap_pyramid(const regtr_overlap_pyr_args* args, void* stream);

/* Ws = triu(W) + triu(W)^T of a (256, 256) matrix, written as the TF32 halves regtr_gemm_tf32x3 reads (Ws = hi + lo,
 * rounded as regtr_split_tf32 rounds), and its adjoint dW += triu(dWs + dWs^T).  One launch each. */
int regtr_sym_weight(const float* W, float* Ws_hi, float* Ws_lo, void* stream);
int regtr_sym_weight_bwd(const float* dWs, float* dW, void* stream);

/* The losses of one batch of B pairs on the N packed coarse tokens (source clouds 0..B-1, then target clouds; offs
 * (2B+1) int32 device starts).  The struct lives in host memory and is passed to the kernels by value; every pointer
 * inside is device memory.  vals (n_vals) receives the fp32 loss values at the indices named by ov_val / corr_val
 * (per decoder layer, -1: that layer has no such loss) and term_val (per InfoNCE term).
 *
 * regtr_loss_pointwise (one launch): per layer l, the BCE with logits of logit[l] against w, meaned over N, and
 *   sum w |corr[l] - gt|_1 / max(sum w, 1e-6) over the source tokens (gt = R x + t of the pair's pose) plus the same
 *   over the target tokens (inverse pose); partial sums in fp64 into ws, and the gradients for a unit upstream
 *   gradient into dlogit (L, N) and dcorr (L, N, 3) (zeros for a layer without the loss).
 * regtr_infonce_match (one launch): src_gt (moved source key points), pos (nearest target token of the pair, -1 if
 *   the target cloud is empty) and anchor (nearest distance < r_p) of every source token; rule in csrc/loss.cu.
 * regtr_infonce_fwd (one launch): per term t and source token i, lse[t, i] = log sum_j exp(s_ij) over the pair's
 *   target tokens that are not ignored, s_ij = <q[t][i], feat[t][j]>, and row_loss[t, i] = lse - s_i,pos(i).
 * regtr_loss_finalize (one launch, one CTA): n_anchor (B), pair_loss[t, b] = sum_anchors row_loss / n_anchor in fp64
 *   (NaN without an anchor), vals[term_val[t]] = mean_b pair_loss, and the pointwise values from ws.
 * regtr_loss_pointwise_bwd (one launch): dlogit_out = g[ov_val[l]] * dlogit, dcorr_out = g[corr_val[l]] * dcorr.
 * regtr_infonce_bwd (two launches): with c_i = anchor_i g[term_val[t]] / (n_anchor(b) B) and
 *   G_ij = c_i (exp(s_ij - lse_i) - [j = pos(i)]):  dq[t] rows of the source tokens = G feat[t],  dfeat[t] rows of
 *   the target tokens = G^T q[t].  Source and target rows are owned by different CTAs: no atomics. */
typedef struct {
    const float* xyz;       /* (N, 3) coarse key points */
    const int32_t* offs;    /* (2B + 1) */
    const float* pose;      /* (B, 3, 4) ground truth */
    const float* w;         /* (N) coarsest overlap level */
    const float* logit;     /* (L, N) */
    const float* corr;      /* (L, N, 3) */
    float* dlogit;          /* (L, N) unit-upstream gradients */
    float* dcorr;           /* (L, N, 3) */
    float* dlogit_out;      /* backward outputs */
    float* dcorr_out;
    const float* q[REGTR_LOSS_MAX_TERMS];     /* (>= n_src, 256): source features times Ws */
    const float* feat[REGTR_LOSS_MAX_TERMS];  /* (N, 256): the term's packed features */
    float* dq[REGTR_LOSS_MAX_TERMS];          /* (>= n_src, 256) */
    float* dfeat[REGTR_LOSS_MAX_TERMS];       /* (N, 256): target rows are written */
    float* src_gt;          /* (N, 3) */
    int32_t* pos;           /* (N) */
    int32_t* anchor;        /* (N) */
    float* lse;             /* (n_terms, N) */
    float* row_loss;        /* (n_terms, N) */
    double* pair_loss;      /* (n_terms, B) */
    int32_t* n_anchor;      /* (B) */
    float* vals;            /* (n_vals) */
    const float* g;         /* (n_vals) upstream gradient of vals */
    double* ws;             /* regtr_loss_ws_bytes(N, L) */
    size_t ws_bytes;
    double rp2, rn2;        /* r_p^2, r_n^2 */
    int N, B, L;
    int max_src, max_tgt;   /* longest source / target cloud (grid sizes) */
    int n_terms, n_vals;
    int ov_val[REGTR_LOSS_MAX_LAYERS], corr_val[REGTR_LOSS_MAX_LAYERS], term_val[REGTR_LOSS_MAX_TERMS];
    int pad_;
} regtr_loss_args;
size_t regtr_loss_ws_bytes(int N, int L);
int regtr_loss_pointwise(const regtr_loss_args* args, const double* norm, void* stream);
int regtr_loss_pointwise_bwd(const regtr_loss_args* args, void* stream);
int regtr_infonce_match(const regtr_loss_args* args, void* stream);
int regtr_infonce_fwd(const regtr_loss_args* args, void* stream);
int regtr_infonce_bwd(const regtr_loss_args* args, const double* norm, void* stream);
int regtr_loss_finalize(const regtr_loss_args* args, const double* norm, void* stream);

/* Batch-global normalisers for data-parallel training, where each rank holds a slice of the pairs.
 * regtr_loss_norms (one launch): out (4 doubles, device) = (N, sum w over the source tokens, sum w over the target
 *   tokens, B) of this call, the sums in the order regtr_loss_pointwise takes them.
 * norm (optional, device; regtr_loss_pointwise, regtr_infonce_bwd, regtr_loss_finalize and the circle loss's
 *   regtr_circle_finalize and regtr_circle_bwd): these four normalisers in place of this call's own.  The BCE is meaned
 *   over norm[0] tokens, the L1 terms divided by max(norm[1], 1e-6) and max(norm[2], 1e-6), the InfoNCE and circle
 *   terms meaned over norm[3] pairs.  With norm = the element-wise sum of every rank's regtr_loss_norms, each rank's
 *   values and gradients are its exact share of the whole batch's, and the shares add up to them; norm = NULL uses
 *   this call's own, bit-identical to passing this call's regtr_loss_norms. */
int regtr_loss_norms(const regtr_loss_args* args, double* out, void* stream);

/* The circle feature loss (CircleLossFull(dist_type='euclidean'), feature_loss_type = 'circle') in place of InfoNCE, on
 * the same regtr_loss_args: feat[t] (N, 256) are the term's packed features, source and target rows alike; q, dq,
 * pos, anchor, lse, row_loss and n_anchor are not read.  The circle-only buffers, all device memory: */
typedef struct {
    int32_t* n_pos;     /* (N) positives of each token: a source token's over its pair's target tokens, a target
                           token's over its pair's source tokens */
    int32_t* n_neg;     /* (N) negatives, the same way */
    int32_t* n_sel;     /* (2B) selected tokens (a positive and a negative) of each cloud, offs order */
    double* lse_pos;    /* (n_terms, N) log-sum-exp of the positive exponents of each token's row / column */
    double* lse_neg;    /* (n_terms, N) of the negative exponents */
} regtr_circle_args;
/* Rule and arithmetic in csrc/loss.cu.  D_ij = sqrt(|f_i - f_j|^2 + 1e-12); positive: key-point distance < r_p,
 * negative: > r_n (source key points moved by the ground truth); z+ = 10 (D - 0.1) max(D - 0.1, 0) on positives,
 * z- = 10 (1.4 - D) max(1.4 - D, 0) on negatives, 0 elsewhere.
 * regtr_circle_match (one launch): src_gt, n_pos and n_neg of every token.
 * regtr_circle_fwd (two launches): lse_pos / lse_neg of every source row over its pair's target tokens (one launch)
 *   and of every target column over its pair's source tokens (the other); -inf when the other cloud is empty.
 * regtr_circle_finalize (one launch, one CTA): n_sel; pair_loss[t, b] = (mean over the selected source tokens +
 *   mean over the selected target tokens of softplus(lse_pos + lse_neg) / 10) / 2 in fp64 (NaN when a side has no
 *   selected token; softplus is x above 20); vals[term_val[t]] = mean_b pair_loss; the pointwise values from ws.
 * regtr_circle_bwd (two launches): with H_ij = (dL/dD_ij) / D_ij for the upstream gradient g,
 *   dfeat[t] rows of the source tokens = sum_j H_ij (f_i - f_j) (one launch) and of the target tokens
 *   sum_i H_ij (f_j - f_i) (the other).  Source and target rows are owned by different CTAs: no atomics.
 * norm (optional): the batch-global normalisers of regtr_loss_norms; the terms are meaned over norm[3] pairs. */
int regtr_circle_match(const regtr_loss_args* args, const regtr_circle_args* circ, void* stream);
int regtr_circle_fwd(const regtr_loss_args* args, const regtr_circle_args* circ, void* stream);
int regtr_circle_finalize(const regtr_loss_args* args, const regtr_circle_args* circ, const double* norm,
                          void* stream);
int regtr_circle_bwd(const regtr_loss_args* args, const regtr_circle_args* circ, const double* norm, void* stream);

/* ---- transformer dropout (training) ------------------------------------------------ */

/* Keep mask (analysis / tests): out[r * cols + j] = 1 if row r, column j of local cloud `cloud` (query cloud of an
 * attention site), head `head`, is kept, for r < rows, j < cols.  out: rows x cols uint8. */
int regtr_dropout_keep_mask(const regtr_dropout_args* args, int cloud, int head, int rows, int cols, uint8_t* out,
                            void* stream);

/* Feed-forward dropout (site 5), in place: h[r, j] = m scale h[r, j] over the n x F packed rows of the clouds of
 * offs (2B + 1, device); max_len: host bound of the cloud lengths. */
int regtr_dropout_rows(float* h, int n, int F, const int32_t* offs, int max_len, const regtr_dropout_args* drop,
                       void* stream);

/* ---- status word helpers (device uint32) ------------------------------------------ */
int regtr_status_clear(uint32_t* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* REGTR_B200_H_ */
