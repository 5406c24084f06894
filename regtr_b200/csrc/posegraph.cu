// Pose-graph optimisation of G independent graphs: Open3D's GlobalOptimizationLevenbergMarquardt with the line
// process of Choi, Zhou and Koltun (2015, section 5), two passes with pruning of the uncertain edges in between.
// The contract, term by term, is the comment of regtr_pose_graph_optimize in include/regtr_b200.h; DESIGN.md lists
// where it departs from Open3D.
//
// One persistent CTA per graph runs both passes and every LM decision: one launch whatever G, N or convergence, no
// host synchronisation.  Every sum has a fixed order (per-thread strided partial sums in ascending index, then a
// fixed shared-memory tree; H and b summed per entry in ascending edge order), so a graph's result does not depend on
// the batch it is in.
#include "rigid.cuh"

namespace {

constexpr int PG_THREADS = 256;
constexpr int PG_S = 49;     // per edge: S = Jx^T Lambda Jx, Jx = [J_s | zeta] (6 x 7)
constexpr int PG_J = 42;     // per edge: Jx itself

struct PgWs {
    double* H;       // 36 * sq_nodes doubles: graph g's dense 6N x 6N system at 36 * sum_{g' < g} N_g'^2
    double* A;       // the same layout: the Cholesky factor of H + lambda I (lower triangle)
    double* S;       // PG_S per edge
    double* Jx;      // PG_J per edge
    double* Pt;      // 12 per node: trial poses
    double* vec;     // 4 vectors of 6N per graph: b, rhs, y, delta; then the factor's diagonal
    int32_t* inc;    // per graph (N + 1) offsets at node_offs[g] + g, then 2E incident edges at 2 edge_offs[g]
    int32_t* pair;   // 2 per edge: (first edge of its node pair, next edge of the same pair or -1)
    size_t total;
};

PgWs carve_pg(void* ws, int G, int n_nodes, int n_edges, long long sq_nodes) {
    PgWs w;
    char* p = (char*)ws;
    size_t off = 0;
    auto take = [&](size_t bytes) { char* r = p ? p + off : nullptr; off += regtr_align(bytes); return (void*)r; };
    const size_t dense = 36 * (size_t)sq_nodes;
    w.H = (double*)take(sizeof(double) * dense);
    w.A = (double*)take(sizeof(double) * dense);
    w.S = (double*)take(sizeof(double) * PG_S * (size_t)n_edges);
    w.Jx = (double*)take(sizeof(double) * PG_J * (size_t)n_edges);
    w.Pt = (double*)take(sizeof(double) * 12 * (size_t)n_nodes);
    w.vec = (double*)take(sizeof(double) * 30 * (size_t)n_nodes);
    w.inc = (int32_t*)take(sizeof(int32_t) * ((size_t)n_nodes + G + 2 * (size_t)n_edges));
    w.pair = (int32_t*)take(sizeof(int32_t) * 2 * (size_t)n_edges);
    w.total = off;
    return w;
}

// ---- 3x4 rigid transforms (row-major, implicit last row 0 0 0 1)
__device__ __forceinline__ void rt_inv(const double* a, double* o) {
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o[4 * r + c] = a[4 * c + r];
        o[4 * r + 3] = -((a[r] * a[3] + a[4 + r] * a[7]) + a[8 + r] * a[11]);
    }
}

__device__ __forceinline__ void rt_mul(const double* a, const double* b, double* o) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 4; ++c) {
            const double v = (a[4 * r] * b[c] + a[4 * r + 1] * b[4 + c]) + a[4 * r + 2] * b[8 + c];
            o[4 * r + c] = c == 3 ? v + a[4 * r + 3] : v;
        }
}

// v(M) = ((M21 - M12) / 2, (M02 - M20) / 2, (M10 - M01) / 2, M03, M13, M23)
__device__ __forceinline__ void vec6(const double* m, double* v) {
    v[0] = 0.5 * (m[9] - m[6]);
    v[1] = 0.5 * (m[2] - m[8]);
    v[2] = 0.5 * (m[4] - m[1]);
    v[3] = m[3]; v[4] = m[7]; v[5] = m[11];
}

// T(delta) = [Rz(d2) Ry(d1) Rx(d0) | d3..5], the update rule of regtr_icp's point-to-plane step
__device__ __forceinline__ void rt_exp(const double* d, double* o) {
    double R[3][3], t[3];
    rigid_from_vec6(d, R, t);
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) o[4 * r + c] = R[r][c];
        o[4 * r + 3] = t[r];
    }
}

// zeta^T Lambda zeta with the inner sums first, the order S[6][6] is summed in
__device__ __forceinline__ double quad6(const double* L, const double* z) {
    double r = 0.0;
    for (int k = 0; k < 6; ++k) {
        double l = 0.0;
        for (int m = 0; m < 6; ++m) l += L[6 * k + m] * z[m];
        r += z[k] * l;
    }
    return r;
}

struct Graph {
    int N, E, n, ref;
    double* P;                  // poses, in place
    const int32_t* edge;        // (E, 2)
    const double* X;
    const double* info;
    const uint8_t* unc;
    double* conf;
    uint8_t* kept;              // the active edge set of the running pass
    double *H, *A, *S, *Jx, *Pt, *b, *rhs, *y, *d, *dg;
    int32_t *inc_off, *inc, *pair;
};

__device__ double block_sum(double v, double* red) {
    const int t = threadIdx.x;
    __syncthreads();
    red[t] = v;
    __syncthreads();
    for (int h = PG_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) red[t] += red[t + h];
        __syncthreads();
    }
    return red[0];
}

__device__ double block_max(double v, double* red) {
    const int t = threadIdx.x;
    __syncthreads();
    red[t] = v;
    __syncthreads();
    for (int h = PG_THREADS / 2; h > 0; h >>= 1) {
        if (t < h) red[t] = fmax(red[t], red[t + h]);
        __syncthreads();
    }
    return red[0];
}

// W = X^-1 P_t^-1 and zeta = v(W P_s) of edge e at poses P
__device__ void edge_zeta(const Graph& g, const double* P, int e, double* W, double* z) {
    double xi[12], ti[12], m[12];
    rt_inv(g.X + 12 * e, xi);
    rt_inv(P + 12 * g.edge[2 * e + 1], ti);
    rt_mul(xi, ti, W);
    rt_mul(W, P + 12 * g.edge[2 * e], m);
    vec6(m, z);
}

// Jx = [J_s | zeta] and S = Jx^T Lambda Jx of every active edge at the current poses.
// J_s[:, k] = v(W A_k P_s): for a rotation generator, W A_k P_s = [R_W K_k R_s | R_W (e_k x t_s)], K_k v = e_k x v;
// for a translation, [0 | R_W e_k].
__device__ void edge_terms(const Graph& g) {
    for (int e = threadIdx.x; e < g.E; e += PG_THREADS) {
        if (!g.kept[e]) continue;
        double W[12], z[6];
        edge_zeta(g, g.P, e, W, z);
        const double* Ps = g.P + 12 * g.edge[2 * e];
        double* J = g.Jx + PG_J * (size_t)e;
        for (int k = 0; k < 3; ++k) {
            const int k1 = (k + 1) % 3, k2 = (k + 2) % 3;
            double m[12];                           // K_k P_s: row k1 = +row k2 of P_s, row k2 = -row k1, row k = 0
            for (int c = 0; c < 4; ++c) { m[4 * k + c] = 0.0; m[4 * k1 + c] = -Ps[4 * k2 + c]; m[4 * k2 + c] = Ps[4 * k1 + c]; }
            double q[12];
            for (int r = 0; r < 3; ++r)
                for (int c = 0; c < 4; ++c) q[4 * r + c] = (W[4 * r] * m[c] + W[4 * r + 1] * m[4 + c]) + W[4 * r + 2] * m[8 + c];
            double v[6];
            vec6(q, v);
            for (int r = 0; r < 6; ++r) J[7 * r + k] = v[r];
        }
        for (int k = 0; k < 3; ++k)
            for (int r = 0; r < 6; ++r) J[7 * r + 3 + k] = r < 3 ? 0.0 : W[4 * (r - 3) + k];
        for (int r = 0; r < 6; ++r) J[7 * r + 6] = z[r];
        const double* L = g.info + 36 * (size_t)e;
        double* S = g.S + PG_S * (size_t)e;
        for (int c = 0; c < 7; ++c) {
            double lj[6];
            for (int k = 0; k < 6; ++k) {
                double l = 0.0;
                for (int m = 0; m < 6; ++m) l += L[6 * k + m] * J[7 * m + c];
                lj[k] = l;
            }
            for (int a = 0; a < 7; ++a) {
                double s = 0.0;
                for (int k = 0; k < 6; ++k) s += J[7 * k + a] * lj[k];
                S[7 * a + c] = s;
            }
        }
    }
}

// Incident active edges of every node in ascending edge order, and per edge the pair links for the off-diagonal
// blocks: the first active edge of each node pair sums all of them in ascending order.
__device__ void build_lists(const Graph& g) {
    for (int v = threadIdx.x; v < g.N; v += PG_THREADS) {
        int cnt = 0;
        for (int e = 0; e < g.E; ++e)
            if (g.kept[e] && (g.edge[2 * e] == v || g.edge[2 * e + 1] == v)) ++cnt;
        g.inc_off[v + 1] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        g.inc_off[0] = 0;
        for (int v = 0; v < g.N; ++v) g.inc_off[v + 1] += g.inc_off[v];
    }
    __syncthreads();
    for (int v = threadIdx.x; v < g.N; v += PG_THREADS) {
        int pos = g.inc_off[v];
        for (int e = 0; e < g.E; ++e)
            if (g.kept[e] && (g.edge[2 * e] == v || g.edge[2 * e + 1] == v)) g.inc[pos++] = e;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < g.E; e += PG_THREADS) {
        if (!g.kept[e]) continue;
        const int s = g.edge[2 * e], t = g.edge[2 * e + 1];
        int first = 1, next = -1;
        for (int p = g.inc_off[s]; p < g.inc_off[s + 1]; ++p) {
            const int f = g.inc[p];
            const int o = g.edge[2 * f] == s ? g.edge[2 * f + 1] : g.edge[2 * f];
            if (f == e || o != t) continue;
            if (f < e) first = 0;
            else if (next < 0) next = f;
        }
        g.pair[2 * e] = first;
        g.pair[2 * e + 1] = next;
    }
    __syncthreads();
}

// H = sum c [J_s J_t]^T Lambda [J_s J_t] and b = -sum c [J_s J_t]^T Lambda zeta over the active edges, J_t = -J_s:
// diagonal blocks +c Q, off-diagonal blocks -c Q (Q = S[0:6, 0:6]), b_s -= c S[:, 6], b_t += c S[:, 6].  Blocks
// without edges keep the zeros written at the start of the pass.
__device__ void assemble(const Graph& g) {
    const int n = g.n;
    for (int it = threadIdx.x; it < 36 * g.N; it += PG_THREADS) {
        const int v = it / 36, a = (it % 36) / 6, c = it % 6;
        double h = 0.0;
        for (int p = g.inc_off[v]; p < g.inc_off[v + 1]; ++p) {
            const int e = g.inc[p];
            h += g.conf[e] * g.S[PG_S * (size_t)e + 7 * a + c];
        }
        g.H[(size_t)(6 * v + a) * n + 6 * v + c] = h;
    }
    for (int it = threadIdx.x; it < 36 * g.E; it += PG_THREADS) {
        const int e = it / 36, a = (it % 36) / 6, c = it % 6;
        if (!g.kept[e] || !g.pair[2 * e]) continue;
        double h = 0.0;
        for (int f = e; f >= 0; f = g.pair[2 * f + 1]) h -= g.conf[f] * g.S[PG_S * (size_t)f + 7 * a + c];
        const int s = g.edge[2 * e], t = g.edge[2 * e + 1];
        g.H[(size_t)(6 * s + a) * n + 6 * t + c] = h;
        g.H[(size_t)(6 * t + a) * n + 6 * s + c] = h;
    }
    for (int it = threadIdx.x; it < n; it += PG_THREADS) {
        const int v = it / 6, k = it % 6;
        double r = 0.0;
        for (int p = g.inc_off[v]; p < g.inc_off[v + 1]; ++p) {
            const int e = g.inc[p];
            const double q = g.conf[e] * g.S[PG_S * (size_t)e + 7 * k + 6];
            r = g.edge[2 * e] == v ? r - q : r + q;
        }
        g.b[it] = r;
    }
    __syncthreads();
}

// F = sum c_e r_e + mu sum (sqrt(c_e) - 1)^2 over the active edges; r_e = S[6][6] at the current poses, or
// recomputed at poses P when P is given
__device__ double objective(const Graph& g, double mu, const double* P, double* red) {
    double f = 0.0;
    for (int e = threadIdx.x; e < g.E; e += PG_THREADS) {
        if (!g.kept[e]) continue;
        double r;
        if (P) {
            double W[12], z[6];
            edge_zeta(g, P, e, W, z);
            r = quad6(g.info + 36 * (size_t)e, z);
        } else {
            r = g.S[PG_S * (size_t)e + 48];
        }
        const double c = g.conf[e], q = sqrt(c) - 1.0;
        f += c * r + mu * (q * q);
    }
    return block_sum(f, red);
}

// Cholesky factor of H + lam I into A (lower triangle) and dg (diagonal); right-looking, one column at a time.  The
// rank-1 update of column j only touches the rows whose entry in column j is nonzero, so sparse graphs (chains with
// a few loops) cost little.  false when a pivot is not positive and finite: every thread reads the same pivot, and
// every thread has read it before any thread returns, so a rejected step's next attempt cannot overwrite A under a
// thread that is still deciding on this one.
__device__ bool cholesky(const Graph& g, double lam, int* rows, int* cnt) {
    const int n = g.n, T = PG_THREADS;
    __syncthreads();                      // every reader of the previous factor (solve, pivots) is done with A
    for (size_t it = threadIdx.x; it < (size_t)n * n; it += T) {
        const int i = (int)(it / n), j = (int)(it % n);
        if (j <= i) g.A[it] = g.H[it] + (i == j ? lam : 0.0);
    }
    if (threadIdx.x < 2) cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int j = 0; j < n; ++j) {
        const double dj = g.A[(size_t)j * n + j];
        if (!(dj > 0.0 && dj <= 1.7976931348623157e308)) {
            __syncthreads();
            return false;
        }
        const double l = sqrt(dj);
        for (int i = j + 1 + threadIdx.x; i < n; i += T) {
            const double v = g.A[(size_t)i * n + j] / l;
            g.A[(size_t)i * n + j] = v;
            if (v != 0.0) rows[atomicAdd(&cnt[j & 1], 1)] = i;
        }
        if (threadIdx.x == 0) { g.dg[j] = l; cnt[(j + 1) & 1] = 0; }
        __syncthreads();
        const int m = cnt[j & 1];
        for (int it = threadIdx.x; it < m * m; it += T) {
            const int ri = rows[it / m], rk = rows[it % m];
            if (rk <= ri) g.A[(size_t)ri * n + rk] -= g.A[(size_t)ri * n + j] * g.A[(size_t)rk * n + j];
        }
        __syncthreads();
    }
    return true;
}

// (L L^T) d = b by forward and backward substitution, one column at a time
__device__ void solve(const Graph& g) {
    const int n = g.n, T = PG_THREADS;
    for (int i = threadIdx.x; i < n; i += T) g.rhs[i] = g.b[i];
    for (int j = 0; j < n; ++j) {
        __syncthreads();
        const double yj = g.rhs[j] / g.dg[j];
        for (int i = j + 1 + threadIdx.x; i < n; i += T) g.rhs[i] -= g.A[(size_t)i * n + j] * yj;
        if (threadIdx.x == 0) g.y[j] = yj;
    }
    for (int j = n - 1; j >= 0; --j) {
        __syncthreads();
        const double dj = g.y[j] / g.dg[j];
        for (int i = threadIdx.x; i < j; i += T) g.y[i] -= g.A[(size_t)j * n + i] * dj;
        if (threadIdx.x == 0) g.d[j] = dj;
    }
    __syncthreads();
}

struct LmOpt {
    int max_iter, max_iter_lm;
    double min_inc, min_res_inc, min_right, min_res, upper, lower;
};

// One Levenberg-Marquardt pass over the active edges (H already zero outside the blocks the edges fill).  Returns
// the outer iterations begun; *F the final objective; *moved set when a step was accepted.
__device__ int lm_pass(const Graph& g, const LmOpt& o, double mu, double* F_out, int* moved, double* red, int* rows,
                       int* cnt) {
    const int n = g.n;
    edge_terms(g);
    __syncthreads();
    assemble(g);
    double F = objective(g, mu, nullptr, red);
    double hmax = 0.0, bmax = 0.0;
    for (int i = threadIdx.x; i < n; i += PG_THREADS) {
        hmax = fmax(hmax, g.H[(size_t)i * n + i]);
        bmax = fmax(bmax, fabs(g.b[i]));
    }
    hmax = block_max(hmax, red);
    bmax = block_max(bmax, red);
    *F_out = F;
    if (!(hmax > 0.0) || bmax < o.min_right) return 0;
    double lam = 1e-5 * hmax, nu = 2.0;
    int iters = 0;
    for (int iter = 0; iter < o.max_iter; ++iter) {
        iters = iter + 1;
        bool stop = false, accepted = false;
        for (int att = 0; att < o.max_iter_lm && !stop && !accepted; ++att) {
            if (cholesky(g, lam, rows, cnt)) {
                solve(g);
                double dd = 0.0, xx = 0.0, den = 0.0;
                for (int i = threadIdx.x; i < n; i += PG_THREADS) {
                    const double di = g.d[i];
                    dd += di * di;
                    den += di * (lam * di + g.b[i]);
                }
                for (int v = threadIdx.x; v < g.N; v += PG_THREADS) {
                    double x6[6];
                    vec6(g.P + 12 * v, x6);
                    for (int k = 0; k < 6; ++k) xx += x6[k] * x6[k];
                }
                dd = sqrt(block_sum(dd, red));
                xx = sqrt(block_sum(xx, red));
                den = block_sum(den, red) + 1e-3;
                if (dd < o.min_inc * (xx + o.min_inc)) { stop = true; break; }
                for (int v = threadIdx.x; v < g.N; v += PG_THREADS) {
                    double u[12];
                    rt_exp(g.d + 6 * v, u);
                    rt_mul(u, g.P + 12 * v, g.Pt + 12 * v);
                }
                __syncthreads();
                const double Fn = objective(g, mu, g.Pt, red);
                const double rho = (F - Fn) / den;
                if (rho > 0.0) {
                    for (int i = threadIdx.x; i < 12 * g.N; i += PG_THREADS) g.P[i] = g.Pt[i];
                    *moved = 1;
                    const bool small = fabs(F - Fn) < o.min_res_inc * F;
                    F = Fn;
                    __syncthreads();
                    if (small) { stop = true; break; }
                    edge_terms(g);
                    __syncthreads();
                    assemble(g);
                    bmax = 0.0;
                    for (int i = threadIdx.x; i < n; i += PG_THREADS) bmax = fmax(bmax, fabs(g.b[i]));
                    if (block_max(bmax, red) < o.min_right) { stop = true; break; }
                    const double a = 1.0 - (2.0 * rho - 1.0) * (2.0 * rho - 1.0) * (2.0 * rho - 1.0);
                    lam *= fmax(o.lower, fmin(o.upper, a));
                    nu = 2.0;
                    accepted = true;
                    break;
                }
            }
            lam *= nu;
            nu *= 2.0;
        }
        if (!accepted) break;                 // stopped, or out of attempts
        // confidences of the uncertain edges at the accepted poses, then F, H and b with them
        for (int e = threadIdx.x; e < g.E; e += PG_THREADS) {
            if (!g.kept[e] || !g.unc[e]) continue;
            const double q = mu / (mu + g.S[PG_S * (size_t)e + 48]);
            g.conf[e] = q * q;
        }
        __syncthreads();
        assemble(g);
        F = objective(g, mu, nullptr, red);
        if (F < o.min_res) break;
    }
    *F_out = F;
    return iters;
}

// mu = preference d^2 mean Lambda[5][5] over the active edges
__device__ double line_process_mu(const Graph& g, double pref_d2, double* red) {
    double s = 0.0, k = 0.0;
    for (int e = threadIdx.x; e < g.E; e += PG_THREADS)
        if (g.kept[e]) { s += g.info[36 * (size_t)e + 35]; k += 1.0; }
    s = block_sum(s, red);
    k = block_sum(k, red);
    return k > 0.0 ? pref_d2 * (s / k) : 0.0;
}

__device__ bool finite_all(const double* p, int n) {
    for (int i = 0; i < n; ++i)
        if (!(fabs(p[i]) <= 1.7976931348623157e308)) return false;
    return true;
}

__global__ void __launch_bounds__(PG_THREADS, 1)
k_pose_graph(const int32_t* __restrict__ node_offs, const int32_t* __restrict__ edge_offs, int n_nodes, int n_edges,
             int max_nodes, long long sq_nodes, double* poses, const int32_t* __restrict__ edges,
             const double* __restrict__ X,
             const double* __restrict__ info, const uint8_t* __restrict__ uncertain, regtr_pose_graph_options opt,
             double* conf, uint8_t* kept, double* __restrict__ result, uint32_t* status, PgWs w) {
    __shared__ double red[PG_THREADS];
    __shared__ int rows[6 * REGTR_POSE_GRAPH_MAX_NODES];
    __shared__ int cnt[2];
    __shared__ int bad;
    __shared__ double ref0[12], gauge[12];
    const int gi = blockIdx.x, t = threadIdx.x;
    const int n0 = node_offs[gi], n1 = node_offs[gi + 1], e0 = edge_offs[gi], e1 = edge_offs[gi + 1];
    double* res = result + 4 * gi;
    // offsets outside the arrays: nothing of this graph can be addressed safely
    if (!(0 <= n0 && n0 <= n1 && n1 <= n_nodes && 0 <= e0 && e0 <= e1 && e1 <= n_edges)) {
        if (t == 0) { atomicOr(status, REGTR_STATUS_INPUT); res[0] = res[1] = res[3] = 0.0; res[2] = nan(""); }
        return;
    }
    __shared__ Graph sg;          // in shared memory: every helper reads it there instead of holding it in registers
    if (t == 0) {
        Graph& g = sg;
        g.N = n1 - n0; g.E = e1 - e0; g.n = 6 * g.N; g.ref = opt.reference_node;
        g.P = poses + 12 * (size_t)n0;
        g.edge = edges + 2 * (size_t)e0;
        g.X = X + 12 * (size_t)e0;
        g.info = info + 36 * (size_t)e0;
        g.unc = uncertain + e0;
        g.conf = conf + e0;
        g.kept = kept + e0;
        long long dense = 0;                // sum of N_g'^2 over the graphs before this one
        for (int k = 0; k < gi; ++k) {
            const long long m = (long long)node_offs[k + 1] - node_offs[k];
            dense += m * m;
        }
        g.H = w.H + 36 * (size_t)dense;
        g.A = w.A + 36 * (size_t)dense;
        g.S = w.S + PG_S * (size_t)e0;
        g.Jx = w.Jx + PG_J * (size_t)e0;
        g.Pt = w.Pt + 12 * (size_t)n0;
        g.b = w.vec + 30 * (size_t)n0;
        g.rhs = g.b + g.n; g.y = g.rhs + g.n; g.d = g.y + g.n; g.dg = g.d + g.n;
        g.inc_off = w.inc + n0 + gi;
        g.inc = w.inc + (size_t)n_nodes + gridDim.x + 2 * (size_t)e0;
        g.pair = w.pair + 2 * (size_t)e0;
        bad = (g.N > max_nodes || dense + (long long)g.N * g.N > sq_nodes ||
               (g.N > 0 && (g.ref < 0 || g.ref >= g.N))) ? 1 : 0;
    }
    __syncthreads();
    const Graph& g = sg;
    __syncthreads();
    for (int e = t; e < g.E; e += PG_THREADS) {
        const int s = g.edge[2 * e], d = g.edge[2 * e + 1];
        if (s < 0 || s >= g.N || d < 0 || d >= g.N || s == d || !finite_all(g.X + 12 * e, 12) ||
            !finite_all(g.info + 36 * (size_t)e, 36))
            bad = 1;
    }
    for (int v = t; v < g.N; v += PG_THREADS)
        if (!finite_all(g.P + 12 * v, 12)) bad = 1;
    __syncthreads();
    if (bad) {
        for (int e = t; e < g.E; e += PG_THREADS) { g.conf[e] = 0.0; g.kept[e] = 0; }
        if (t == 0) { atomicOr(status, REGTR_STATUS_INPUT); res[0] = res[1] = res[3] = 0.0; res[2] = nan(""); }
        return;
    }
    for (int e = t; e < g.E; e += PG_THREADS) { g.conf[e] = 1.0; g.kept[e] = 1; }
    if (t < 12 && g.N > 0) ref0[t] = g.P[12 * g.ref + t];
    for (size_t i = t; i < (size_t)g.n * g.n; i += PG_THREADS) g.H[i] = 0.0;
    __syncthreads();
    const LmOpt o{opt.max_iteration, opt.max_iteration_lm, opt.min_relative_increment,
                  opt.min_relative_residual_increment, opt.min_right_term, opt.min_residual, opt.upper_scale_factor,
                  opt.lower_scale_factor};
    const double pref_d2 = opt.preference_loop_closure * opt.max_correspondence_distance *
                           opt.max_correspondence_distance;
    int moved = 0;
    double F = 0.0;
    // pass 1: every edge
    build_lists(g);
    int it1 = lm_pass(g, o, line_process_mu(g, pref_d2, red), &F, &moved, red, rows, cnt);
    // prune the uncertain edges the line process switched off, clear their blocks, pass 2 on the rest
    __syncthreads();
    for (int it = t; it < 36 * g.E; it += PG_THREADS) {
        const int e = it / 36, a = (it % 36) / 6, c = it % 6;
        if (!g.kept[e] || !g.pair[2 * e]) continue;
        const int s = g.edge[2 * e], d = g.edge[2 * e + 1];
        g.H[(size_t)(6 * s + a) * g.n + 6 * d + c] = 0.0;
        g.H[(size_t)(6 * d + a) * g.n + 6 * s + c] = 0.0;
    }
    __syncthreads();
    double k = 0.0;
    for (int e = t; e < g.E; e += PG_THREADS) {
        if (g.unc[e] && g.conf[e] < opt.edge_prune_threshold) g.kept[e] = 0;
        k += g.kept[e] ? 1.0 : 0.0;
    }
    k = block_sum(k, red);
    build_lists(g);
    int it2 = lm_pass(g, o, line_process_mu(g, pref_d2, red), &F, &moved, red, rows, cnt);
    // gauge: P_n <- P_ref^0 P_ref^-1 P_n, the reference node written back bit for bit
    __syncthreads();
    if (moved && g.N > 0) {
        if (t == 0) {
            double inv[12];
            rt_inv(g.P + 12 * g.ref, inv);
            rt_mul(ref0, inv, gauge);
        }
        __syncthreads();
        for (int v = t; v < g.N; v += PG_THREADS) {
            double q[12];
            if (v == g.ref) {
                for (int i = 0; i < 12; ++i) q[i] = ref0[i];
            } else {
                rt_mul(gauge, g.P + 12 * v, q);
            }
            for (int i = 0; i < 12; ++i) g.P[12 * v + i] = q[i];
        }
    }
    if (t == 0) { res[0] = it1; res[1] = it2; res[2] = F; res[3] = k; }
}

}  // namespace

extern "C" {

size_t regtr_pose_graph_ws_bytes(int G, int n_nodes, int n_edges, long long sq_nodes) {
    if (G < 0 || n_nodes < 0 || n_edges < 0 || sq_nodes < 0) return 0;
    return carve_pg(nullptr, G, n_nodes, n_edges, sq_nodes).total;
}

int regtr_pose_graph_optimize(const int32_t* node_offs, const int32_t* edge_offs, int G, int n_nodes, int n_edges,
                              int max_nodes, long long sq_nodes, double* poses, const int32_t* edges, const double* X,
                              const double* info, const uint8_t* uncertain, const regtr_pose_graph_options* opt,
                              double* confidence, uint8_t* kept, double* result, uint32_t* status, void* ws,
                              size_t ws_bytes, void* stream) {
    if (max_nodes > REGTR_POSE_GRAPH_MAX_NODES) return REGTR_ERR_UNSUPPORTED;
    if (!node_offs || !edge_offs || !opt || !result || !status || G <= 0 || n_nodes < 0 || n_edges < 0 ||
        max_nodes < 0 || sq_nodes < 0 || !ws)
        return REGTR_ERR_ARG;
    if ((n_nodes > 0 && !poses) || (n_edges > 0 && (!edges || !X || !info || !uncertain || !confidence || !kept)))
        return REGTR_ERR_ARG;
    const regtr_pose_graph_options o = *opt;
    if (!(o.max_correspondence_distance > 0.0) || !(o.edge_prune_threshold >= 0.0) ||
        !(o.preference_loop_closure >= 0.0) || o.reference_node < 0 || o.max_iteration < 0 ||
        o.max_iteration_lm < 1 || !(o.min_relative_increment >= 0.0) || !(o.min_relative_residual_increment >= 0.0) ||
        !(o.min_right_term >= 0.0) || !(o.min_residual >= 0.0) || !(o.upper_scale_factor > 0.0) ||
        !(o.lower_scale_factor > 0.0))
        return REGTR_ERR_ARG;
    PgWs w = carve_pg(ws, G, n_nodes, n_edges, sq_nodes);
    if (ws_bytes < w.total) return REGTR_ERR_WORKSPACE;
    k_pose_graph<<<G, PG_THREADS, 0, (cudaStream_t)stream>>>(node_offs, edge_offs, n_nodes, n_edges, max_nodes, sq_nodes,
                                                             poses, edges, X, info, uncertain, o, confidence, kept,
                                                             result, status, w);
    REGTR_CHECK_LAUNCH();
    return REGTR_OK;
}

}  // extern "C"
