"""Float64 numpy restatement of the information matrix (regtr_registration_information) and of the pose-graph
optimiser (regtr_pose_graph_optimize): the contract in include/regtr_b200.h, term by term, with the same update
rule, stop tests and two passes, and numpy's dense Cholesky in place of the kernel's."""
import numpy as np
from scipy.spatial import cKDTree

GEN = []
for k in range(3):                          # rotation generators: for x, (1,2) = -1 and (2,1) = +1, cyclically
    a = np.zeros((4, 4))
    a[(k + 1) % 3, (k + 2) % 3] = -1.0
    a[(k + 2) % 3, (k + 1) % 3] = 1.0
    GEN.append(a)
for k in range(3):                          # translations
    a = np.zeros((4, 4))
    a[k, 3] = 1.0
    GEN.append(a)


def h44(p):
    p = np.asarray(p, np.float64)
    out = np.eye(4)
    out[:3] = p[:3]
    return out


def rinv(p):
    p = h44(p)
    out = np.eye(4)
    out[:3, :3] = p[:3, :3].T
    out[:3, 3] = -p[:3, :3].T @ p[:3, 3]
    return out


def vec6(m):
    return np.array([(m[2, 1] - m[1, 2]) / 2, (m[0, 2] - m[2, 0]) / 2, (m[1, 0] - m[0, 1]) / 2, m[0, 3], m[1, 3],
                     m[2, 3]])


def rt_exp(d):
    sa, ca, sb, cb, sc, cc = np.sin(d[0]), np.cos(d[0]), np.sin(d[1]), np.cos(d[1]), np.sin(d[2]), np.cos(d[2])
    Rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
    Ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
    Rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
    out = np.eye(4)
    out[:3, :3] = Rz @ Ry @ Rx
    out[:3, 3] = d[3:]
    return out


def information(src, tgt, pose, radius):
    """Lambda of one pair: sum G^T G over the source points (moved by pose) whose nearest target point is strictly
    within radius (ties to the lowest index), q that target point."""
    src, tgt = np.asarray(src, np.float64), np.asarray(tgt, np.float64)
    p = np.asarray(pose, np.float64)
    out = np.zeros((6, 6))
    if len(src) == 0 or len(tgt) == 0:
        return out
    s = ((src[:, :1] * p[0, 0] + src[:, 1:2] * p[0, 1]) + src[:, 2:3] * p[0, 2]) + p[0, 3]
    m = [s]
    for r in (1, 2):
        m.append(((src[:, :1] * p[r, 0] + src[:, 1:2] * p[r, 1]) + src[:, 2:3] * p[r, 2]) + p[r, 3])
    moved = np.concatenate(m, 1)
    tree = cKDTree(tgt)
    for i, q in enumerate(moved):
        cand = tree.query_ball_point(q, radius * (1 + 1e-9))
        best, bj = radius * radius, -1
        for j in sorted(cand):
            d = q - tgt[j]
            d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
            if d2 < best:
                best, bj = d2, j
        if bj < 0:
            continue
        x, y, z = tgt[bj]
        G = np.array([[0, z, -y, 1, 0, 0], [-z, 0, x, 0, 1, 0], [y, -x, 0, 0, 0, 1]], np.float64)
        out += G.T @ G
    return out


def edge_terms(P, s, t, X, L):
    """(zeta, J_s) of an edge at poses P (N,4,4)."""
    W = rinv(X) @ rinv(P[t])
    zeta = vec6(W @ P[s])
    J = np.stack([vec6(W @ A @ P[s]) for A in GEN], 1)
    return zeta, J


class Graph:
    def __init__(self, poses, edges, X, info, uncertain):
        self.P = np.stack([h44(p) for p in poses])
        self.edges = np.asarray(edges, np.int64).reshape(-1, 2)
        self.X = np.stack([h44(x) for x in X]) if len(X) else np.zeros((0, 4, 4))
        self.info = np.asarray(info, np.float64).reshape(-1, 6, 6)
        self.unc = np.asarray(uncertain, bool).reshape(-1)


def _system(g, P, conf, active):
    n = 6 * len(P)
    H, b, r = np.zeros((n, n)), np.zeros(n), np.zeros(len(g.edges))
    for e in np.flatnonzero(active):
        s, t = g.edges[e]
        zeta, J = edge_terms(P, s, t, g.X[e], g.info[e])
        L = g.info[e]
        Q = J.T @ L @ J
        q = J.T @ L @ zeta
        r[e] = zeta @ L @ zeta
        c = conf[e]
        for a, sa in ((s, 1.0), (t, -1.0)):
            b[6 * a:6 * a + 6] -= sa * c * q
            for bb, sb in ((s, 1.0), (t, -1.0)):
                H[6 * a:6 * a + 6, 6 * bb:6 * bb + 6] += sa * sb * c * Q
    return H, b, r


def _objective(g, P, conf, active, mu):
    F = 0.0
    for e in np.flatnonzero(active):
        s, t = g.edges[e]
        zeta, _ = edge_terms(P, s, t, g.X[e], g.info[e])
        F += conf[e] * (zeta @ g.info[e] @ zeta) + mu * (np.sqrt(conf[e]) - 1.0) ** 2
    return F


def _lm(g, P, conf, active, mu, o):
    """One LM pass; -> (P, conf, iterations, F, moved)."""
    H, b, r = _system(g, P, conf, active)
    F = _objective(g, P, conf, active, mu)
    n = H.shape[0]
    hmax = H.diagonal().max() if n else 0.0
    moved = False
    if not active.any() or not hmax > 0.0 or np.abs(b).max() < o['min_right_term']:
        return P, conf, 0, F, moved
    lam, nu = 1e-5 * hmax, 2.0
    iters = 0
    for it in range(o['max_iteration']):
        iters = it + 1
        accepted = stop = False
        for _ in range(o['max_iteration_lm']):
            try:
                Lc = np.linalg.cholesky(H + lam * np.eye(n))
                ok = True
            except np.linalg.LinAlgError:
                ok = False
                o['failed_factorisations'] = o.get('failed_factorisations', 0) + 1
            if ok:
                d = np.linalg.solve(Lc.T, np.linalg.solve(Lc, b))
                x = np.concatenate([vec6(p) for p in P])
                if np.linalg.norm(d) < o['min_relative_increment'] * (np.linalg.norm(x) + o['min_relative_increment']):
                    stop = True
                    break
                Pn = np.stack([rt_exp(d[6 * k:6 * k + 6]) @ P[k] for k in range(len(P))])
                Fn = _objective(g, Pn, conf, active, mu)
                rho = (F - Fn) / (d @ (lam * d + b) + 1e-3)
                if rho > 0:
                    P, moved = Pn, True
                    small = abs(F - Fn) < o['min_relative_residual_increment'] * F
                    F = Fn
                    if small:
                        stop = True
                        break
                    H, b, r = _system(g, P, conf, active)
                    if np.abs(b).max() < o['min_right_term']:
                        stop = True
                        break
                    lam *= max(o['lower_scale_factor'], min(o['upper_scale_factor'], 1 - (2 * rho - 1) ** 3))
                    nu = 2.0
                    accepted = True
                    break
            lam *= nu
            nu *= 2.0
        if not accepted or stop:
            break
        conf = conf.copy()
        for e in np.flatnonzero(active & g.unc):
            conf[e] = (mu / (mu + r[e])) ** 2
        H, b, r = _system(g, P, conf, active)
        F = _objective(g, P, conf, active, mu)
        if F < o['min_residual']:
            break
    return P, conf, iters, F, moved


DEFAULTS = dict(edge_prune_threshold=0.25, preference_loop_closure=1.0, reference_node=0, max_iteration=100,
                max_iteration_lm=20, min_relative_increment=1e-6, min_relative_residual_increment=1e-6,
                min_right_term=1e-6, min_residual=1e-6, upper_scale_factor=2.0 / 3.0, lower_scale_factor=1.0 / 3.0)


def optimize(poses, edges, X, info, uncertain, max_correspondence_distance, **kw):
    """-> dict(poses (N,3,4), confidence (E,), kept (E,) bool, result (4,) = it1, it2, F, kept count)."""
    o = dict(DEFAULTS, **kw)
    g = Graph(poses, edges, X, info, uncertain)
    E = len(g.edges)
    P0 = g.P.copy()
    conf = np.ones(E)
    active = np.ones(E, bool)
    pref_d2 = o['preference_loop_closure'] * max_correspondence_distance ** 2

    def mu_of(a):
        return pref_d2 * g.info[a, 5, 5].mean() if a.any() else 0.0

    P, conf, it1, F, m1 = _lm(g, g.P, conf, active, mu_of(active), o)
    active = ~(g.unc & (conf < o['edge_prune_threshold']))
    P, conf, it2, F, m2 = _lm(g, P, conf, active, mu_of(active), o)
    if m1 or m2:
        ref = o['reference_node']
        G = P0[ref] @ rinv(P[ref])
        P = np.stack([P0[ref] if k == ref else G @ P[k] for k in range(len(P))])
    return dict(poses=P[:, :3], confidence=conf, kept=active, result=np.array([it1, it2, F, active.sum()], float),
                failed_factorisations=o.get('failed_factorisations', 0))


def residual_and_jacobian(P, s, t, X):
    """zeta and J_s, J_t of one edge (host self-checks)."""
    zeta, J = edge_terms(np.stack([h44(p) for p in P]), s, t, X, None)
    return zeta, J, -J


def random_pose(rng, deg, trans):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(deg) * rng.uniform(-1, 1)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    out = np.eye(4)
    out[:3, :3] = np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)
    out[:3, 3] = rng.uniform(-trans, trans, 3)
    return out


def info_of_points(pts):
    out = np.zeros((6, 6))
    for x, y, z in pts:
        G = np.array([[0, z, -y, 1, 0, 0], [-z, 0, x, 0, 1, 0], [y, -x, 0, 0, 0, 1]], np.float64)
        out += G.T @ G
    return out


def noisy_graph(seed, N, loop_span=3, all_pairs=False, wrong_frac=0.0, noise_deg=0.3, noise_t=0.005, n_pts=400):
    """A graph on N true poses: odometry edges (j -> j-1) and loop closures (j -> i for 2 <= j - i <= loop_span, or
    every pair), X the true relative pose times small noise; a fraction of the loop closures replaced by gross errors.
    -> dict(truth (N,4,4), init (N,4,4) the odometry chain, edges (E,2), X (E,4,4), info (E,6,6), uncertain, wrong)."""
    rng = np.random.default_rng(seed)
    truth = [np.eye(4)]
    for _ in range(N - 1):
        step = random_pose(rng, 15.0, 0.3)
        truth.append(truth[-1] @ step)
    truth = np.stack(truth)
    edges, X, info, unc, wrong = [], [], [], [], []
    for j in range(1, N):
        for i in range(j):
            if not (j == i + 1 or all_pairs or j - i <= loop_span):
                continue
            rel = rinv(truth[i]) @ truth[j]
            bad = j != i + 1 and rng.random() < wrong_frac
            X.append(random_pose(rng, 40.0, 1.0) @ rel if bad else random_pose(rng, noise_deg, noise_t) @ rel)
            pts = rng.uniform(-1.5, 1.5, (n_pts, 3)) * [1.0, 0.8, 0.6]
            info.append(info_of_points(pts))
            edges.append((j, i)); unc.append(j != i + 1); wrong.append(bad)
    E = np.asarray(edges, np.int64).reshape(-1, 2)
    X = np.stack(X)
    init = [np.eye(4)]
    for j in range(1, N):
        e = [k for k in range(len(E)) if E[k, 0] == j and E[k, 1] == j - 1][0]
        init.append(init[-1] @ X[e])
    return dict(truth=truth, init=np.stack(init), edges=E, X=X, info=np.stack(info), uncertain=np.asarray(unc),
                wrong=np.asarray(wrong))


def pose_error(P, truth):
    """Largest rotation (Frobenius) and translation error of P against truth after aligning node 0."""
    G = h44(truth[0]) @ rinv(P[0])
    Pa = np.stack([G @ h44(p) for p in P])
    return max(np.abs(Pa[:, :3, :3] - truth[:, :3, :3]).max(), np.abs(Pa[:, :3, 3] - truth[:, :3, 3]).max())
