"""Float64 numpy restatement of generalized ICP and of robust point-to-plane ICP (`ops.icp` with
method='generalized', or with a loss other than 'l2'); not collected: no test_ prefix.

Correspondences, fitness, RMSE, the stop test, the 6x6 solve (the identity without correspondences or when
|det J^T J| < 1e-6 or det is not finite) and the update R = Rz(x2) Ry(x1) Rx(x0), t = x[3:] are those of
tests/icp_oracle.py and tests/icp_plane_oracle.py.

Robust kernels (Open3D's RobustKernel::Weight of residual r with parameter k): l2 1; huber 1 if |r| <= k else k / |r|;
cauchy 1 / (1 + (r/k)^2); gm k / (k + r^2)^2; tukey (1 - (r/k)^2)^2 if |r| <= k else 0.

Point-to-plane under a kernel: r = (p - q) . n, J = [p x n ; n], J^T J += w(r) J J^T, J^T r += w(r) J r.

Generalized ICP (TransformationEstimationForGeneralizedICP(epsilon, kernel)): a the moved source normal (the caller's
normal rotated by init, then by every update), b the target normal, Cs = I - (1 - eps) a a^T, Ct = I - (1 - eps) b b^T,
M = Cs + Ct; numpy.linalg.eigh(M) = (lam, Q) and W = Q diag(1 / sqrt(lam)) Q^T; a correspondence with an eigenvalue
that is not > 0 or not finite leaves the update (not k).  The rows w_i of W give r_i = w_i . (p - q) and
J_i = W_i [-[p]x | I] = [p x w_i ; w_i], each with weight w(r_i).
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from icp_oracle import compose, correspondences, transform
from icp_plane_oracle import _fit, vec6_to_pose

LOSSES = ('l2', 'huber', 'cauchy', 'gm', 'tukey')


def weight(loss: str, k, r) -> np.ndarray:
    """Open3D's RobustKernel::Weight, elementwise."""
    r = np.asarray(r, np.float64)
    if loss == 'l2':
        return np.ones_like(r)
    if loss == 'huber':
        a = np.abs(r)
        return np.where(a <= k, 1.0, k / np.where(a > 0, a, 1.0))
    if loss == 'cauchy':
        return 1.0 / (1.0 + (r / k) ** 2)
    if loss == 'gm':
        return k / (k + r * r) ** 2
    if loss == 'tukey':
        return np.where(np.abs(r) <= k, (1.0 - (r / k) ** 2) ** 2, 0.0)
    raise ValueError(loss)


def covariance(n, epsilon: float) -> np.ndarray:
    """(m,3) normals -> (m,3,3) I - (1 - eps) n n^T."""
    n = np.asarray(n, np.float64).reshape(-1, 3)
    return np.eye(3)[None] - (1.0 - epsilon) * n[:, :, None] * n[:, None, :]


def information_sqrt(M):
    """(m,3,3) symmetric -> (W (m,3,3) = M^-1/2 by eigh, ok (m,) every eigenvalue > 0 and finite)."""
    M = np.asarray(M, np.float64).reshape(-1, 3, 3)
    W = np.zeros_like(M)
    fin = np.isfinite(M).all(axis=(1, 2))
    ok = np.zeros(M.shape[0], bool)
    if fin.any():
        lam, Q = np.linalg.eigh(M[fin])
        good = (lam > 0).all(axis=1) & np.isfinite(lam).all(axis=1)
        idx = np.nonzero(fin)[0][good]
        lam, Q = lam[good], Q[good]
        W[idx] = np.einsum('mij,mj,mkj->mik', Q, 1.0 / np.sqrt(lam), Q)
        ok[idx] = True
    return W, ok


def _accumulate(p, rows, res, w):
    """Rows (m,3) normals-like vectors with residuals res (m,) and weights w (m,) -> (J^T J, J^T r)."""
    J = np.concatenate([np.cross(p, rows), rows], axis=1)
    Jw = J * w[:, None]
    return Jw.T @ J, Jw.T @ res


def plane_system(p, q, n, loss='l2', k=None):
    r = ((p[:, 0] - q[:, 0]) * n[:, 0] + (p[:, 1] - q[:, 1]) * n[:, 1]) + (p[:, 2] - q[:, 2]) * n[:, 2]
    return _accumulate(p, n, r, weight(loss, k, r))


def gicp_system(p, q, a, b, epsilon=1e-3, loss='l2', k=None):
    """-> (J^T J (6,6), J^T r (6,)) of generalized ICP's correspondences (p moved source, q target, a moved source
    normal, b target normal)."""
    W, ok = information_sqrt(covariance(a, epsilon) + covariance(b, epsilon))
    p, q, W = p[ok], q[ok], W[ok]
    d = p - q
    jtj, jtr = np.zeros((6, 6)), np.zeros(6)
    for i in range(3):
        rows = W[:, i, :]
        r = (rows * d).sum(axis=1)
        h, v = _accumulate(p, rows, r, weight(loss, k, r))
        jtj += h
        jtr += v
    return jtj, jtr


def solve_update(jtj, jtr, k: int) -> np.ndarray:
    """SolveLinearSystemPSD and TransformVector6dToMatrix4d: (3,4)."""
    if k == 0:
        return np.eye(3, 4)
    det = np.linalg.det(jtj)
    if not np.isfinite(det) or abs(det) < 1e-6:
        return np.eye(3, 4)
    return vec6_to_pose(np.linalg.solve(jtj, -jtr))


def rotate(m, n):
    """Normals (m,3) by the rotation of the (3,4) transform m."""
    r = np.zeros((3, 4))
    r[:, :3] = np.asarray(m)[:, :3]
    return transform(r, n)


def icp(src, tgt, tgt_normals, init, r: float, max_iteration: int = 30, relative_fitness: float = 1e-6,
        relative_rmse: float = 1e-6, method: str = 'generalized', src_normals=None, epsilon: float = 1e-3,
        loss: str = 'l2', loss_k: float = None):
    """-> dict(pose (3,4), fitness, rmse, k, iterations, nn) for one pair; method 'generalized' or
    'point_to_plane'."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    nt = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
    T = np.asarray(init, np.float64).reshape(3, 4).copy()
    p = transform(T, src)
    a = rotate(T, np.asarray(src_normals, np.float64).reshape(-1, 3)) if method == 'generalized' else None
    tree = cKDTree(tgt) if tgt.shape[0] else None
    nn, d2 = correspondences(p, tgt, r, tree)
    fitness, rmse, k = _fit(nn, d2, src.shape[0])
    it = 0
    for i in range(max_iteration):
        m = nn >= 0
        if method == 'generalized':
            jtj, jtr = gicp_system(p[m], tgt[nn[m]], a[m], nt[nn[m]], epsilon, loss, loss_k)
        else:
            jtj, jtr = plane_system(p[m], tgt[nn[m]], nt[nn[m]], loss, loss_k)
        upd = solve_update(jtj, jtr, int(m.sum()))
        T = compose(upd, T)
        p = transform(upd, p)
        if a is not None:
            a = rotate(upd, a)
        it = i + 1
        nn, d2 = correspondences(p, tgt, r, tree)
        prev_f, prev_r = fitness, rmse
        fitness, rmse, k = _fit(nn, d2, src.shape[0])
        if abs(prev_f - fitness) < relative_fitness and abs(prev_r - rmse) < relative_rmse:
            break
    return dict(pose=T, fitness=fitness, rmse=rmse, k=k, iterations=it, nn=nn)


def icp_batch(src_list, tgt_list, normals_list, init, r: float, max_iteration: int = 30,
              relative_fitness: float = 1e-6, relative_rmse: float = 1e-6, method: str = 'generalized',
              src_normals_list=None, epsilon: float = 1e-3, loss: str = 'l2', loss_k: float = None):
    """`ops.icp`'s layout: -> (pose (B,3,4), result (B,4) = fitness, rmse, k, iterations), float64 numpy."""
    init = np.asarray(init, np.float64).reshape(-1, 3, 4)
    sn = src_normals_list if src_normals_list is not None else [None] * len(src_list)
    outs = [icp(s, t, nm, p, r, max_iteration, relative_fitness, relative_rmse, method, a, epsilon, loss, loss_k)
            for s, t, nm, p, a in zip(src_list, tgt_list, normals_list, init, sn)]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['fitness'], o['rmse'], o['k'], o['iterations']] for o in outs], np.float64).reshape(-1, 4))
