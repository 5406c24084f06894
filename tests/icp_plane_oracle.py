"""Float64 numpy + scipy restatement of normal estimation (`ops.estimate_normals`) and point-to-plane ICP (`ops.icp`
with method='point_to_plane'); not collected: no test_ prefix.

Normals (Open3D's estimate_normals(KDTreeSearchParamHybrid(r, max_nn)) oriented towards the origin, with the library's
tie and boundary rules):

* Neighbours of point i: the points of its cloud with d2 = (dx dx + dy dy) + dz dz strictly below r * r (i itself
  included), the max_nn smallest by (d2, index).  Candidates come from cKDTree.query_ball_point at r * (1 + 1e-9).
* Covariance: the mean of the neighbours, then the centred sum of outer products / count; numpy.linalg.eigh; the
  normal is the eigenvector of the smallest eigenvalue, negated when (nx px + ny py) + nz pz > 0.
* Fewer than 3 neighbours: the zero vector.

Point-to-plane ICP (Open3D's TransformationEstimationPointToPlane): the correspondences, fitness, RMSE and stop test of
tests/icp_oracle.py; each iteration r = (p - q) . n and J = [p x n ; n] per correspondence, the 6x6 normal equations
J^T J x = -J^T r solved by numpy.linalg.solve, the identity when there are no correspondences or |det J^T J| < 1e-6
or det is not finite (SolveLinearSystemPSD), and the update R = Rz(x2) Ry(x1) Rx(x0), t = x[3:].
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from icp_oracle import compose, correspondences, transform


def neighbours(xyz: np.ndarray, r: float, max_nn: int, tree: cKDTree = None):
    """-> (q, j, d2): the neighbour pairs (point q, neighbour j) grouped by q in ascending q and, within q, ascending
    (d2, j), at most max_nn per point."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    n = xyz.shape[0]
    if n == 0:
        e = np.zeros(0, np.int64)
        return e, e, np.zeros(0)
    tree = cKDTree(xyz) if tree is None else tree
    cand = tree.query_ball_point(xyz, r * (1.0 + 1e-9))
    lens = np.fromiter((len(c) for c in cand), np.int64, count=n)
    q = np.repeat(np.arange(n), lens)
    j = np.concatenate([np.asarray(c, np.int64) for c in cand])
    dx, dy, dz = (xyz[q, a] - xyz[j, a] for a in range(3))
    dd = (dx * dx + dy * dy) + dz * dz
    keep = dd < r * r
    q, j, dd = q[keep], j[keep], dd[keep]
    order = np.lexsort((j, dd, q))
    q, j, dd = q[order], j[order], dd[order]
    start = np.searchsorted(q, q, side='left')
    keep = np.arange(q.shape[0]) - start < max_nn
    return q[keep], j[keep], dd[keep]


def estimate_normals(xyz, r: float, max_nn: int = 30, return_eigvals: bool = False):
    """One cloud -> (normals (n,3), counts (n,)) [, eigenvalues (n,3) ascending]."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    n = xyz.shape[0]
    q, j, _ = neighbours(xyz, r, max_nn)
    counts = np.bincount(q, minlength=n)
    normals = np.zeros((n, 3))
    lam = np.zeros((n, 3))
    has = counts > 0
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])[has]
    mean = np.zeros((n, 3))
    mean[has] = np.add.reduceat(xyz[j], start, axis=0) / counts[has, None]
    d = xyz[j] - mean[q]
    cov = np.zeros((n, 3, 3))
    cov[has] = np.add.reduceat(d[:, :, None] * d[:, None, :], start, axis=0) / counts[has, None, None]
    ok = counts >= 3
    if ok.any():
        w, v = np.linalg.eigh(cov[ok])
        nrm = v[:, :, 0]
        p = xyz[ok]
        s = (nrm[:, 0] * p[:, 0] + nrm[:, 1] * p[:, 1]) + nrm[:, 2] * p[:, 2]
        nrm[s > 0] *= -1.0
        normals[ok] = nrm
        lam[ok] = w
    return (normals, counts, lam) if return_eigvals else (normals, counts)


def vec6_to_pose(x) -> np.ndarray:
    """Open3D's TransformVector6dToMatrix4d as a (3,4) transform: R = Rz(x2) Ry(x1) Rx(x0), t = x[3:]."""
    a, b, c = x[0], x[1], x[2]
    rx = np.array([[1.0, 0.0, 0.0], [0.0, np.cos(a), -np.sin(a)], [0.0, np.sin(a), np.cos(a)]])
    ry = np.array([[np.cos(b), 0.0, np.sin(b)], [0.0, 1.0, 0.0], [-np.sin(b), 0.0, np.cos(b)]])
    rz = np.array([[np.cos(c), -np.sin(c), 0.0], [np.sin(c), np.cos(c), 0.0], [0.0, 0.0, 1.0]])
    out = np.empty((3, 4))
    out[:, :3] = rz @ ry @ rx
    out[:, 3] = x[3:6]
    return out


def plane_system(p: np.ndarray, q: np.ndarray, n: np.ndarray):
    """-> (J^T J (6,6), J^T r (6,)) of the correspondences (p moved source, q target, n target normal)."""
    r = ((p[:, 0] - q[:, 0]) * n[:, 0] + (p[:, 1] - q[:, 1]) * n[:, 1]) + (p[:, 2] - q[:, 2]) * n[:, 2]
    J = np.concatenate([np.cross(p, n), n], axis=1)
    return J.T @ J, J.T @ r


def plane_update(p: np.ndarray, q: np.ndarray, n: np.ndarray) -> np.ndarray:
    """TransformationEstimationPointToPlane.ComputeTransformation as a (3,4) transform."""
    if p.shape[0] == 0:
        return np.eye(3, 4)
    jtj, jtr = plane_system(p, q, n)
    det = np.linalg.det(jtj)
    if not np.isfinite(det) or abs(det) < 1e-6:
        return np.eye(3, 4)
    return vec6_to_pose(np.linalg.solve(jtj, -jtr))


def _fit(nn, d2, n_src):
    m = nn >= 0
    k = int(m.sum())
    fitness = k / n_src if n_src else 0.0
    rmse = float(np.sqrt(d2[m].sum() / k)) if k else 0.0
    return fitness, rmse, k


def icp(src, tgt, tgt_normals, init, r: float, max_iteration: int = 30, relative_fitness: float = 1e-6,
        relative_rmse: float = 1e-6):
    """-> dict(pose (3,4), fitness, rmse, k, iterations, nn) for one pair."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    nrm = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
    T = np.asarray(init, np.float64).reshape(3, 4).copy()
    p = transform(T, src)
    tree = cKDTree(tgt) if tgt.shape[0] else None
    nn, d2 = correspondences(p, tgt, r, tree)
    fitness, rmse, k = _fit(nn, d2, src.shape[0])
    it = 0
    for i in range(max_iteration):
        m = nn >= 0
        upd = plane_update(p[m], tgt[nn[m]], nrm[nn[m]])
        T = compose(upd, T)
        p = transform(upd, p)
        it = i + 1
        nn, d2 = correspondences(p, tgt, r, tree)
        prev_f, prev_r = fitness, rmse
        fitness, rmse, k = _fit(nn, d2, src.shape[0])
        if abs(prev_f - fitness) < relative_fitness and abs(prev_r - rmse) < relative_rmse:
            break
    return dict(pose=T, fitness=fitness, rmse=rmse, k=k, iterations=it, nn=nn)


def icp_batch(src_list, tgt_list, normals_list, init, r: float, max_iteration: int = 30,
              relative_fitness: float = 1e-6, relative_rmse: float = 1e-6):
    """`ops.icp`'s layout: -> (pose (B,3,4), result (B,4) = fitness, rmse, k, iterations), float64 numpy."""
    init = np.asarray(init, np.float64).reshape(-1, 3, 4)
    outs = [icp(s, t, nm, p, r, max_iteration, relative_fitness, relative_rmse)
            for s, t, nm, p in zip(src_list, tgt_list, normals_list, init)]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['fitness'], o['rmse'], o['k'], o['iterations']] for o in outs], np.float64).reshape(-1, 4))
