"""Float64 numpy + scipy restatement of point-to-point ICP (`ops.icp`; not collected: no test_ prefix).

Open3D's registration_icp with TransformationEstimationPointToPoint(with_scaling=False) and
ICPConvergenceCriteria(relative_fitness, relative_rmse, max_iteration), with the library's determinism rules:

* P = init . source, each coordinate ((r0 x + r1 y) + r2 z) + t; T = init.
* Correspondences: for every point of P the nearest target point with squared distance ((dx dx + dy dy) + dz dz)
  strictly below r * r, the lowest target index on equal distances.  Candidates come from cKDTree.query_ball_point at
  r * (1 + 1e-9); the winner is then picked by that squared distance and that rule.
  fitness = k / n_src, inlier_rmse = sqrt(sum d2 / k), both 0 with k = 0.
* Each iteration: Eigen's umeyama without scaling on the correspondences (means, cross-covariance of the demeaned
  points / k, numpy.linalg.svd, the reflection fix when det(U) det(V) < 0, R = U S V^T, t = mean_tgt - R mean_src;
  the identity with k = 0), T = update . T, P moved by the update in place, re-match; stop when
  |d fitness| < relative_fitness and |d rmse| < relative_rmse.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


def transform(m: np.ndarray, p: np.ndarray) -> np.ndarray:
    """(3,4) m applied to (n,3) p in the kernel's operation order."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((m[a, 0] * x + m[a, 1] * y) + m[a, 2] * z) + m[a, 3] for a in range(3)], axis=1)


def compose(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """a . b as rigid (3,4) transforms, in the kernel's operation order."""
    out = np.empty((3, 4))
    for i in range(3):
        for j in range(4):
            s = (a[i, 0] * b[0, j] + a[i, 1] * b[1, j]) + a[i, 2] * b[2, j]
            out[i, j] = s + a[i, 3] if j == 3 else s
    return out


def correspondences(p: np.ndarray, tgt: np.ndarray, r: float, tree: cKDTree = None):
    """-> nn (n,) int64 (target index or -1), d2 (n,) float64 (inf where unmatched)."""
    n = p.shape[0]
    nn = np.full(n, -1, np.int64)
    d2 = np.full(n, np.inf)
    if n == 0 or tgt.shape[0] == 0:
        return nn, d2
    tree = cKDTree(tgt) if tree is None else tree
    cand = tree.query_ball_point(p, r * (1.0 + 1e-9))
    lens = np.fromiter((len(c) for c in cand), np.int64, count=n)
    if lens.sum() == 0:
        return nn, d2
    q = np.repeat(np.arange(n), lens)
    j = np.concatenate([np.asarray(c, np.int64) for c in cand if len(c)])
    dx, dy, dz = (p[q, a] - tgt[j, a] for a in range(3))
    dd = (dx * dx + dy * dy) + dz * dz
    keep = dd < r * r
    q, j, dd = q[keep], j[keep], dd[keep]
    order = np.lexsort((j, dd, q))                  # per query: smallest d2, then lowest index
    q, j, dd = q[order], j[order], dd[order]
    first = np.ones(q.shape[0], bool)
    first[1:] = q[1:] != q[:-1]
    nn[q[first]] = j[first]
    d2[q[first]] = dd[first]
    return nn, d2


def _fit(nn, d2, n_src):
    m = nn >= 0
    k = int(m.sum())
    fitness = k / n_src if n_src else 0.0
    rmse = float(np.sqrt(d2[m].sum() / k)) if k else 0.0
    return fitness, rmse, k


def umeyama(src: np.ndarray, dst: np.ndarray) -> np.ndarray:
    """Eigen::umeyama(src^T, dst^T, false) as a (3,4) transform; the identity without points."""
    if src.shape[0] == 0:
        return np.eye(3, 4)
    ms, md = src.mean(axis=0), dst.mean(axis=0)
    sigma = (dst - md).T @ (src - ms) / src.shape[0]
    u, _, vt = np.linalg.svd(sigma)
    s = np.eye(3)
    if np.linalg.det(u) * np.linalg.det(vt) < 0:
        s[2, 2] = -1.0
    rot = u @ s @ vt
    out = np.empty((3, 4))
    out[:, :3] = rot
    out[:, 3] = md - rot @ ms
    return out


def icp(src, tgt, init, r: float, max_iteration: int = 30, relative_fitness: float = 1e-6,
        relative_rmse: float = 1e-6):
    """-> dict(pose (3,4), fitness, rmse, k, iterations, nn) for one pair."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    T = np.asarray(init, np.float64).reshape(3, 4).copy()
    p = transform(T, src)
    tree = cKDTree(tgt) if tgt.shape[0] else None
    nn, d2 = correspondences(p, tgt, r, tree)
    fitness, rmse, k = _fit(nn, d2, src.shape[0])
    it = 0
    for i in range(max_iteration):
        m = nn >= 0
        upd = umeyama(p[m], tgt[nn[m]])
        T = compose(upd, T)
        p = transform(upd, p)
        it = i + 1
        nn, d2 = correspondences(p, tgt, r, tree)
        prev_f, prev_r = fitness, rmse
        fitness, rmse, k = _fit(nn, d2, src.shape[0])
        if abs(prev_f - fitness) < relative_fitness and abs(prev_r - rmse) < relative_rmse:
            break
    return dict(pose=T, fitness=fitness, rmse=rmse, k=k, iterations=it, nn=nn)


def icp_batch(src_list, tgt_list, init, r: float, max_iteration: int = 30, relative_fitness: float = 1e-6,
              relative_rmse: float = 1e-6):
    """`ops.icp`'s layout: -> (pose (B,3,4), result (B,4) = fitness, rmse, k, iterations), float64 numpy."""
    init = np.asarray(init, np.float64).reshape(-1, 3, 4)
    outs = [icp(s, t, p, r, max_iteration, relative_fitness, relative_rmse) for s, t, p in zip(src_list, tgt_list, init)]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['fitness'], o['rmse'], o['k'], o['iterations']] for o in outs], np.float64).reshape(-1, 4))
