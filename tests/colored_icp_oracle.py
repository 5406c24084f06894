"""Float64 numpy restatement of colour gradients (`ops.color_gradients`) and colored ICP (`ops.icp` with
method='colored'); not collected: no test_ prefix.

Gradients (Open3D's InitializePointCloudForColoredICP with KDTreeSearchParamHybrid(r, max_nn)):

* Neighbours of point p: those of tests/icp_plane_oracle.py's normal estimation (own cloud, d2 strictly below r * r,
  p included, the max_nn smallest by (d2, index)), nn of them.  Intensity it = ((r + g) + b) / 3.
* Gradient 0 when nn < 4 or p's normal n is zero.  Otherwise A has rows v_i - p (v_i = q_i - ((q_i - p) . n) n) for the
  entries i >= 1, then (nn - 1) n; b has it_i - it_p, then 0.  (A^T A) x = A^T b by numpy.linalg.solve, the gradient 0
  when |det A^T A| < 1e-6 or det is not finite (SolveLinearSystemPSD).

Colored ICP (Open3D's TransformationEstimationForColoredICP(lambda_geometric, kernel)): the correspondences, fitness,
RMSE, stop test and update of tests/gicp_oracle.py's point-to-plane; per correspondence with a non-zero target normal n
(p moved source, q target, d the target's gradient, l = lambda_geometric) the geometric row r = sqrt(l) (p - q) . n,
J = [p x sqrt(l) n ; sqrt(l) n] and the photometric row, with p' = p - ((p - q) . n) n, is0 = d . (p' - q) + it_q and
m = (d . n) n - d: r = sqrt(1 - l) (is_p - is0), J = [p x sqrt(1 - l) m ; sqrt(1 - l) m]; each row weighted by the
robust kernel of its own r.

`texture` is the procedural colouring of the tests: no coloured scan exists among the fixtures, so a cloud is coloured
by a smooth function of world position, evaluated after moving it by its ground-truth pose, so that both clouds of a
pair agree where they overlap.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

from gicp_oracle import _fit, solve_update, weight
from icp_oracle import compose, correspondences, transform
from icp_plane_oracle import neighbours


def texture(world: np.ndarray, scale: float = 1.0) -> np.ndarray:
    """Smooth rgb in [0, 1] of world positions (n,3): three sinusoids of different directions and wavelengths (about
    0.3 to 0.5 m at scale 1)."""
    w = np.asarray(world, np.float64).reshape(-1, 3) / scale
    r = 0.5 + 0.4 * np.sin(13.0 * w[:, 0] + 7.0 * w[:, 1] + 1.0)
    g = 0.5 + 0.4 * np.sin(11.0 * w[:, 1] - 9.0 * w[:, 2] + 2.0)
    b = 0.5 + 0.4 * np.sin(17.0 * w[:, 2] + 5.0 * w[:, 0] + 3.0)
    return np.stack([r, g, b], axis=1)


def colour_pair(src, tgt, pose, scale: float = 1.0):
    """-> (src_rgb, tgt_rgb): `texture` of the target as it lies and of the source moved by its ground-truth pose
    (3,4) source -> target."""
    return texture(transform(np.asarray(pose, np.float64), np.asarray(src, np.float64)), scale), texture(tgt, scale)


def intensity(rgb) -> np.ndarray:
    c = np.asarray(rgb, np.float64).reshape(-1, 3)
    return ((c[:, 0] + c[:, 1]) + c[:, 2]) / 3.0


def color_gradients(xyz, normals, rgb, r: float, max_nn: int = 30) -> np.ndarray:
    """One cloud -> gradients (n,3)."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    nrm = np.asarray(normals, np.float64).reshape(-1, 3)
    it = intensity(rgb)
    n = xyz.shape[0]
    q, j, _ = neighbours(xyz, r, max_nn)
    counts = np.bincount(q, minlength=n)
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    out = np.zeros((n, 3))
    for p in np.nonzero((counts >= 4) & nrm.any(axis=1))[0]:
        nb = j[start[p] + 1:start[p] + counts[p]]
        v, c = xyz[p], nrm[p]
        qs = xyz[nb]
        d = ((qs[:, 0] - v[0]) * c[0] + (qs[:, 1] - v[1]) * c[1]) + (qs[:, 2] - v[2]) * c[2]
        A = np.concatenate([(qs - d[:, None] * c[None, :]) - v[None, :], (counts[p] - 1.0) * c[None, :]], axis=0)
        b = np.concatenate([it[nb] - it[p], [0.0]])
        ata, atb = A.T @ A, A.T @ b
        det = np.linalg.det(ata)
        if np.isfinite(det) and abs(det) >= 1e-6:
            out[p] = np.linalg.solve(ata, atb)
    return out


def _accumulate(p, rows, res, w):
    J = np.concatenate([np.cross(p, rows), rows], axis=1)
    Jw = J * w[:, None]
    return Jw.T @ J, Jw.T @ res


def colored_system(p, q, n, grad, it_q, is_p, lambda_geometric=0.968, loss='l2', k=None):
    """-> (J^T J (6,6), J^T r (6,)) of colored ICP's correspondences (p moved source, q target, n target normal,
    grad its gradient, it_q its intensity, is_p the source's intensity)."""
    keep = n.any(axis=1)
    p, q, n, grad, it_q, is_p = p[keep], q[keep], n[keep], grad[keep], it_q[keep], is_p[keep]
    sl, sp = np.sqrt(lambda_geometric), np.sqrt(1.0 - lambda_geometric)
    g = ((p[:, 0] - q[:, 0]) * n[:, 0] + (p[:, 1] - q[:, 1]) * n[:, 1]) + (p[:, 2] - q[:, 2]) * n[:, 2]
    rg = sl * g
    jtj, jtr = _accumulate(p, sl * n, rg, weight(loss, k, rg))
    u = (p - g[:, None] * n) - q
    is0 = ((grad[:, 0] * u[:, 0] + grad[:, 1] * u[:, 1]) + grad[:, 2] * u[:, 2]) + it_q
    dn = (grad[:, 0] * n[:, 0] + grad[:, 1] * n[:, 1]) + grad[:, 2] * n[:, 2]
    m = dn[:, None] * n - grad
    ri = sp * (is_p - is0)
    h, v = _accumulate(p, sp * m, ri, weight(loss, k, ri))
    return jtj + h, jtr + v


def icp(src, tgt, tgt_normals, src_colors, tgt_colors, tgt_grad, init, r: float, max_iteration: int = 30,
        relative_fitness: float = 1e-6, relative_rmse: float = 1e-6, lambda_geometric: float = 0.968,
        loss: str = 'l2', loss_k: float = None, trace: list = None):
    """-> dict(pose (3,4), fitness, rmse, k, iterations, nn) for one pair.  trace: a list that receives
    (pose, fitness, rmse, k) after every round, round 0 (the initial pose) first."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    nt = np.asarray(tgt_normals, np.float64).reshape(-1, 3)
    gt = np.asarray(tgt_grad, np.float64).reshape(-1, 3)
    is_ = intensity(src_colors)
    it_ = intensity(tgt_colors)
    T = np.asarray(init, np.float64).reshape(3, 4).copy()
    p = transform(T, src)
    tree = cKDTree(tgt) if tgt.shape[0] else None
    nn, d2 = correspondences(p, tgt, r, tree)
    fitness, rmse, k = _fit(nn, d2, src.shape[0])
    if trace is not None:
        trace.append((T.copy(), fitness, rmse, k))
    it = 0
    for i in range(max_iteration):
        m = nn >= 0
        j = nn[m]
        jtj, jtr = colored_system(p[m], tgt[j], nt[j], gt[j], it_[j], is_[m], lambda_geometric, loss, loss_k)
        upd = solve_update(jtj, jtr, int(m.sum()))
        T = compose(upd, T)
        p = transform(upd, p)
        it = i + 1
        nn, d2 = correspondences(p, tgt, r, tree)
        prev_f, prev_r = fitness, rmse
        fitness, rmse, k = _fit(nn, d2, src.shape[0])
        if trace is not None:
            trace.append((T.copy(), fitness, rmse, k))
        if abs(prev_f - fitness) < relative_fitness and abs(prev_r - rmse) < relative_rmse:
            break
    return dict(pose=T, fitness=fitness, rmse=rmse, k=k, iterations=it, nn=nn)


def icp_batch(src_list, tgt_list, normals_list, src_colors, tgt_colors, grad_list, init, r: float,
              max_iteration: int = 30, relative_fitness: float = 1e-6, relative_rmse: float = 1e-6,
              lambda_geometric: float = 0.968, loss: str = 'l2', loss_k: float = None):
    """`ops.icp`'s layout: -> (pose (B,3,4), result (B,4) = fitness, rmse, k, iterations), float64 numpy."""
    init = np.asarray(init, np.float64).reshape(-1, 3, 4)
    outs = [icp(s, t, nm, sc, tc, g, p, r, max_iteration, relative_fitness, relative_rmse, lambda_geometric, loss,
                loss_k)
            for s, t, nm, sc, tc, g, p in zip(src_list, tgt_list, normals_list, src_colors, tgt_colors, grad_list,
                                              init)]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['fitness'], o['rmse'], o['k'], o['iterations']] for o in outs], np.float64).reshape(-1, 4))
