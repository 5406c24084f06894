"""Float64 numpy + scipy restatement of RANSAC over correspondences (`ops.ransac`; not collected: no test_ prefix).

Open3D's registration_ransac_based_on_correspondence(source, target, corres, max_correspondence_distance,
TransformationEstimationPointToPoint(False), ransac_n, [CorrespondenceCheckerBasedOnEdgeLength(edge_length),
CorrespondenceCheckerBasedOnDistance(distance)], RANSACConvergenceCriteria(max_iteration, confidence)), with one
deterministic sequential rule in place of Open3D's OpenMP schedule, whose results cannot be reproduced:

* Correspondences (a_i, c_i) are coordinates (Open3D's index form: a = src[corres[:,0]], c = tgt[corres[:,1]]); the
  valid ones (mask) in their original order are 0..n-1.  ransac_n < 3, n < ransac_n or a radius that is not positive:
  Open3D's empty result (identity, fitness 0, rmse 0, 0 hypotheses walked and validated, winner -1).
* Hypothesis k draws index j < ransac_n as mulhi32(w, n), w word j & 3 of Philox4x32-10 at counter
  (k, pair, j >> 2, 0x52534143) with key (seed lo, seed hi), pair = pair_base + b: with replacement, as Open3D's
  rand_gen(), and the same whatever the batch or the chunking.
* Estimation: `icp_oracle.umeyama` on the sample (means, cross-covariance / n, SVD, reflection fix,
  t = mean_c - R mean_a).
* Deliberate deviation 1: a sample with a repeated index, or whose cross-covariance has singular values
  S[1] <= 1e-12 S[0], is rejected like a failed checker (in Open3D its outcome depends on Eigen's SVD of a
  rank-deficient matrix).
* Checkers in Open3D's order after the estimation, each off at 0 or None: edge length s rejects when, for a pair
  i < j of the sample, |a_i - a_j| < |c_i - c_j| s or |c_i - c_j| < |a_i - a_j| s; distance d rejects when
  |T a_i - c_i| > d for a sample point.  Norms are sqrt((dx dx + dy dy) + dz dz).
* Validation: the whole source moved by T (`icp_oracle.transform`), `icp_oracle.correspondences` (nearest target with
  d2 strictly below r^2, lowest index on ties), fitness = k / n_src, inlier_rmse = sqrt(sum d2 / k), the sum in the
  device's order (`fixed_sum`).  Every validated hypothesis counts one validation.
* Walk k = 0, 1, ... while k < est_k, est_k = max_iteration at first.  A result is better when its fitness is higher,
  or equal with a lower rmse (IsBetterRANSACThan); the best starts at fitness 0, rmse 0, identity.  On every
  improvement d = log(1 - confidence) / log(1 - fitness^ransac_n) (the power as ransac_n - 1 products) sets
  est_k = ceil(d) when d < est_k.  Deliberate deviation 2: d = -inf (a fitness so small that 1 - fitness^n rounds to
  1; Open3D's int cast of ceil(-inf) is undefined) leaves est_k alone, so the rule applies for 0 <= d < est_k only.
  No final refit on the inliers, as in Open3D.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.spatial import cKDTree

import icp_oracle as I
from dropout_rule import philox

WORD3 = 0x52534143
BLOCK = 1024                 # source points per validation block
CHAIN = 256                  # per-block chains, as regtr_registration_fit sums a cloud
LANES = 32                   # chains over the blocks


def draws(seed: int, pair: int, ks, n: int, ransac_n: int) -> np.ndarray:
    """(len(ks), ransac_n) int64 sample indices of hypotheses ks of global pair `pair` out of n valid ones."""
    ks = np.asarray(ks, np.uint64).reshape(-1, 1)
    out = np.empty((ks.shape[0], ransac_n), np.int64)
    for g in range((ransac_n + 3) // 4):
        w = philox((ks, pair, g, WORD3), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        for e in range(4):
            j = 4 * g + e
            if j < ransac_n:
                out[:, j] = ((w[e][:, 0] * np.uint64(n)) >> np.uint64(32)).astype(np.int64)
    return out


def norm3(d: np.ndarray) -> np.ndarray:
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def edge_ok(a: np.ndarray, c: np.ndarray, s) -> bool:
    """CorrespondenceCheckerBasedOnEdgeLength(s) on the sample rows a, c (always true when off)."""
    if not s:
        return True
    for i in range(a.shape[0]):
        for j in range(i + 1, a.shape[0]):
            da, dc = float(norm3(a[i] - a[j])), float(norm3(c[i] - c[j]))
            if da < dc * s or dc < da * s:
                return False
    return True


def distance_ok(T: np.ndarray, a: np.ndarray, c: np.ndarray, d) -> bool:
    """CorrespondenceCheckerBasedOnDistance(d) on the sample rows (always true when off)."""
    if not d:
        return True
    return not bool(np.any(norm3(I.transform(T, a) - c) > d))


def degenerate(a: np.ndarray, c: np.ndarray) -> bool:
    """Deviation 1's singular-value test of the sample's cross-covariance."""
    sigma = (c - c.mean(axis=0)).T @ (a - a.mean(axis=0)) / a.shape[0]
    S = np.linalg.svd(sigma, compute_uv=False)
    return not S[1] > 1e-12 * S[0]


def hypothesis(a: np.ndarray, c: np.ndarray, idx, edge_length=None, distance=None):
    """-> (accepted, T (3,4)) for the sample idx of the valid correspondences a, c."""
    idx = np.asarray(idx, np.int64)
    if len(set(idx.tolist())) != idx.shape[0]:
        return False, None
    sa, sc = a[idx], c[idx]
    if not edge_ok(sa, sc, edge_length):
        return False, None
    if degenerate(sa, sc):
        return False, None
    T = I.umeyama(sa, sc)
    if not distance_ok(T, sa, sc, distance):
        return False, None
    return True, T


def _tree(v: np.ndarray) -> float:
    v = v.copy()
    h = v.shape[0] // 2
    while h:
        v[:h] = v[:h] + v[h:2 * h]
        h //= 2
    return float(v[0])


def _chains(v: np.ndarray, width: int) -> np.ndarray:
    """Element i added to chain i % width, in ascending order."""
    pad = np.zeros((-v.shape[0]) % width)
    rows = np.concatenate([v, pad]).reshape(-1, width)
    acc = np.zeros(width)
    for r in rows:
        acc = acc + r
    return acc


def fixed_sum(d2: np.ndarray) -> float:
    """The device's order of sum d2 (0 for unmatched points): blocks of BLOCK points, each by CHAIN chains and a
    halving tree; the block sums by LANES chains and a halving tree."""
    nb = (d2.shape[0] + BLOCK - 1) // BLOCK
    if nb == 0:
        return 0.0
    parts = np.array([_tree(_chains(d2[j * BLOCK:(j + 1) * BLOCK], CHAIN)) for j in range(nb)])
    return _tree(_chains(parts, LANES))


def matches(p: np.ndarray, tgt: np.ndarray, r: float, tree: cKDTree = None, k: int = 8):
    """`icp_oracle.correspondences` (same rule, same result) through the k nearest candidates of cKDTree.query;
    a point whose k-th candidate is still a contender falls back to icp_oracle's ball query."""
    n = p.shape[0]
    if n == 0 or tgt.shape[0] == 0:
        return I.correspondences(p, tgt, r, tree)
    tree = cKDTree(tgt) if tree is None else tree
    k = min(k, tgt.shape[0])
    _, j = tree.query(p, k=k, distance_upper_bound=r * (1.0 + 1e-9))
    j = j.reshape(n, k)
    ok = j < tgt.shape[0]
    js = np.where(ok, j, 0)
    d = p[:, None, :] - tgt[js]
    dd = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    dd = np.where(ok & (dd < r * r), dd, np.inf)
    key = np.where(np.isfinite(dd), js, np.iinfo(np.int64).max)
    order = np.lexsort((key, dd), axis=1)[:, 0]
    rows = np.arange(n)
    best, bj = dd[rows, order], js[rows, order]
    nn = np.where(np.isfinite(best), bj, -1).astype(np.int64)
    d2 = best.copy()
    unsure = ok[:, -1] & np.isfinite(dd[:, -1]) & (dd[:, -1] <= best * (1.0 + 1e-9))
    if unsure.any():
        nu, du = I.correspondences(p[unsure], tgt, r, tree)
        nn[unsure], d2[unsure] = nu, du
    return nn, d2


def validate(src: np.ndarray, tgt: np.ndarray, T: np.ndarray, r: float, tree=None):
    """-> (fitness, rmse, k) of the source moved by T."""
    nn, d2 = matches(I.transform(T, src), tgt, r, tree)
    m = nn >= 0
    k = int(m.sum())
    fitness = k / src.shape[0] if src.shape[0] else 0.0
    rmse = math.sqrt(fixed_sum(np.where(m, d2, 0.0)) / k) if k else 0.0
    return fitness, rmse, k


def est_k_update(est_k: int, fitness: float, confidence: float, ransac_n: int) -> int:
    """The stop rule after an improvement (deviation 2 included)."""
    pw = fitness
    for _ in range(ransac_n - 1):
        pw = pw * fitness
    with np.errstate(divide='ignore', invalid='ignore'):
        d = float(np.float64(np.log(1.0 - confidence)) / np.float64(np.log(1.0 - pw)))
    if d >= 0.0 and d < est_k:
        return int(math.ceil(d))
    return est_k


def better(fit, rmse, best_fit, best_rmse) -> bool:
    return fit > best_fit or (fit == best_fit and rmse < best_rmse)


def empty_result():
    return dict(pose=np.eye(3, 4), fitness=0.0, rmse=0.0, iterations=0, validations=0, best=-1, k=0)


def ransac(src, tgt, corr_src, corr_tgt, r: float, max_iteration: int = 100000, confidence: float = 0.999,
           ransac_n: int = 3, edge_length=0.9, distance=None, mask=None, seed: int = 0, pair: int = 0):
    """-> dict(pose (3,4), fitness, rmse, iterations, validations, best, k) for one pair (global index `pair`)."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    a = np.asarray(corr_src, np.float64).reshape(-1, 3)
    c = np.asarray(corr_tgt, np.float64).reshape(-1, 3)
    if mask is not None:
        keep = np.asarray(mask, bool)
        a, c = a[keep], c[keep]
    n = a.shape[0]
    if ransac_n < 3 or n < ransac_n or not r > 0.0:
        return empty_result()
    tree = cKDTree(tgt) if tgt.shape[0] else None
    best = empty_result()
    est_k, k, vals = max_iteration, 0, 0
    batch = 1024
    while k < est_k:
        idx = draws(seed, pair, np.arange(k, k + batch), n, ransac_n)
        for row in idx:
            if k >= est_k:
                break
            ok, T = hypothesis(a, c, row, edge_length, distance)
            if ok:
                fit, rmse, kk = validate(src, tgt, T, r, tree)
                vals += 1
                if better(fit, rmse, best['fitness'], best['rmse']):
                    best.update(pose=T, fitness=fit, rmse=rmse, best=k, k=kk)
                    est_k = est_k_update(est_k, fit, confidence, ransac_n)
            k += 1
    best.update(iterations=k, validations=vals)
    return best


def ransac_batch(src_list, tgt_list, corr_src, corr_tgt, r: float, max_iteration: int = 100000,
                 confidence: float = 0.999, ransac_n: int = 3, edge_length=0.9, distance=None, corr_mask=None,
                 seed: int = 0, pair_base: int = 0):
    """`ops.ransac`'s layout: -> (pose (B,3,4), result (B,5) = fitness, rmse, walked, validated, winner), float64."""
    outs = [ransac(s, t, a, c, r, max_iteration, confidence, ransac_n, edge_length, distance,
                   None if corr_mask is None else corr_mask[b], seed, pair_base + b)
            for b, (s, t, a, c) in enumerate(zip(src_list, tgt_list, corr_src, corr_tgt))]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['fitness'], o['rmse'], o['iterations'], o['validations'], o['best']] for o in outs],
                     np.float64).reshape(-1, 5))
