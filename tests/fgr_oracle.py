"""Float64 numpy restatement of Fast Global Registration (`ops.fgr`, `ops.fgr_feature_matching`; not collected: no
test_ prefix).

Open3D's registration_fgr_based_on_correspondence / registration_fgr_based_on_feature_matching with
FastGlobalRegistrationOption (Zhou, Park and Koltun, ECCV 2016), restated as one deterministic rule.  Per pair b, with
global index pair = pair_base + b:

1. Correspondences (a_i, c_i) are coordinates in their original order; masked-out ones are dropped, leaving n.  The
   feature-matching variant uses the mutual matches of `fpfh_oracle.feature_match` (no fallback: min_mutual 0) in
   source-index order: source point i -> target point nn[i].
2. Normalisation over the whole clouds: mu_s, mu_t the clouds' means, each sum in the device's fixed order
   (`block_sum` with PREP_THREADS chains) divided by the point count (0 for an empty cloud); sigma the largest
   |p - mu| over both clouds.  use_absolute_scale: sigma_g = 1, par0 = sigma; otherwise sigma_g = sigma, par0 = 1.
   Points are used as (p - mu) / sigma_g, component by component.
3. Tuple test (tuple_test and n > 0): trials k = 0, 1, ... < 100 n in order; trial k draws indices mulhi32(w_e, n),
   e = 0, 1, 2, w the words of Philox4x32-10 at counter (k, pair, 0, 0x46475254) with key (seed lo, seed hi), with
   replacement.  It passes when, for the edges (0,1), (1,2), (2,0) of the normalised points,
   l_s tuple_scale < l_t and l_t < l_s / tuple_scale.  A pass appends its three correspondences in draw order; the
   walk stops right after the pass that brings the tuple count to maximum_tuple_count.  The correspondence set
   becomes the 3 x tuples list, duplicates included.  Without the test, the n correspondences are used as they are.
4. Fewer than 10 correspondences: the identity pose (and par0 as the final par).
5. GNC: T = I, par = par0.  Iteration itr runs over the correspondences in order, q the normalised target point moved
   by every earlier update: r = p - q, s = (par / (r.r + par))^2; the rows J_x = (0, -q_z, q_y, -1, 0, 0),
   J_y = (q_z, 0, -q_x, 0, -1, 0), J_z = (-q_y, q_x, 0, 0, 0, -1) with residuals r_x, r_y, r_z add (J_a J_b) s to
   J^T J and (J_a r) s to J^T r, row x, then y, then z.  Correspondence c goes to chain c % SOLVE_THREADS, and the
   chains are combined by `block_sum`.  J^T J x = -J^T r is solved by LDL^T (`solve6`, the device's solve6_ldlt);
   delta = Rz(x2) Ry(x1) Rx(x0), t = (x3, x4, x5); T = delta T and every q moves by delta.  Then, with decrease_mu,
   itr % 4 == 0 and par > maximum_correspondence_distance: par /= division_factor.
6. Pose: T maps the normalised target onto the normalised source; the source -> target pose is Open3D's
   GetInvTransformationOriginalScale: R' = R^T, t' = -R^T (-R mu_t + sigma_g t + mu_s).
7. Result row: correspondences entering the solve, tuples kept (0 without the test), trials walked, final par.

Products, sums and norms are rounded one by one (no contraction); norms are sqrt((dx dx + dy dy) + dz dz).

Deviations from Open3D, deliberate or possible:
* The tuple test draws from Philox as above; Open3D draws rand() % n after srand(0), whose sequence depends on the C
  library.
* Sums run in the fixed order above; Open3D sums sequentially (means) or in Eigen's order (normal equations).
* A failed solve (|det J^T J| < 1e-6 or not finite) leaves T and the points unchanged for that iteration, instead of
  whatever Open3D's solver returns there.
* sigma = 0 (every point at the mean, or no points) is taken as 1; Open3D divides by it.  An empty cloud's mean is 0.
* Fewer than 10 correspondences give the identity pose.  Open3D's solve returns the identity there, and depending on
  the version maps it to the original scale (a translation between the means) or not.
* par0 is 1 (relative scale) or sigma (absolute scale) as in step 2; Open3D versions differ in which of their two
  scale values they pass to the solve.
* Feature matching ties go to the lower index (`fpfh_oracle.feature_match`); Open3D's KD-tree order is unspecified.
"""
from __future__ import annotations

import numpy as np

import fpfh_oracle as FO
from dropout_rule import philox

WORD3 = 0x46475254           # "FGRT": counter word 3 of every tuple draw
PREP_THREADS = 512           # chains of the means
SOLVE_THREADS = 256          # chains of the normal equations
WARP = 32


def tree(v: np.ndarray) -> np.ndarray:
    """Halving tree along axis 0 (a power of two long): v[:h] += v[h:2h]."""
    v = np.array(v, np.float64, copy=True)
    h = v.shape[0] // 2
    while h:
        v[:h] = v[:h] + v[h:2 * h]
        h //= 2
    return v[0]


def chains(terms: np.ndarray, width: int) -> np.ndarray:
    """terms (n, k, ...): item i goes to chain i % width, which adds its k terms in order, items ascending."""
    n = terms.shape[0]
    pad = np.zeros(((-n) % width,) + terms.shape[1:])
    rows = np.concatenate([terms, pad]).reshape((-1, width) + terms.shape[1:])
    acc = np.zeros((width,) + terms.shape[2:])
    for r in rows:
        for k in range(terms.shape[1]):
            acc = acc + r[:, k]
    return acc


def block_sum(acc: np.ndarray) -> np.ndarray:
    """The device's block reduction of per-thread chains acc (threads, ...): each warp's 32 lanes by a halving tree
    (the xor butterfly), then the warp sums by a halving tree."""
    w = acc.reshape((-1, WARP) + acc.shape[1:])
    return tree(np.stack([tree(x) for x in w]))


def norm3(d: np.ndarray) -> np.ndarray:
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def mean(p: np.ndarray) -> np.ndarray:
    if p.shape[0] == 0:
        return np.zeros(3)
    return block_sum(chains(p[:, None, :], PREP_THREADS)) / float(p.shape[0])


def normalisation(src: np.ndarray, tgt: np.ndarray, use_absolute_scale: bool = False):
    """-> (mu_s, mu_t, sigma_g, par0)."""
    mu_s, mu_t = mean(src), mean(tgt)
    sigma = 0.0
    for p, mu in ((src, mu_s), (tgt, mu_t)):
        if p.shape[0]:
            sigma = max(sigma, float(norm3(p - mu).max()))
    if not sigma > 0.0:
        sigma = 1.0
    return (mu_s, mu_t, 1.0, sigma) if use_absolute_scale else (mu_s, mu_t, sigma, 1.0)


def tuple_draws(seed: int, pair: int, ks, n: int) -> np.ndarray:
    """(len(ks), 3) int64 indices of trials ks of global pair `pair` out of n correspondences."""
    ks = np.asarray(ks, np.uint64)
    w = philox((ks, pair, 0, WORD3), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    return np.stack([((w[e] * np.uint64(n)) >> np.uint64(32)).astype(np.int64) for e in range(3)], 1)


def tuple_passes(a: np.ndarray, c: np.ndarray, idx: np.ndarray, scale: float) -> np.ndarray:
    """(K,) bool: the tuple test of the draws idx (K,3) on the normalised a, c."""
    ok = np.ones(idx.shape[0], bool)
    for e0, e1 in ((0, 1), (1, 2), (2, 0)):
        ls = norm3(a[idx[:, e0]] - a[idx[:, e1]])
        lt = norm3(c[idx[:, e0]] - c[idx[:, e1]])
        ok &= (ls * scale < lt) & (lt < ls / scale)
    return ok


def tuple_walk(a: np.ndarray, c: np.ndarray, seed: int, pair: int, scale: float, cap: int, batch: int = 8192):
    """-> (indices (3 tuples,) into a / c, tuples, trials walked)."""
    n = a.shape[0]
    kept, walked = [], 0
    total = 100 * n
    for k0 in range(0, total, batch):
        ks = np.arange(k0, min(k0 + batch, total))
        idx = tuple_draws(seed, pair, ks, n)
        hits = np.nonzero(tuple_passes(a, c, idx, scale))[0]
        room = cap - len(kept)
        if len(hits) >= room:
            kept.extend(idx[hits[:room]])
            return np.asarray(kept, np.int64).reshape(-1), cap, int(ks[hits[room - 1]]) + 1
        kept.extend(idx[hits])
        walked = int(ks[-1]) + 1
    return np.asarray(kept, np.int64).reshape(-1), len(kept), walked


def solve6(H: np.ndarray, v: np.ndarray):
    """solve6_ldlt: A x = -v for the symmetric A (6,6) by LDL^T without pivoting; None when |det| < 1e-6 or det is
    not finite."""
    L = np.zeros((6, 6))
    D = np.zeros(6)
    det = 1.0
    for j in range(6):
        d = H[j, j]
        for k in range(j):
            d -= L[j, k] * L[j, k] * D[k]
        D[j] = d
        det *= d
        for i in range(j + 1, 6):
            a = H[i, j]
            for k in range(j):
                a -= L[i, k] * L[j, k] * D[k]
            L[i, j] = a / d
    if not abs(det) >= 1e-6 or np.isinf(det):
        return None
    y = np.zeros(6)
    for i in range(6):
        a = -v[i]
        for k in range(i):
            a -= L[i, k] * y[k]
        y[i] = a
    x = np.zeros(6)
    for i in range(5, -1, -1):
        a = y[i] / D[i]
        for k in range(i + 1, 6):
            a -= L[k, i] * x[k]
        x[i] = a
    return x


def rigid_from_vec6(x) -> np.ndarray:
    """(4,4): R = Rz(x2) Ry(x1) Rx(x0), t = x[3:] (Open3D's TransformVector6dToMatrix4d)."""
    sa, ca, sb, cb, sc, cc = np.sin(x[0]), np.cos(x[0]), np.sin(x[1]), np.cos(x[1]), np.sin(x[2]), np.cos(x[2])
    M = np.eye(4)
    M[:3, :3] = [[cc * cb, cc * sb * sa - sc * ca, cc * sb * ca + sc * sa],
                 [sc * cb, sc * sb * sa + cc * ca, sc * sb * ca - cc * sa],
                 [-sb, cb * sa, cb * ca]]
    M[:3, 3] = x[3:6]
    return M


def move(M: np.ndarray, q: np.ndarray) -> np.ndarray:
    """((m0 x + m1 y) + m2 z) + m3 per row."""
    return np.stack([((M[r, 0] * q[:, 0] + M[r, 1] * q[:, 1]) + M[r, 2] * q[:, 2]) + M[r, 3] for r in range(3)], 1)


def compose(D: np.ndarray, T: np.ndarray) -> np.ndarray:
    """D T for two rigid (4,4), each entry ((d0 t0 + d1 t1) + d2 t2) (+ d3)."""
    out = np.eye(4)
    for r in range(3):
        for c in range(4):
            out[r, c] = (D[r, 0] * T[0, c] + D[r, 1] * T[1, c]) + D[r, 2] * T[2, c] + (D[r, 3] if c == 3 else 0.0)
    return out


UPPER = [(a, b) for a in range(6) for b in range(a, 6)]


def gnc_terms(p: np.ndarray, q: np.ndarray, par: float) -> np.ndarray:
    """(n, 3, 27): per correspondence and row x, y, z the 21 upper J^T J terms (J_a J_b) s and the 6 J^T r terms
    (J_a r) s."""
    r = p - q
    tmp = par / (((r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]) + r[:, 2] * r[:, 2]) + par)
    s = tmp * tmp
    z, one = np.zeros(len(p)), np.ones(len(p))
    J = np.stack([np.stack([z, -q[:, 2], q[:, 1], -one, z, z], 1),
                  np.stack([q[:, 2], z, -q[:, 0], z, -one, z], 1),
                  np.stack([-q[:, 1], q[:, 0], z, z, z, -one], 1)], 1)            # (n, 3, 6)
    out = np.empty((len(p), 3, 27))
    for e, (a, b) in enumerate(UPPER):
        out[:, :, e] = (J[:, :, a] * J[:, :, b]) * s[:, None]
    for a in range(6):
        out[:, :, 21 + a] = (J[:, :, a] * r) * s[:, None]
    return out


def gnc(p: np.ndarray, q: np.ndarray, par0: float, iteration_number: int = 64,
        maximum_correspondence_distance: float = 0.025, division_factor: float = 1.4, decrease_mu: bool = True):
    """-> (T (4,4) normalised target -> normalised source, final par); the identity below 10 correspondences."""
    par = float(par0)
    T = np.eye(4)
    if p.shape[0] < 10:
        return T, par
    q = q.copy()
    for itr in range(iteration_number):
        s = block_sum(chains(gnc_terms(p, q, par), SOLVE_THREADS))
        H = np.zeros((6, 6))
        for e, (a, b) in enumerate(UPPER):
            H[a, b] = H[b, a] = s[e]
        x = solve6(H, s[21:])
        if x is not None:
            D = rigid_from_vec6(x)
            T = compose(D, T)
            q = move(D, q)
        if decrease_mu and itr % 4 == 0 and par > maximum_correspondence_distance:
            par = par / division_factor
    return T, par


def par_schedule(par0: float, iteration_number: int, maximum_correspondence_distance: float, division_factor: float,
                 decrease_mu: bool = True):
    """The par of every iteration (before its update) and the final par, as `gnc` walks them."""
    par, out = float(par0), []
    for itr in range(iteration_number):
        out.append(par)
        if decrease_mu and itr % 4 == 0 and par > maximum_correspondence_distance:
            par = par / division_factor
    return out, par


def original_scale(T: np.ndarray, mu_s, mu_t, sigma_g: float) -> np.ndarray:
    """GetInvTransformationOriginalScale -> (3,4) source -> target."""
    R, t = T[:3, :3], T[:3, 3]
    out = np.zeros((3, 4))
    out[:, :3] = R.T
    out[:, 3] = -R.T @ (-R @ mu_t + t * sigma_g + mu_s)
    return out


def fgr(src, tgt, corr_src, corr_tgt, mask=None, maximum_correspondence_distance: float = 0.025,
        iteration_number: int = 64, division_factor: float = 1.4, decrease_mu: bool = True,
        use_absolute_scale: bool = False, tuple_test: bool = False, tuple_scale: float = 0.95,
        maximum_tuple_count: int = 1000, seed: int = 0, pair: int = 0):
    """One pair (global index `pair`) -> dict(pose (3,4), T (4,4), n_corr, tuples, trials, par, idx, mu_s, mu_t,
    sigma_g, par0)."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    a = np.asarray(corr_src, np.float64).reshape(-1, 3)
    c = np.asarray(corr_tgt, np.float64).reshape(-1, 3)
    if mask is not None:
        keep = np.asarray(mask, bool)
        a, c = a[keep], c[keep]
    mu_s, mu_t, sg, par0 = normalisation(src, tgt, use_absolute_scale)
    an, cn = (a - mu_s) / sg, (c - mu_t) / sg
    idx, tuples, trials = np.arange(a.shape[0]), 0, 0
    if tuple_test and a.shape[0] > 0:
        idx, tuples, trials = tuple_walk(an, cn, seed, pair, tuple_scale, maximum_tuple_count)
    T, par = gnc(an[idx], cn[idx], par0, iteration_number, maximum_correspondence_distance, division_factor,
                 decrease_mu)
    pose = np.eye(3, 4) if len(idx) < 10 else original_scale(T, mu_s, mu_t, sg)
    return dict(pose=pose, T=T, n_corr=len(idx), tuples=tuples, trials=trials, par=par, idx=idx, mu_s=mu_s,
                mu_t=mu_t, sigma_g=sg, par0=par0)



def fgr_batch(src_list, tgt_list, corr_src, corr_tgt, corr_mask=None, pair_base: int = 0, **kw):
    """`ops.fgr`'s layout: -> (pose (B,3,4), result (B,4) = correspondences, tuples, trials, par), float64."""
    outs = [fgr(s, t, a, c, None if corr_mask is None else corr_mask[b], pair=pair_base + b, **kw)
            for b, (s, t, a, c) in enumerate(zip(src_list, tgt_list, corr_src, corr_tgt))]
    return (np.stack([o['pose'] for o in outs]),
            np.array([[o['n_corr'], o['tuples'], o['trials'], o['par']] for o in outs], np.float64).reshape(-1, 4))


def fgr_feature_matching(src, tgt, fs, ft, tuple_test: bool = True, **kw):
    """Open3D's registration_fgr_based_on_feature_matching: the mutual matches of `fpfh_oracle.feature_match`, then
    `fgr` over src[i] -> tgt[nn[i]].  -> (fgr's dict, feature_match's dict)."""
    src = np.asarray(src, np.float64).reshape(-1, 3)
    tgt = np.asarray(tgt, np.float64).reshape(-1, 3)
    m = FO.feature_match(fs, ft, True, 0)
    return fgr(src, tgt, src, tgt[m['nn']], m['mask'], tuple_test=tuple_test, **kw), m
