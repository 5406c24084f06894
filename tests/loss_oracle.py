"""References, input families and a kernel model for the training-loss kernels (csrc/loss.cu).  CPU only; shared by
tests/test_gpu_loss_domain.py and tests/test_loss_sharpness.py.

Geometry: the rule of loss.cu's header restated in numpy.  Source key points are moved by the ground-truth pose in
fp32 in the order of x @ R^T + t (target key points by its inverse, for the correspondence loss); squared distances
are float64 sums of squared coordinate differences of the fp32 points, compared with r_p^2 and r_n^2 taken in float64;
a source token's positive is its nearest target (ties to the lowest index), it is an anchor when that distance is
strictly below r_p, and targets strictly inside r_n other than the positive are ignored.  The circle counts n_pos /
n_neg are the tokens of the other cloud strictly inside r_p / strictly outside r_n, n_sel the tokens with both.

References: the InfoNCE and circle terms of `losses.infonce_loss` / `losses.circle_loss`, the overlap BCE, the
correspondence L1 and `losses.compute_overlaps`, restated with the geometry decisions as inputs (near a threshold
torch.cdist may decide otherwise), evaluated by torch in float64 (the truth) and in fp32 (the other side of the fp32
yardstick, tests/grad_yardstick.py).

Invariant: per pair and InfoNCE term, sum_j d tgt_feat_j = 0 in exact arithmetic (a vector added to every target
shifts each row's logits by one constant); per pair and circle term, the sum over both clouds is 0 (the circle loss
depends on feature differences only).  Checked against the fp32 reference's own deviation, as
tests/attention_oracle.py does.  A kernel whose softmax rows do not sum to 1 breaks the InfoNCE one.

Model: the kernels' fp32 arithmetic in numpy, for tests/test_loss_sharpness.py.  InfoNCE: q = a Ws rounded to fp32
(the 3xTF32 GEMM is as accurate as fp32), one fmaf chain per logit in ascending channel order, the log-sum-exp summed
in fp64 of fp32 expf and rounded to fp32, backward weights c_i (expf(s - lse) - [j = pos]) and fmaf chains over the
rows of the other cloud in ascending order.  Circle: one fmaf chain of squared channel differences per distance,
fp64 log-sum-exps and softplus.  BCE and the pyramid: their fp32 per-token steps, fp64 sums.
Emulated wrong kernels (`variant`), each one small change to the model:
  anchor_le        an anchor at distance <= r_p instead of < r_p
  ignore_positive  the ignore mask drops the positive too
  mean_all_rows    the pair loss is the mean over all source rows, not over the anchors
  tail_dropped     the last partial 32-row tile of targets is dropped
  lse_fp32         the log-sum-exp is summed in fp32 instead of fp64
  bce_src_norm     the BCE is normalised by the source token count instead of all tokens
  circle_skip_zero circle entries outside the positive / negative sets are left out of the log-sum-exps instead of
                   entering as exp(0)
  pyr_div_k        the pyramid divides by the pool width K instead of the count of valid slots
"""
import numpy as np
import torch
import torch.nn.functional as F

from grad_yardstick import FACTOR, FLOOR

D = 256
TM = 32
PW = 256
VARIANTS = ('anchor_le', 'ignore_positive', 'mean_all_rows', 'tail_dropped', 'lse_fp32', 'bce_src_norm',
            'circle_skip_zero', 'pyr_div_k')
FAMILIES = ('model', 'flat', 'shared', 'peaked', 'margins', 'edges', 'pointwise')

f32 = np.float32


# ------------------------------------------------------------------------------------------------------- geometry

def move(x, P, inverse=False):
    """R x + t of a (3, 4) fp32 pose (inverse: R^T x - R^T t) on (n, 3) fp32 points, the kernel's fp32 steps."""
    x, P = np.asarray(x, f32), np.asarray(P, f32)
    if inverse:
        r = P[:, :3].T
        t = -((r[:, 0] * P[0, 3] + r[:, 1] * P[1, 3]) + r[:, 2] * P[2, 3])
    else:
        r, t = P[:, :3], P[:, 3]
    out = np.empty_like(x)
    for j in range(3):
        out[:, j] = ((x[:, 0] * r[j, 0] + x[:, 1] * r[j, 1]) + x[:, 2] * r[j, 2]) + t[j]
    return out


def dist2(a, b):
    """(n, m) float64 squared distances of fp32 points, summed in the kernel's order."""
    d = [np.asarray(a, f32)[:, None, k].astype(np.float64) - np.asarray(b, f32)[None, :, k].astype(np.float64)
         for k in range(3)]
    return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


def offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def geometry(xyz, lens, pose, r_p, r_n, variant=None):
    """Every geometric decision of a packed batch.  -> dict: gt (N, 3) fp32 ground-truth positions of the
    correspondence loss (moved sources, inverse-moved targets), pos (N) global index of
    each source's positive (-1: empty target cloud; target rows -1 too), anchor (N) int32, n_anchor (B), per pair
    'ignore' (ns, nt) bool and 'g2' (ns, nt) float64, n_pos / n_neg (N), n_sel (2B)."""
    B, N, offs = len(lens) // 2, sum(lens), offsets(lens)
    rp2, rn2 = float(r_p) * float(r_p), float(r_n) * float(r_n)
    xyz = np.asarray(xyz, f32)
    gt = np.zeros((N, 3), f32)
    pos, anchor = np.full(N, -1, np.int64), np.zeros(N, np.int32)
    n_pos, n_neg = np.zeros(N, np.int32), np.zeros(N, np.int32)
    ignore, g2s = [], []
    for b in range(B):
        s, t = slice(offs[b], offs[b + 1]), slice(offs[B + b], offs[B + b + 1])
        gt[s] = move(xyz[s], pose[b])
        gt[t] = move(xyz[t], pose[b], inverse=True)
        g2 = dist2(gt[s], xyz[t])
        g2s.append(g2)
        ns, nt = g2.shape
        if nt:
            p = np.argmin(g2, axis=1)                      # first minimum: ties to the lowest index
            d = g2[np.arange(ns), p]
            pos[s] = p + offs[B + b]
            anchor[s] = (d <= rp2) if variant == 'anchor_le' else (d < rp2)
            ig = g2 < rn2
            ig[np.arange(ns), p] = False
        else:
            ig = np.zeros((ns, 0), bool)
        ignore.append(ig)
        n_pos[s], n_neg[s] = (g2 < rp2).sum(1), (g2 > rn2).sum(1)
        n_pos[t], n_neg[t] = (g2 < rp2).sum(0), (g2 > rn2).sum(0)
    sel = (n_pos > 0) & (n_neg > 0)
    n_sel = np.array([int(sel[offs[c]:offs[c + 1]].sum()) for c in range(2 * B)], np.int32)
    n_anchor = np.array([int(anchor[offs[b]:offs[b + 1]].sum()) for b in range(B)], np.int32)
    return dict(gt=gt, pos=pos, anchor=anchor, n_anchor=n_anchor, ignore=ignore, g2=g2s, n_pos=n_pos, n_neg=n_neg,
                n_sel=n_sel, rp2=rp2, rn2=rn2, lens=list(lens), B=B, offs=offs)


# ----------------------------------------------------------------------------------------------------- references

def sym(W):
    Wt = torch.triu(W)
    return Wt + Wt.T


def infonce_pairs(feat, Ws, geo):
    """Per-pair InfoNCE losses (list of 0-d tensors; NaN constant for a pair without an anchor) of the packed (N, D)
    features, with the geometry decisions of `geo`: logits (a Ws) p^T, ignored entries -inf, lse - positive logit,
    mean over the anchors."""
    B, offs, out = geo['B'], geo['offs'], []
    for b in range(B):
        s0, s1, t0, t1 = offs[b], offs[b + 1], offs[B + b], offs[B + b + 1]
        anc = torch.from_numpy(geo['anchor'][s0:s1].astype(bool))
        if not bool(anc.any()):
            out.append(torch.tensor(float('nan'), dtype=feat.dtype))
            continue
        a, p = feat[s0:s1][anc], feat[t0:t1]
        logits = (a @ Ws) @ p.T
        logits = logits.masked_fill(torch.from_numpy(geo['ignore'][b])[anc], float('-inf'))
        pos = torch.from_numpy(geo['pos'][s0:s1] - t0)[anc]
        rl = torch.logsumexp(logits, -1) - logits.gather(1, pos[:, None])[:, 0]
        out.append(rl.sum() / int(anc.sum()))
    return out


def circle_pairs(feat, geo):
    """Per-pair circle losses (CircleLossFull(dist_type='euclidean')) with the geometry decisions of `geo`: feature
    distances sqrt(|a - b|^2 + 1e-12) from explicit differences, z+ / z- on the positive / negative entries and 0
    (exp(0) = 1 in the log-sum-exps) elsewhere, softplus (linear above 20) / 10, mean over the selected rows plus mean
    over the selected columns, halved; NaN where a selection is empty."""
    B, offs, out = geo['B'], geo['offs'], []
    for b in range(B):
        s0, s1, t0, t1 = offs[b], offs[b + 1], offs[B + b], offs[B + b + 1]
        if s1 == s0 or t1 == t0:
            out.append(torch.tensor(float('nan'), dtype=feat.dtype))
            continue
        a, p = feat[s0:s1], feat[t0:t1]
        Dm = torch.sqrt(torch.cdist(a, p, compute_mode='donot_use_mm_for_euclid_dist') ** 2 + 1e-12)
        g2 = torch.from_numpy(geo['g2'][b])
        pm, nm = g2 < geo['rp2'], g2 > geo['rn2']
        u = Dm - 0.1
        zp = torch.where(pm, 10.0 * u * u.clamp_min(0).detach(), torch.zeros_like(Dm))
        v = 1.4 - Dm
        zn = torch.where(nm, 10.0 * v * v.clamp_min(0).detach(), torch.zeros_like(Dm))
        row = F.softplus(torch.logsumexp(zp, -1) + torch.logsumexp(zn, -1)) / 10.0
        col = F.softplus(torch.logsumexp(zp, -2) + torch.logsumexp(zn, -2)) / 10.0
        rs = torch.from_numpy(((geo['n_pos'][s0:s1] > 0) & (geo['n_neg'][s0:s1] > 0)))
        cs = torch.from_numpy(((geo['n_pos'][t0:t1] > 0) & (geo['n_neg'][t0:t1] > 0)))
        out.append((row[rs].mean() + col[cs].mean()) / 2)
    return out


def norms_of(case, geo):
    """(token count, source sum w, target sum w, pair count) of a batch, float64, in the order of regtr_loss_norms."""
    w, offs, B = case['w'].astype(np.float64), geo['offs'], geo['B']
    return np.array([float(offs[-1]), w[:offs[B]].sum(), w[offs[B]:].sum(), float(B)])


def reference(case, dtype, norm=None, grad=True):
    """Every loss value (in the order of ops.LossGeometry.keys()) and, with grad, d (sum_k g_k val_k) / d (both_un,
    cond, corr, logit, W, W_un), in `dtype` on the CPU.  norm: the batch normalisers to divide by (default: this
    batch's own).  -> (vals (n_keys,), grads dict)."""
    geo = case['geo']
    nm = norms_of(case, geo) if norm is None else np.asarray(norm, np.float64)
    cast = lambda a: torch.from_numpy(np.asarray(a)).to(dtype).requires_grad_(grad)
    x = {k: cast(case[k]) for k in ('both_un', 'cond', 'corr', 'logit')}
    circle = case['loss'] == 'circle'
    if not circle:
        x['W'], x['W_un'] = cast(case['W']), cast(case['W_un'])
    offs, B = geo['offs'], geo['B']
    n_src = offs[B]
    w = torch.from_numpy(case['w']).to(dtype)
    gt = torch.from_numpy(geo['gt']).to(dtype)
    vals = {}
    for l in case['overlap_on']:
        vals[f'overlap_{l}'] = F.binary_cross_entropy_with_logits(x['logit'][l, :, 0], w, reduction='sum') / nm[0]
    terms = [(f'feature_{l}', x['cond'][l], 'W') for l in case['feature_on']] + [('feature_un', x['both_un'], 'W_un')]
    for key, feat, wk in terms:
        pairs = circle_pairs(feat, geo) if circle else infonce_pairs(feat, sym(x[wk]), geo)
        vals[key] = torch.stack(pairs).sum() / nm[3]
    for l in case['corr_on']:
        err = (x['corr'][l] - gt).abs().sum(-1) * w
        vals[f'corr_{l}'] = err[:n_src].sum() / max(nm[1], 1e-6) + err[n_src:].sum() / max(nm[2], 1e-6)
    keys = case['keys']
    v = torch.stack([vals[k] for k in keys])
    grads = {}
    if grad:
        g = torch.from_numpy(case['g']).to(dtype)
        total = (v * g).sum()               # NaN where a pair has no anchor; its finite pairs still take gradient
        leaves = list(x.values())
        gs = torch.autograd.grad(total, leaves, allow_unused=True)
        grads = {k: (torch.zeros_like(t) if d is None else d) for (k, t), d in zip(x.items(), gs)}
    return v.detach(), grads


def pyramid(pyr0, pools, n_prev, dtype):
    """compute_overlaps in `dtype`: each level the mean of the previous level over the valid pool slots (index <
    n_prev), summed in ascending slot order, clamped to [0, 1]; a row without a valid slot is NaN."""
    out = [torch.from_numpy(np.asarray(pyr0)).to(dtype)]
    for pool, n in zip(pools, n_prev):
        pool = torch.from_numpy(np.asarray(pool, np.int64))
        valid = pool < n
        g = torch.where(valid, out[-1][pool.clamp_max(max(n - 1, 0))], torch.zeros((), dtype=dtype))
        s = torch.zeros(pool.shape[0], dtype=dtype)
        for k in range(pool.shape[1]):
            s = s + g[:, k]
        out.append((s / valid.sum(1)).clamp(0, 1))
    return out


# ------------------------------------------------------------------------------------------------------- invariant

def invariant_rows(case, got, fp32, ref):
    """Per pair and feature term: the deviation of the kernel's and the fp32 reference's sum of d feat from 0 (InfoNCE:
    over the target tokens; circle: over both clouds), max over the channels.  got / fp32 / ref: dicts with 'cond'
    and 'both_un' gradients.  -> [(term, pair, kernel deviation, fp32 deviation, bound)], bound = FACTOR x fp32
    deviation + FLOOR x max|float64 gradient over those tokens|."""
    geo, out = case['geo'], []
    offs, B = geo['offs'], geo['B']
    terms = [(f'feature_{l}', lambda d, l=l: d['cond'][l]) for l in case['feature_on']] + \
        [('feature_un', lambda d: d['both_un'])]
    for key, pick in terms:
        if float(case['g'][case['keys'].index(key)]) == 0.0:
            continue
        for b in range(B):
            if geo['n_anchor'][b] == 0 and case['loss'] == 'infonce':
                continue
            rows = np.r_[offs[B + b]:offs[B + b + 1]] if case['loss'] == 'infonce' else \
                np.r_[offs[b]:offs[b + 1], offs[B + b]:offs[B + b + 1]]
            if len(rows) < 2:
                continue
            r = torch.from_numpy(rows)
            dev = [float(pick(d).detach().double().cpu()[r].sum(0).abs().max()) for d in (got, fp32)]
            scale = float(pick(ref).detach().double()[r].abs().max())
            if scale == 0.0:
                continue
            out.append((key, b, dev[0], dev[1], FACTOR * dev[1] + FLOOR * scale))
    return out


def invariant_failures(rows):
    return [r for r in rows if not r[2] <= r[4]]


# --------------------------------------------------------------------------------------------------------- inputs

def _rotation(rng):
    q, r = np.linalg.qr(rng.normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q * np.linalg.det(q)


def _layer_norm_rows(x):
    x = x - x.mean(-1, keepdims=True)
    return x / x.std(-1, keepdims=True)


def make_case(lens, family, seed, loss='infonce', n_layers=2, feature_on=(1,), overlap_on=(1,), corr_on=(1,),
              wt_un=1.0, no_anchor_pairs=()):
    """A seeded packed batch of `lens` (B source clouds then B target clouds) for ops.loss_forward, as numpy arrays.
    family (FAMILIES):
      model      LayerNorm-like rows and W of std 0.1: logits of +-50-100, as at initialisation
      flat       W of std 1e-4: every softmax row near uniform
      shared     target features share an offset 3x their spread: a wrong sum_j P reaches d src through it
      peaked     an anchor's features are its positive's plus noise and W = 0.033 I: the positive's logit stands about
                 17 above the rest, whose hundreds of exp(-17) terms an fp32 running sum drops
      margins    features tied to the key points at three noise scales: circle distances around 0.1 and 1.4 and
                 positive exponents past softplus' threshold of 20
      edges      key points on a 1/8 grid under a signed-permutation pose (every distance exact): key points exactly
                 at r_p = 0.25 and r_n = 0.5, equidistant ties, duplicate points, a pair whose rows have only their
                 positive unmasked
      pointwise  overlap logits of +-30, corr equal to the fp32 ground truth on every third token (sign(0) = 0),
                 overlap weights 0, 1 and fractional
    no_anchor_pairs: pairs whose targets are moved 100 away (no anchor, no positive)."""
    rng = np.random.default_rng(seed)
    B, N, offs = len(lens) // 2, sum(lens), offsets(lens)
    edges = family == 'edges'
    r_p, r_n = (0.25, 0.5) if edges else (0.2, 0.4)
    xyz = np.zeros((N, 3), f32)
    pose = np.zeros((B, 3, 4), f32)
    for b in range(B):
        ns, nt = lens[b], lens[B + b]
        s, t = slice(offs[b], offs[b + 1]), slice(offs[B + b], offs[B + b + 1])
        if edges:
            R = np.eye(3)[rng.permutation(3)] * rng.choice([-1.0, 1.0], 3)
            T = rng.integers(-8, 9, 3) / 8.0
            side = 1.0 + 0.125 * np.cbrt(max(ns, nt))
            grid = lambda n: (rng.integers(0, int(side * 8) + 1, (n, 3)) / 8.0)
            tgt = grid(nt)
            if b == 0 and nt:                          # duplicate target points
                tgt[1::7] = tgt[0::7][:len(tgt[1::7])]
            src_w = grid(ns)
            if B > 1 and b == 1 and nt:                # a tight pair: every target within r_n of every source
                tgt = np.full((nt, 3), 4.0) + rng.integers(0, 2, (nt, 3)) / 8.0
                src_w = np.full((ns, 3), 4.0) + rng.integers(0, 2, (ns, 3)) / 8.0
            src = (src_w - T) @ R                      # R^T (y - T) exactly: entries of R are 0 and +-1
        else:
            R, T = _rotation(rng), rng.uniform(-1, 1, 3)
            side = 0.3 * np.cbrt(max(nt, 1))           # about one target per r_p-ball
            tgt = rng.uniform(0, side, (nt, 3))
            k = rng.integers(0, max(nt, 1), ns)
            near = tgt[k] + rng.normal(0, 0.08, (ns, 3)) if nt else rng.uniform(0, side, (ns, 3))
            far = rng.uniform(0, side, (ns, 3))
            src_w = np.where(rng.random((ns, 1)) < 0.7, near, far)
            src = (src_w - T) @ R
        if b in no_anchor_pairs:
            T = T + 100.0
        pose[b, :, :3], pose[b, :, 3] = R, T
        xyz[s], xyz[t] = src, tgt
    geo = geometry(xyz, lens, pose, r_p, r_n)
    nl = n_layers

    def feats(n_rows, lat):
        base = rng.normal(size=(n_rows, D))
        if family in ('margins', 'edges') and loss == 'circle':
            P = np.linalg.qr(rng.normal(size=(D, 3)))[0]
            scale = rng.choice([0.005, 0.3, 1.0], size=(n_rows, 1))
            return (0.3 * lat + scale * rng.normal(size=(n_rows, 3))) @ P.T + 0.001 * base
        x = _layer_norm_rows(base)
        if family == 'shared':
            off = 3.0 * rng.normal(size=D)
            x[offs[B]:] += off
        return x

    lat = np.concatenate([geo['gt'][:offs[B]], xyz[offs[B]:]]).astype(np.float64)

    def peaked(x):
        src = np.nonzero(geo['anchor'])[0]
        x[src] = x[geo['pos'][src]] + 0.05 * rng.normal(size=(len(src), D))
        return x
    pk = peaked if family == 'peaked' else (lambda x: x)
    both_un = pk(feats(N, lat))
    cond = np.stack([pk(feats(N, lat)) for _ in range(nl)])
    wstd = 1e-4 if family == 'flat' else 0.1
    W, W_un = rng.normal(0, wstd, (D, D)), rng.normal(0, wstd, (D, D))
    if family == 'peaked':
        W, W_un = 0.033 * np.eye(D) + rng.normal(0, 1e-4, (D, D)), 0.033 * np.eye(D) + rng.normal(0, 1e-4, (D, D))
    gt = geo['gt'].astype(np.float64)
    corr = gt[None] + rng.normal(0, 0.05, (nl, N, 3))
    logit = rng.normal(0, 3.0, (nl, N, 1))
    w = rng.random(N)
    if family == 'pointwise':
        logit = rng.choice([-30.0, 30.0, 0.0, 1e-3], size=(nl, N, 1)) + rng.normal(0, 1e-3, (nl, N, 1))
        w = rng.choice([0.0, 1.0, 0.25, 0.625], size=N)
        corr[:, ::3] = gt[None, ::3]
    else:
        w = np.where(rng.random(N) < 0.3, np.round(w), w)
    keys = [f'overlap_{i}' for i in overlap_on] + [f'feature_{i}' for i in feature_on] + ['feature_un'] + \
        [f'corr_{i}' for i in corr_on]
    g = rng.uniform(0.5, 2.0, len(keys))
    g[keys.index('feature_un')] *= wt_un
    case = dict(lens=list(lens), loss=loss, family=family, xyz=xyz, pose=pose, w=w.astype(f32),
                both_un=both_un.astype(f32), cond=cond.astype(f32), corr=corr.astype(f32), logit=logit.astype(f32),
                W=W.astype(f32), W_un=W_un.astype(f32), r_p=r_p, r_n=r_n, overlap_on=list(overlap_on),
                feature_on=list(feature_on), corr_on=list(corr_on), keys=keys, g=g.astype(f32), geo=geo)
    if family == 'pointwise':                        # corr exactly the fp32 ground truth on every third token
        case['corr'][:, ::3] = geo['gt'][None, ::3]
    return case


def subset(case, pairs):
    """The same inputs restricted to the given pairs (in that order), geometry recomputed."""
    B, offs = case['geo']['B'], case['geo']['offs']
    rows = np.concatenate([np.r_[offs[b]:offs[b + 1]] for b in pairs] +
                          [np.r_[offs[B + b]:offs[B + b + 1]] for b in pairs]).astype(np.int64)
    lens = [case['lens'][b] for b in pairs] + [case['lens'][B + b] for b in pairs]
    out = dict(case, lens=lens, xyz=case['xyz'][rows], pose=case['pose'][list(pairs)], w=case['w'][rows],
               both_un=case['both_un'][rows], cond=case['cond'][:, rows], corr=case['corr'][:, rows],
               logit=case['logit'][:, rows])
    out['geo'] = geometry(out['xyz'], lens, out['pose'], case['r_p'], case['r_n'])
    out['rows'] = rows
    return out


# ---------------------------------------------------------------------------------------------------- kernel model

def _fma(a, b, c):
    """fmaf on fp32 operands: the exact product (float64 holds it), the sum rounded once to fp32 (via float64)."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def model_logits(q, p):
    """(n, m) fp32 logits: one fmaf chain per entry over the channels in ascending order."""
    acc = np.zeros((q.shape[0], p.shape[0]), f32)
    for k in range(q.shape[1]):
        acc = _fma(q[:, k:k + 1], p[None, :, k], acc)
    return acc


def model_infonce(case, feat, W, geo=None, variant=None, g=1.0):
    """The InfoNCE kernels on one term.  -> dict: pair (B,) fp64 pair losses, value (fp32), d_src (rows of the
    source clouds, via dQ Ws), d_tgt (rows of the target clouds), both in packed (N, D) fp32."""
    geo = geo or geometry(case['xyz'], case['lens'], case['pose'], case['r_p'], case['r_n'],
                          variant if variant == 'anchor_le' else None)
    B, offs = geo['B'], geo['offs']
    W64 = np.asarray(W, np.float64)
    Ws = np.triu(W64) + np.triu(W64).T
    N = offs[-1]
    feat = np.asarray(feat, f32)
    q_all = (feat.astype(np.float64) @ Ws).astype(f32)
    pair = np.full(B, np.nan)
    dq, dfeat = np.zeros((N, D), f32), np.zeros((N, D), f32)
    for b in range(B):
        s0, s1, t0, t1 = offs[b], offs[b + 1], offs[B + b], offs[B + b + 1]
        ns, nt = s1 - s0, t1 - t0
        if ns == 0 or nt == 0:
            continue
        q, p = q_all[s0:s1], feat[t0:t1]
        s = model_logits(q, p)
        ign = geo['ignore'][b].copy()
        pos = geo['pos'][s0:s1] - t0
        if variant == 'ignore_positive':
            ign[np.arange(ns), pos] = geo['g2'][b][np.arange(ns), pos] < geo['rn2']
        if variant == 'tail_dropped' and nt % TM:
            ign[:, nt // TM * TM:] = True
        s = np.where(ign, f32(-np.inf), s)
        m = s.max(1)
        e = np.exp((s - m[:, None]).astype(f32)).astype(f32)
        if variant == 'lse_fp32':
            tot = np.zeros(ns, f32)
            for j in range(nt):
                tot = (tot + e[:, j]).astype(f32)
            lse = (m.astype(np.float64) + np.log(tot.astype(np.float64))).astype(f32)
        else:
            lse = (m.astype(np.float64) + np.log(e.astype(np.float64).sum(1))).astype(f32)
        spos = s[np.arange(ns), pos]
        row = (lse - spos).astype(f32)
        anc = geo['anchor'][s0:s1].astype(bool)
        n_anc = int(anc.sum())
        if variant == 'mean_all_rows':
            pair[b] = row.astype(np.float64).sum() / ns
        elif n_anc:
            pair[b] = row[anc].astype(np.float64).sum() / n_anc
        if not n_anc:
            continue
        c = np.where(anc, f32(g / (n_anc * B)), f32(0))
        onehot = np.zeros((ns, nt), f32)
        onehot[np.arange(ns), pos] = 1
        P = np.exp((s - lse[:, None]).astype(f32)).astype(f32)
        G = np.where(np.isfinite(s), (c[:, None] * (P - onehot)).astype(f32), f32(0))
        acc = np.zeros((ns, D), f32)
        for j in range(nt):
            acc = _fma(G[:, j:j + 1], p[j][None], acc)
        dq[s0:s1] = acc
        acc = np.zeros((nt, D), f32)
        for i in range(ns):
            acc = _fma(G[i][:, None], q[i][None], acc)
        dfeat[t0:t1] = acc
    dfeat[:offs[B]] = (dq[:offs[B]].astype(np.float64) @ Ws).astype(f32)
    value = f32(np.sum(pair) / B)
    return dict(pair=pair, value=value, dfeat=dfeat, geo=geo)


def model_circle(case, feat, variant=None):
    """The circle kernels' value of one term: fmaf-chain distances, fp64 log-sum-exps, softplus.  -> (pair, value)."""
    geo = geometry(case['xyz'], case['lens'], case['pose'], case['r_p'], case['r_n'])
    B, offs = geo['B'], geo['offs']
    feat = np.asarray(feat, f32)
    pair = np.full(B, np.nan)
    for b in range(B):
        s0, s1, t0, t1 = offs[b], offs[b + 1], offs[B + b], offs[B + b + 1]
        if s1 == s0 or t1 == t0:
            continue
        a, p = feat[s0:s1], feat[t0:t1]
        acc = np.zeros((len(a), len(p)), f32)
        for k in range(D):
            d = (a[:, k:k + 1] - p[None, :, k]).astype(f32)
            acc = _fma(d, d, acc)
        dist = np.sqrt((acc + f32(1e-12)).astype(f32)).astype(f32)
        pm, nm = geo['g2'][b] < geo['rp2'], geo['g2'][b] > geo['rn2']
        u, v = (dist - f32(0.1)).astype(f32), (f32(1.4) - dist).astype(f32)
        zp = np.where(pm, (f32(10) * u) * np.maximum(u, f32(0)), f32(0)).astype(f32)
        zn = np.where(nm, (f32(10) * v) * np.maximum(v, f32(0)), f32(0)).astype(f32)

        def lse(z, mask, axis):
            if variant == 'circle_skip_zero':
                z = np.where(mask, z, f32(-np.inf))
            m = z.max(axis, keepdims=True)
            with np.errstate(invalid='ignore'):
                e = np.exp((z - m).astype(f32)).astype(np.float64)
            return np.squeeze(m, axis).astype(np.float64) + np.log(e.sum(axis))

        def soft(x):
            with np.errstate(over='ignore'):
                return np.where(x > 20, x, np.log1p(np.exp(np.minimum(x, 20))))
        rows = soft(lse(zp, pm, 1) + lse(zn, nm, 1)) / 10
        cols = soft(lse(zp, pm, 0) + lse(zn, nm, 0)) / 10
        rs = (geo['n_pos'][s0:s1] > 0) & (geo['n_neg'][s0:s1] > 0)
        cs = (geo['n_pos'][t0:t1] > 0) & (geo['n_neg'][t0:t1] > 0)
        with np.errstate(invalid='ignore'):
            pair[b] = (rows[rs].sum() / rs.sum() + cols[cs].sum() / cs.sum()) / 2
    return pair, f32(np.sum(pair) / B)


def model_bce(case, layer, variant=None):
    """The pointwise kernel's BCE value and d logit of one layer: fp32 per token, fp64 sum in token order."""
    x, y = case['logit'][layer, :, 0].astype(f32), case['w'].astype(f32)
    N, n_src = len(x), case['geo']['offs'][case['geo']['B']]
    n = n_src if variant == 'bce_src_norm' else N
    t = (np.maximum(x, f32(0)) - x * y + np.log1p(np.exp(-np.abs(x))).astype(f32)).astype(f32)
    d = ((f32(1) / (f32(1) + np.exp(-x).astype(f32)) - y) / f32(n)).astype(f32)
    return f32(t.astype(np.float64).sum() / n), d


def model_pyramid(pyr0, pools, n_prev, variant=None):
    """The pyramid kernel: fp32 sum over the valid slots in ascending order, divided by their count (K with
    pyr_div_k), clamped; 0 / 0 stays NaN."""
    out = [np.asarray(pyr0, f32)]
    for pool, n in zip(pools, n_prev):
        pool = np.asarray(pool, np.int64)
        valid = (pool >= 0) & (pool < n)
        s = np.zeros(len(pool), f32)
        for k in range(pool.shape[1]):
            s = (s + np.where(valid[:, k], out[-1][np.where(valid[:, k], pool[:, k], 0)], f32(0))).astype(f32)
        cnt = np.full(len(pool), pool.shape[1]) if variant == 'pyr_div_k' else valid.sum(1)
        with np.errstate(invalid='ignore', divide='ignore'):
            v = (s / cnt.astype(f32)).astype(f32)
        out.append(np.where(v < 0, f32(0), np.where(v > 1, f32(1), v)).astype(f32))
    return out


def pyramid_case(K, n_levels=4, n0=700, seed=0):
    """Level-0 0/1 overlap masks and pooling tables of width K for n_levels levels: every valid slot below n_prev,
    shadow slots (n_prev) between them, and at each level a last row of only shadow slots (NaN).  -> (pyr0, pools, n_prev)."""
    rng = np.random.default_rng(seed + K)
    pyr0 = (rng.random(n0) < 0.4).astype(f32)
    pools, n_prev, n = [], [], n0
    for _ in range(n_levels - 1):
        m = max(n // 3, 2)
        pool = rng.integers(0, n - 1, (m, K))                 # the previous level's NaN row stays unreferenced
        if K > 1:
            pool[rng.random((m, K)) < 0.3] = n
        pool[-1] = n
        pools.append(pool.astype(np.int32))
        n_prev.append(n)
        n = m
    return pyr0, pools, n_prev


# ---------------------------------------------------------------------------------------------------- the domain

# Tokens per cloud the grid puts on either side of a pair: every 32-row tile edge, the 256-token chunk edge, the
# configs' clouds and long ones.
EDGE_LENS = (0, 1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 700, 1500)
# (id, source lens, target lens, family, n_layers, feature_on, feature_un weight, pairs without an anchor)
_B1 = [(31, 33), (32, 65), (33, 31), (63, 64), (64, 63), (65, 32), (1, 257), (257, 1), (255, 256), (256, 255),
       (700, 1500), (1500, 700)]
_INFONCE_FAM = ('model', 'flat', 'shared', 'peaked', 'edges', 'pointwise')
_CIRCLE_FAM = ('margins', 'model', 'edges', 'pointwise')


def _lens16():
    rng = np.random.default_rng(16)
    return [int(v) for v in rng.integers(340, 460, 16)], [int(v) for v in rng.integers(340, 460, 16)]


def domain_cases():
    """The grid of tests/test_gpu_loss_domain.py: every tile edge at B = 1 for both losses, an empty cloud on either
    side, the 3DMatch and ModelNet batch shapes at the configs' 6 layers, 8 layers with 7 feature layers (all 8 term
    slots) and every layer's pointwise losses, B = 8 with a pair without an anchor, and B = 16 of about 400 tokens per
    cloud (N about 12800: 50 chunks of the pointwise kernel).  -> [(id, loss, kwargs of make_case)]."""
    out = []
    for loss, fams in (('infonce', _INFONCE_FAM), ('circle', _CIRCLE_FAM)):
        for i, (ns, nt) in enumerate(_B1):
            fam = fams[i % len(fams)]
            layers = dict(n_layers=1, feature_on=(0,), overlap_on=(0,), corr_on=(0,)) if i % 3 == 0 else {}
            out.append((f'{loss}-{ns}x{nt}-{fam}', loss, dict(lens=[ns, nt], family=fam, seed=i, wt_un=float(i % 2),
                                                              **layers)))
        l6 = dict(n_layers=6, feature_on=(5,), overlap_on=(5,), corr_on=(5,))
        l8 = dict(n_layers=8, feature_on=tuple(range(1, 8)), overlap_on=tuple(range(8)), corr_on=tuple(range(8)))
        s16, t16 = _lens16()
        out += [
            (f'{loss}-empty', loss, dict(lens=[0, 45, 40, 0], family=fams[0], seed=20)),
            (f'{loss}-3dmatch-b2', loss, dict(lens=[412, 429, 339, 325], family=fams[1], seed=21, **l6)),
            (f'{loss}-modelnet-b4', loss, dict(lens=[601, 531, 560, 655, 612, 523, 590, 640], family=fams[0],
                                                seed=22, wt_un=0.0, **l6)),
            (f'{loss}-8layers-b2', loss, dict(lens=[70, 33, 64, 95], family='edges', seed=23, **l8)),
            (f'{loss}-b8', loss, dict(lens=[31, 90, 256, 1, 120, 65, 33, 200, 40, 64, 257, 20, 33, 100, 31, 150],
                                      family=fams[2 % len(fams)], seed=24, no_anchor_pairs=(5,))),
            (f'{loss}-b16', loss, dict(lens=s16 + t16, family=fams[1], seed=25, n_layers=1, feature_on=(0,),
                                       overlap_on=(0,), corr_on=(0,))),
        ]
    return out
