"""Generate tests/golden/circle.npz from the UNMODIFIED reference's circle feature loss.

Run where the reference is present:

    python tests/golden/make_circle_golden.py

Two parts, both produced by the reference's own modules through oracle/ref_bridge.py:
  * model level: `RegTR.compute_loss` with `feature_loss_type='circle'` on the `fwd_modelnet_b1` and
    `fwd_3dmatch_small_b2` forwards (seeded weights from `random_state_dict`, which has no `feature_criterion*.W` for
    this loss, and the seeded loss inputs of tests/golden/eval_inputs.py), then `total.backward()`: every loss value
    and, per parameter, the gradient's norm, sum and the entries of `eval_inputs.grad_sample_index`.
  * loss level: `CircleLossFull(dist_type='euclidean', r_p, r_n)` called directly, in float64, on seeded feature and
    coordinate sets whose feature distances span about [0, 2.5]: every branch of the loss is taken (positive entries
    on both sides of the 0.1 margin, negative entries on both sides of 1.4, softplus arguments on both sides of its
    threshold 20, rows without a positive, a one-token cloud, uneven sizes, a pair with nothing selected).  The inputs
    are stored as fp32, the value and the gradients of both feature sets as the float64 results.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import eval_inputs as ei  # noqa: E402
from make_golden import FORWARD_CASES, _np  # noqa: E402
from oracle import ref_bridge  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

MODEL_CASES = ('fwd_modelnet_b1', 'fwd_3dmatch_small_b2')

# loss-level sets: name -> (seed, r_p, r_n, [(n_src, n_tgt, target offset), ...])
LOSS_SETS = {
    'single': (101, 0.35, 0.6, [(48, 40, 0.0)]),
    'uneven': (102, 0.35, 0.6, [(30, 21, 0.0), (37, 9, 0.0), (22, 33, 0.0)]),
    # a one-token cloud leaves every column (rows) of its pair with a single entry: nothing selected there, NaN
    'one_token': (103, 0.35, 0.6, [(1, 26, 0.0), (14, 1, 0.0)]),
    'nan': (104, 0.35, 0.6, [(20, 25, 0.0), (15, 18, 10.0)]),
}


def model_fixture(case, fx):
    cfg_name, wseed, makers = FORWARD_CASES[case][:3]
    cfg = get_config(cfg_name, feature_loss_type='circle')
    sd = random_state_dict(cfg, wseed)
    assert not any(k.startswith('feature_criterion') for k in sd)
    model = ref_bridge.build_reference_model(cfg, sd)              # strict=True
    model.eval()
    for p_ in model.parameters():
        p_.requires_grad_(p_.is_floating_point())
    pairs = [mk() for mk in makers]
    batch = {'src_xyz': [torch.from_numpy(p['src_xyz']) for p in pairs],
             'tgt_xyz': [torch.from_numpy(p['tgt_xyz']) for p in pairs]}
    pred = model(batch)
    batch.update(ei.loss_inputs(pairs, [int(x.shape[0]) for x in batch['src_xyz']],
                                [int(x.shape[0]) for x in batch['tgt_xyz']]))
    losses = model.compute_loss(pred, batch)
    losses['total'].backward()
    for k, v in losses.items():
        fx[f'{case}|loss_{k}'] = _np(v)
    n = 0
    for name, p_ in model.named_parameters():
        if p_.grad is None:
            continue
        g = p_.grad.detach().double().reshape(-1)
        idx = ei.grad_sample_index(name, g.numel())
        fx[f'{case}|g|{name}'] = np.concatenate([[float(g.norm()), float(g.sum())], g[torch.from_numpy(idx)].numpy()])
        n += 1
    print(case, {k: float(v) for k, v in losses.items()}, 'parameters with a gradient:', n)


def make_pair(rng, P, ns, nt, shift):
    """Key points in a 1.5 m box; features = P @ latent + 0.001 noise, latent = 0.3 xyz + a per-token noise of scale
    0.005, 0.3 or 1.0, so that feature distances of geometric neighbours range from ~0.02 to ~2.5."""
    def side(n, off):
        xyz = rng.uniform(0.0, 1.5, (n, 3)) + off
        lat = 0.3 * (xyz - off) + rng.choice([0.005, 0.3, 1.0], size=(n, 1)) * rng.normal(size=(n, 3))
        feat = lat @ P.T + 0.001 * rng.normal(size=(n, 256))
        return feat.astype(np.float32), xyz.astype(np.float32)
    sf, sx = side(ns, 0.0)
    tf, tx = side(nt, shift)
    return sf, tf, sx, tx


def branch_census(pairs, r_p, r_n):
    """Float64 counts of the branches the set exercises (numpy, independent of torch)."""
    c = dict(pos_lo=0, pos_hi=0, neg_lo=0, neg_hi=0, sp_lin=0, sp_log=0, no_pos_row=0, margin=np.inf)
    for sf, tf, sx, tx in pairs:
        g = np.sqrt(((sx[:, None, :].astype(np.float64) - tx[None].astype(np.float64)) ** 2).sum(-1))
        if g.size:
            c['margin'] = min(c['margin'], np.abs(g / r_p - 1).min(), np.abs(g / r_n - 1).min())
        d = np.sqrt(((sf[:, None, :].astype(np.float64) - tf[None].astype(np.float64)) ** 2).sum(-1) + 1e-12)
        pm, nm = g < r_p, g > r_n
        c['pos_lo'] += int((pm & (d < 0.1)).sum()); c['pos_hi'] += int((pm & (d > 0.1)).sum())
        c['neg_lo'] += int((nm & (d < 1.4)).sum()); c['neg_hi'] += int((nm & (d > 1.4)).sum())
        zp = np.where(pm, 10 * (d - 0.1) * np.maximum(d - 0.1, 0), 0.0)
        zn = np.where(nm, 10 * (1.4 - d) * np.maximum(1.4 - d, 0), 0.0)
        lse = lambda z, ax: np.log(np.exp(z).sum(ax)) if z.shape[ax] else np.full(z.shape[1 - ax], -np.inf)
        for ax, sel in ((1, (pm.sum(1) > 0) & (nm.sum(1) > 0)), (0, (pm.sum(0) > 0) & (nm.sum(0) > 0))):
            x = (lse(zp, ax) + lse(zn, ax))[sel]
            c['sp_lin'] += int((x > 20).sum()); c['sp_log'] += int((x <= 20).sum())
        c['no_pos_row'] += int(((pm.sum(1) == 0) & (nm.sum(1) > 0)).sum())
    return c


def loss_fixture(name, fx):
    seed, r_p, r_n, shapes = LOSS_SETS[name]
    rng = np.random.default_rng(seed)
    P = np.linalg.qr(rng.normal(size=(256, 3)))[0]
    pairs = [make_pair(rng, P, ns, nt, shift) for ns, nt, shift in shapes]
    census = branch_census(pairs, r_p, r_n)
    assert census['margin'] > 1e-6, census
    crit = ref_bridge.modules().regtr.CircleLossFull(dist_type='euclidean', r_p=r_p, r_n=r_n)
    t = lambda a: torch.from_numpy(a).double()
    sf = [t(p[0]).requires_grad_(True) for p in pairs]
    tf = [t(p[1]).requires_grad_(True) for p in pairs]
    val = crit(sf, tf, [t(p[2]) for p in pairs], [t(p[3]) for p in pairs])
    val.backward()
    fx[f'{name}|lens'] = np.array([p[0].shape[0] for p in pairs] + [p[1].shape[0] for p in pairs], np.int32)
    fx[f'{name}|radii'] = np.array([r_p, r_n])
    fx[f'{name}|feat'] = np.concatenate([p[0] for p in pairs] + [p[1] for p in pairs])
    fx[f'{name}|xyz'] = np.concatenate([p[2] for p in pairs] + [p[3] for p in pairs])
    fx[f'{name}|value'] = _np(val)
    fx[f'{name}|grad'] = np.concatenate([_np(g.grad) for g in sf] + [_np(g.grad) for g in tf]).astype(np.float32)
    print(name, float(val.detach()), census)
    return census


if __name__ == '__main__':
    torch.manual_seed(0)
    fx = {}
    totals = {}
    for name in LOSS_SETS:
        for k, v in loss_fixture(name, fx).items():
            totals[k] = min(totals.get(k, np.inf), v) if k == 'margin' else totals.get(k, 0) + v
    assert all(totals[k] > 0 for k in ('pos_lo', 'pos_hi', 'neg_lo', 'neg_hi', 'sp_lin', 'sp_log', 'no_pos_row'))
    for case in MODEL_CASES:
        model_fixture(case, fx)
    path = os.path.join(HERE, 'circle.npz')
    np.savez_compressed(path, **fx)
    print(path, os.path.getsize(path) // 1024, 'KiB')
