"""Time Fast Global Registration against RANSAC on the same device FPFH features of the real 3DMatch fixtures
(tests/golden/real), at B = 1 and B = 8 (the three fixtures repeated).

    python scripts/bench_fgr.py [--voxel 0.05] [--reps 10] [--iters 100000] [--out FILE]

Both clouds of every pair are downsampled at V, their normals estimated at 2 V / 30 and their FPFH features computed at
5 V / 100 once, outside the timed window.  Then, per B, after one warm-up call of each:
  fgr      `ops.fgr_feature_matching` (Open3D's defaults, maximum correspondence distance 0.5 V), broken down into
           match (`ops.feature_match`, the mutual matches) and solve (`ops.fgr`: preparation and GNC, 2 launches);
  ransac   `ops.ransac_feature_matching` at 1.5 V with the distance checker at 1.5 V, --iters, confidence 0.999.
CUDA events around each call: the median and the spread (min..max) of --reps runs, in ms per call (all B pairs).  A
torch.profiler run of its own then gives the device time of the two FGR kernels.  One JSON line per B, then one
summary line with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

from regtr_b200 import eval as E
from regtr_b200 import ops

REAL = os.path.join(ROOT, 'tests', 'golden', 'real')
FIXTURES = ('real_3dmatch_redkitchen_0_5', 'real_3dmatch_sun3d_hotel3_8_15', 'real_3dmatch_sun3d_home_38_41')


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')[:2]]
    except Exception:                       # noqa: BLE001 -- no nvidia-smi: the name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--voxel', type=float, default=0.05)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--iters', type=int, default=100000)
    ap.add_argument('--out', help='Also write the JSON lines to this file')
    return ap


def features(voxel):
    """-> (src_down, tgt_down, src_feat, tgt_feat): device tensors of the three fixtures."""
    clouds = []
    for fx in FIXTURES:
        inp = np.load(os.path.join(REAL, fx + '_input.npz'))
        clouds.append((inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)))
    down = E.fpfh_downsample([s for s, _ in clouds] + [t for _, t in clouds], voxel)
    normals = ops.estimate_normals(down, 2 * voxel, 30)
    feats = ops.fpfh(down, normals, 5 * voxel, 100)
    n = len(FIXTURES)
    return down[:n], down[n:], feats[:n], feats[n:]


def timed(fn, reps):
    """fn() -> ms per call of reps calls, each between two CUDA events."""
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def stats(row, key, t):
    row[f'{key}_ms'] = float(np.median(t))
    row[f'{key}_ms_min'] = float(min(t))
    row[f'{key}_ms_max'] = float(max(t))


def kernel_times(fn):
    """Device time (ms) of the FGR kernels in one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ('k_fgr_prepare', 'k_fgr_solve'):
            if k in e.key:
                out[k + '_ms'] = out.get(k + '_ms', 0.0) + e.device_time_total / 1e3
    return out


def main(argv=None):
    opt = parser().parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('bench_fgr.py needs a CUDA device')
    name, power = card()
    V = opt.voxel
    s_all, t_all, fs_all, ft_all = features(V)
    rows = []
    for B in (1, 8):
        pick = [b % len(FIXTURES) for b in range(B)]
        s, t = [s_all[k] for k in pick], [t_all[k] for k in pick]
        fs, ft = [fs_all[k] for k in pick], [ft_all[k] for k in pick]
        src64 = [x.to(torch.float64) for x in s]
        fgr_kw = dict(maximum_correspondence_distance=0.5 * V, tuple_test=True)
        match = lambda: ops.feature_match(fs, ft, t, True, 0)
        _, corr_tgt, mask, _ = match()
        solve = lambda: ops.fgr(s, t, src64, corr_tgt, mask, **fgr_kw)
        whole = lambda: ops.fgr_feature_matching(s, t, fs, ft, maximum_correspondence_distance=0.5 * V)
        ransac = lambda: ops.ransac_feature_matching(s, t, fs, ft, True, 1.5 * V, max_iteration=opt.iters,
                                                     distance=1.5 * V)
        for fn in (match, solve, whole, ransac):
            fn()
        torch.cuda.synchronize()
        _, res, n_mut = whole()
        _, rres, _ = ransac()
        row = dict(B=B, voxel=V, n_src=float(np.mean([x.shape[0] for x in s])),
                   n_tgt=float(np.mean([x.shape[0] for x in t])), n_mutual=float(n_mut.float().mean()),
                   fgr_correspondences=float(res[:, 0].mean()), fgr_trials=float(res[:, 2].mean()),
                   ransac_hypotheses=float(rres[:, 2].mean()))
        stats(row, 'fgr', timed(whole, opt.reps))
        stats(row, 'fgr_match', timed(match, opt.reps))
        stats(row, 'fgr_solve', timed(solve, opt.reps))
        stats(row, 'ransac', timed(ransac, opt.reps))
        row.update(kernel_times(solve))
        rows.append(row)
        print(json.dumps(row), flush=True)
    summary = dict(card=name, power_limit=power, reps=opt.reps, iters=opt.iters)
    print(json.dumps(summary))
    if opt.out:
        with open(opt.out, 'w') as fh:
            fh.write(''.join(json.dumps(r) + '\n' for r in rows + [summary]))


if __name__ == '__main__':
    main()
