"""Time RANSAC over correspondences (`ops.ransac`) per pair at B = 1 and B = 8, on the real 3DMatch fixtures with a
gt.log pose and on synthetic 3DMatch-shaped pairs, with RegTR-like correspondences (keypoints of both clouds mapped
by the ground truth plus 1 cm of noise, a share of them ending at a random target point instead) at inlier ratios
0.5, 0.2 and 0.05, for max_iteration 1e3, 1e4 and 1e5.

    python scripts/bench_ransac.py [--radius 0.0375] [--m 1000] [--reps 5] [--data real,synthetic]
        [--ratios 0.5,0.2,0.05] [--iters 1000,10000,100000] [--out FILE]

CUDA events after one warm-up call: the median and the spread (min..max) of --reps calls, divided by B for ms per
pair.  Each row also reports the hypotheses walked and validated (mean over the pairs), the launch count of one
call, and the mean rotation / translation error of the poses.  One JSON line per row, then one summary line with the
card name and power limit read in the same run."""
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
from regtr_b200.synthetic import make_3dmatch_pair

REAL = os.path.join(ROOT, 'tests', 'golden', 'real')
FIXTURES = (('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
            ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3'))


def real_pairs():
    """(src, tgt, pose (3,4)) of the fixtures with a gt.log pose (entry (i, j) maps cloud_bin_j onto cloud_bin_i)."""
    out = []
    for fx, scene in FIXTURES:
        keys, traj = E.read_trajectory(os.path.join(REAL, 'benchmarks', '3DMatch', scene, 'gt.log'))
        inp = np.load(os.path.join(REAL, fx + '_input.npz'))
        a, b = inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)
        src_first = os.path.basename(str(inp['src_file'])) == f'cloud_bin_{int(keys[0][1])}.pth'
        out.append((a, b, traj[0][:3]) if src_first else (b, a, traj[0][:3]))
    return out


def synthetic_pairs(n=8):
    return [(p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), np.asarray(p['pose'], np.float64))
            for p in (make_3dmatch_pair(8000 + k) for k in range(n))]


def regtr_like(src, tgt, pose, m, inliers, seed, noise=0.01):
    """m two-way correspondences: m / 2 source keypoints -> their place in the target, m / 2 target keypoints <- their
    place in the source; a share 1 - inliers of them end at a random point of the other cloud."""
    rng = np.random.default_rng(seed)
    R, t = pose[:, :3], pose[:, 3]
    a_s = src[rng.integers(0, len(src), m // 2)]
    c_t = tgt[rng.integers(0, len(tgt), m - m // 2)]
    a = np.concatenate([a_s, (c_t - t) @ R])
    c = np.concatenate([a_s @ R.T + t, c_t]) + rng.normal(scale=noise / np.sqrt(3.0), size=(m, 3))
    bad = rng.random(m) >= inliers
    c[bad] = tgt[rng.integers(0, len(tgt), int(bad.sum()))]
    return a, c


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')[:2]]
    except Exception:                       # noqa: BLE001 -- no nvidia-smi: the name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def rot_trans_err(pose, gt):
    cos = (np.trace(pose[:, :3].T @ gt[:, :3]) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(cos, -1.0, 1.0)))), float(np.linalg.norm(pose[:, 3] - gt[:, 3]))


def parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--radius', type=float, default=0.0375)
    ap.add_argument('--m', type=int, default=1000, help='Correspondences per pair')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--data', default='real,synthetic')
    ap.add_argument('--ratios', default='0.5,0.2,0.05')
    ap.add_argument('--iters', default='1000,10000,100000')
    ap.add_argument('--out', help='Also write the JSON lines to this file')
    return ap


def main(argv=None):
    opt = parser().parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('bench_ransac.py needs a CUDA device')
    name, power = card()
    rows = []
    sources = {'real': real_pairs, 'synthetic': synthetic_pairs}
    for data in opt.data.split(','):
        base = sources[data]()
        for ratio in (float(v) for v in opt.ratios.split(',')):
            corr = [regtr_like(s, t, p, opt.m, ratio, 100 + k) for k, (s, t, p) in enumerate(base)]
            for iters in (int(v) for v in opt.iters.split(',')):
                for B in (1, 8):
                    idx = [k % len(base) for k in range(B)]
                    args = ([base[k][0] for k in idx], [base[k][1] for k in idx], [corr[k][0] for k in idx],
                            [corr[k][1] for k in idx], opt.radius, iters)
                    status = ops.new_status(torch.device('cuda'))
                    ops.ransac(*args, status=status)                                     # warm-up
                    times = []
                    for _ in range(opt.reps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        before = ops.LAUNCHES
                        e0.record()
                        pose, res = ops.ransac(*args, status=status)
                        e1.record()
                        torch.cuda.synchronize()
                        launches = ops.LAUNCHES - before
                        times.append(e0.elapsed_time(e1) / B)
                    ops.check_fit_status(status, opt.radius, 'ransac')
                    pose, res = pose.cpu().numpy(), res.cpu().numpy()
                    errs = np.array([rot_trans_err(pose[b], base[k][2]) for b, k in enumerate(idx)])
                    row = dict(data=data, inlier_ratio=ratio, max_iteration=iters, B=B,
                               ms_per_pair=float(np.median(times)), ms_min=float(min(times)),
                               ms_max=float(max(times)), walked=float(res[:, 2].mean()),
                               validations=float(res[:, 3].mean()), fitness=float(res[:, 0].mean()),
                               launches=launches, rot_err_deg=float(errs[:, 0].mean()),
                               trans_err=float(errs[:, 1].mean()))
                    rows.append(row)
                    print(json.dumps(row), flush=True)
    summary = dict(card=name, power_limit=power, radius=opt.radius, m=opt.m, reps=opt.reps)
    print(json.dumps(summary))
    if opt.out:
        with open(opt.out, 'w') as fh:
            fh.write(''.join(json.dumps(r) + '\n' for r in rows + [summary]))


if __name__ == '__main__':
    main()
