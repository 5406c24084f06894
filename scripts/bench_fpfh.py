"""Time the classical global registration (`eval.fpfh_register`'s stages) per stage at B = 1 and B = 8 on synthetic
3DMatch-shaped pairs, downsampled at 5 cm and at 2.5 cm (about 20k points, the full resolution of the 3DMatch
fragments), and the feature-match kernel's achieved FP64 rate.

    python scripts/bench_fpfh.py [--voxels 0.05,0.025] [--reps 5] [--iters 100000] [--out FILE]

Stages: downsample (`ops.grid_subsample`), normals (2 V, 30), fpfh (5 V, 100), match (`ops.feature_match` with the
mutual filter), ransac (1.5 V, distance checker 1.5 V, --iters, confidence 0.999).  CUDA events around each stage after
one warm-up run of every shape: the median and the spread (min..max) of --reps runs, in ms per call (all B pairs).
The feature match does 3 * 33 * n_s * n_t FP64 operations per pair (a subtract, a multiply and an add per feature
component, one sweep giving both directions); its rate is that count over the match time, set against 17 TFLOP/s, half
of the H100 SXM data sheet's 34 TFLOP/s FP64 (which counts an FMA as two operations: a contraction-free loop issues
three instructions for three operations).  One JSON line per row, then one summary line with the card name and power
limit read in the same run."""
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

FP64_NO_FMA = 17e12        # half of the data sheet's 34 TFLOP/s FP64 (non-tensor, FMA counted as two)


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
    ap.add_argument('--voxels', default='0.05,0.025')
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--iters', type=int, default=100000)
    ap.add_argument('--out', help='Also write the JSON lines to this file')
    return ap


def run_once(src, tgt, voxel, iters):
    """One registration, stage by stage: -> ({stage: ms}, (n_s, n_t) per pair, n_mutual)."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    B = len(src)
    ev[0].record()
    down = E.fpfh_downsample(src + tgt, voxel)
    ev[1].record()
    normals = ops.estimate_normals(down, 2 * voxel, 30)
    ev[2].record()
    feats = ops.fpfh(down, normals, 5 * voxel, 100)
    ev[3].record()
    corr_src, corr_tgt, mask, n_mut = ops.feature_correspondences(down[:B], down[B:], feats[:B], feats[B:])
    ev[4].record()
    r = 1.5 * voxel
    ops.ransac(down[:B], down[B:], corr_src, corr_tgt, r, iters, corr_mask=mask, distance=r)
    ev[5].record()
    torch.cuda.synchronize()
    names = ('downsample', 'normals', 'fpfh', 'match', 'ransac')
    ms = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}
    sizes = [(int(down[b].shape[0]), int(down[B + b].shape[0])) for b in range(B)]
    return ms, sizes, n_mut.cpu().numpy()


def main(argv=None):
    opt = parser().parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit('bench_fpfh.py needs a CUDA device')
    name, power = card()
    pairs = [make_3dmatch_pair(9000 + k) for k in range(8)]
    rows = []
    for voxel in (float(v) for v in opt.voxels.split(',')):
        for B in (1, 8):
            src = [p['src_xyz'].astype(np.float64) for p in pairs[:B]]
            tgt = [p['tgt_xyz'].astype(np.float64) for p in pairs[:B]]
            run_once(src, tgt, voxel, opt.iters)                                          # warm-up
            runs = [run_once(src, tgt, voxel, opt.iters) for _ in range(opt.reps)]
            sizes, n_mut = runs[0][1], runs[0][2]
            row = dict(voxel=voxel, B=B, n_src=float(np.mean([s for s, _ in sizes])),
                       n_tgt=float(np.mean([t for _, t in sizes])), n_mutual=float(n_mut.mean()))
            for k in runs[0][0]:
                t = [r[0][k] for r in runs]
                row[f'{k}_ms'] = float(np.median(t))
                row[f'{k}_ms_min'] = float(min(t))
                row[f'{k}_ms_max'] = float(max(t))
            flops = sum(3 * 33 * s * t for s, t in sizes)
            rate = flops / (row['match_ms'] * 1e-3)
            row.update(match_fp64_tflops=rate / 1e12, match_share_of_no_fma_peak=rate / FP64_NO_FMA,
                       match_floor_ms=flops / FP64_NO_FMA * 1e3)
            rows.append(row)
            print(json.dumps(row), flush=True)
    summary = dict(card=name, power_limit=power, reps=opt.reps, iters=opt.iters)
    print(json.dumps(summary))
    if opt.out:
        with open(opt.out, 'w') as fh:
            fh.write(''.join(json.dumps(r) + '\n' for r in rows + [summary]))


if __name__ == '__main__':
    main()
