"""Score existing est.log files on the 3DMatch / 3DLoMatch benchmark (the reference's `evaluate_3dmatch.py`):

    python scripts/evaluate_3dmatch.py --results_dir <dir> [--benchmark 3DMatch|3DLoMatch] \
        [--gt datasets/3dmatch/benchmarks] [--use_dgr]

Reads <results_dir>/<benchmark>/<scene>/est.log (as written by scripts/eval_3dmatch.py) against
<gt>/<benchmark>/<scene>/gt.log and gt.info, and prints the reference's summary: Predator's registration recall, or
with --use_dgr the Deep Global Registration success rate (RRE < 15 deg, RTE < 30 cm).  Per-pair errors go to
<results_dir>/individual_errors.csv (individual_errors_dgr.csv with --use_dgr); the recall mode also leaves
flag.npy / errors.npy in every scene folder, as the reference does."""
import argparse
import csv
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from regtr_b200 import eval as E  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--results_dir', type=str, default='../logdev', help='Path to results (estimated transforms)')
ap.add_argument('--benchmark', choices=['3DMatch', '3DLoMatch'], default='3DMatch')
ap.add_argument('--gt', type=str, default=os.path.join('datasets', '3dmatch', 'benchmarks'),
                help='Directory holding the 3DMatch / 3DLoMatch ground-truth folders')
ap.add_argument('--use_dgr', action='store_true', help='If set, will evaluate using DGR success metrics (<15deg, 30cm)')
opt = ap.parse_args()

benchmark_dir = os.path.join(opt.gt, opt.benchmark)
results_dir = os.path.join(opt.results_dir, opt.benchmark)
if opt.use_dgr:
    out, per_scene = E.benchmark_dgr(results_dir, benchmark_dir)
    with open(os.path.join(opt.results_dir, 'individual_errors_dgr.csv'), 'w', newline='') as fh:
        w = csv.writer(fh)
        w.writerow(['scene', 'index', 'rre', 'rte', 'success'])
        for scene, d in per_scene.items():
            for i in range(len(d['rre'])):
                w.writerow([scene, i, repr(float(d['rre'][i])), repr(float(d['rte'][i])), int(d['success'][i])])
else:
    out, recall, per_scene = E.benchmark_3dmatch(results_dir, benchmark_dir, save_flags=True)
    with open(os.path.join(opt.results_dir, 'individual_errors.csv'), 'w', newline='') as fh:
        w = csv.writer(fh)
        w.writerow(['scene', 'src', 'tgt', 'errors'])
        for scene in per_scene:
            pairs, _ = E.read_trajectory(os.path.join(results_dir, scene, 'est.log'))
            for (src, tgt, _), err in zip(pairs, per_scene[scene]['errors']):
                w.writerow([scene, src, tgt, repr(float(err))])
print(out)
