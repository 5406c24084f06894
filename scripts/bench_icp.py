"""Time point-to-point ICP (`ops.icp`) on synthetic 3DMatch-shaped pairs (~20k points per cloud), starting from the
ground truth perturbed by a few degrees and centimetres, at B = 1 and B = 8; and the float64 CPU oracle
(tests/icp_oracle.py) on the same inputs.

    python scripts/bench_icp.py [--iters 30] [--radius 0.0375] [--blocks 7] [--reps 10]

CUDA events after warm-up: `--blocks` blocks of `--reps` calls each; the median and the spread (min..max) of the
per-call block means.  Prints one JSON line with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import numpy as np
import torch

from regtr_b200 import ops
from regtr_b200.synthetic import make_3dmatch_pair


def perturbed_pairs(B, seed0=7000, deg=4.0, metres=0.04):
    import icp_oracle as I
    import train_data_oracle as O
    out = []
    for b in range(B):
        p = make_3dmatch_pair(seed0 + b)
        rng = np.random.default_rng(seed0 + b)
        axis = rng.normal(size=3)
        d = np.eye(3, 4)
        d[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
        d[:, 3] = rng.normal(size=3) * metres / np.sqrt(3.0)
        out.append((p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), I.compose(d, p['pose'])))
    return out


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')[:2]]
    except Exception:                       # noqa: BLE001 -- no nvidia-smi: the name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def time_device(pairs, iters, radius, blocks, reps):
    dev = torch.device('cuda:0')
    src = [torch.from_numpy(s).to(dev) for s, _, _ in pairs]
    tgt = [torch.from_numpy(t).to(dev) for _, t, _ in pairs]
    init = torch.from_numpy(np.stack([p for _, _, p in pairs])).to(dev)
    status = ops.new_status(dev)
    for _ in range(3):
        ops.icp(src, tgt, init, radius, iters, status=status)
    torch.cuda.synchronize()
    ops.check_fit_status(status, radius, 'icp')
    before = ops.LAUNCHES
    _, res = ops.icp(src, tgt, init, radius, iters, status=status)
    launches = ops.LAUNCHES - before
    per_call = []
    for _ in range(blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            ops.icp(src, tgt, init, radius, iters, status=status)
        b.record()
        b.synchronize()
        per_call.append(a.elapsed_time(b) / reps)
    ops.check_fit_status(status, radius, 'icp')
    return per_call, launches, res.cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--radius', type=float, default=0.0375)
    ap.add_argument('--blocks', type=int, default=7)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--cpu-reps', type=int, default=1)
    opt = ap.parse_args()
    import icp_oracle as I
    name, power = card()
    out = {'card': name, 'power_limit': power, 'iters': opt.iters, 'radius': opt.radius}
    for B in (1, 8):
        pairs = perturbed_pairs(B)
        ms, launches, res = time_device(pairs, opt.iters, opt.radius, opt.blocks, opt.reps)
        cpu = []
        for _ in range(opt.cpu_reps):
            t0 = time.perf_counter()
            I.icp_batch([s for s, _, _ in pairs], [t for _, t, _ in pairs], np.stack([p for _, _, p in pairs]),
                        opt.radius, opt.iters)
            cpu.append((time.perf_counter() - t0) * 1e3)
        out[f'B{B}'] = {'points_per_cloud': int(np.mean([len(s) for s, _, _ in pairs] + [len(t) for _, t, _ in pairs])),
                        'gpu_ms_median': float(np.median(ms)), 'gpu_ms_min': float(min(ms)),
                        'gpu_ms_max': float(max(ms)), 'launches_per_call': launches,
                        'iterations_needed': [int(v) for v in res[:, 3]],
                        'fitness': [round(float(v), 4) for v in res[:, 0]],
                        'cpu_oracle_ms_median': float(np.median(cpu))}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
