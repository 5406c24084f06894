"""Time the preparation of 3DMatch training batches (regtr_b200.augment.TrainingPrep: overlap ground truth + the
reference's four augmentations) on the GPU, and the CPU route it replaces on one thread (data.compute_overlap with
scipy's cKDTree plus the float64 transforms of tests/train_data_oracle.py).

    python scripts/bench_train_data.py [--steps K] [--warmup W]

GPU arms: 1 and 8 synthetic ~20k-point pairs (synthetic.make_3dmatch_pair) and the two real benchmark pairs, host
inputs in pinned float64 memory, CUDA events around each call after W warm-up calls.  Prints one JSON line with the
card's name and power limit.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import train_data_oracle as O  # noqa: E402
from regtr_b200 import augment as A  # noqa: E402
from regtr_b200 import data as D  # noqa: E402
from regtr_b200.synthetic import make_3dmatch_pair  # noqa: E402

CFG = SimpleNamespace(overlap_radius=0.0375, perturb_pose='small', augment_noise=0.005)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def batch(pairs):
    return {'src_xyz': [torch.from_numpy(s).pin_memory() for s, _, _ in pairs],
            'tgt_xyz': [torch.from_numpy(t).pin_memory() for _, t, _ in pairs],
            'pose': torch.from_numpy(np.stack([p for _, _, p in pairs]))}


def time_gpu(pairs, steps, warmup):
    prep, b = A.TrainingPrep(CFG), batch(pairs)
    for _ in range(warmup):
        prep(b)
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        prep(b)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    prep.check()
    return float(np.median(ms)), float(min(ms))


def time_cpu(pairs, reps=3):
    torch.set_num_threads(1)
    rng = np.random.default_rng(0)
    best = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for s, t, p in pairs:
            sm, tm, corr = D.compute_overlap(s @ p[:, :3].T + p[:, 3], t, CFG.overlap_radius)
            d = dict(src_xyz=s, tgt_xyz=t, pose=p, src_overlap=sm, tgt_overlap=tm, correspondences=corr)
            d = O.rigid_perturb(d, O.pose_small(1.0, 0.3, 0.5, np.ones(3)), True, True)
            d = O.jitter(d, rng.normal(scale=0.005, size=s.shape), rng.normal(scale=0.005, size=t.shape))
            d = O.shuffle_points(d, rng.permutation(len(s))[:30000], rng.permutation(len(t))[:30000])
            O.random_swap(d, True)
        best.append((time.perf_counter() - t0) * 1e3 / len(pairs))
    return float(min(best))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'the GPU arms need cuda:0'
    name, power = card()
    synth = []
    for i in range(8):
        p = make_3dmatch_pair(900 + i)
        synth.append((p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), p['pose'].astype(np.float64)))
    real = [(s, t, p) for s, t, p, _ in O.real_pairs(os.path.join(ROOT, 'tests', 'golden'))]
    res = {'card': name, 'power_limit': power, 'steps': args.steps,
           'points_per_pair_synthetic': float(np.mean([len(s) + len(t) for s, t, _ in synth]))}
    for label, pairs in (('synthetic_1', synth[:1]), ('synthetic_8', synth), ('real_2', real)):
        med, best = time_gpu(pairs, args.steps, args.warmup)
        res[f'gpu_ms_{label}'] = round(med, 4)
        res[f'gpu_ms_{label}_min'] = round(best, 4)
        res[f'gpu_ms_per_pair_{label}'] = round(med / len(pairs), 4)
    res['cpu_ms_per_pair_synthetic_1thread'] = round(time_cpu(synth[:2]), 2)
    res['cpu_ms_per_pair_real_1thread'] = round(time_cpu(real), 2)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
