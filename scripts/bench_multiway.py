"""Time multiway registration on a synthetic scene of 3DMatch-sized fragments (~20k points each).

    python scripts/bench_multiway.py [--n 60] [--batch_pairs 8] [--reps 3]

Reports, in one JSON line with the card's name and power limit:
  register_pairs_per_s   RegTR (random weights, 3dmatch config) on all N (N - 1) / 2 pairs, eager forwards of
                         --batch_pairs pairs (`multiway.register_pairs`);
  information_kernel_ms_per_pair  the `regtr_registration_information` launches alone on all pairs in batches of 64
                         (clouds stacked and matches from `ops.overlap_nn` prepared beforehand), per pair;
  registration_information_op_ms_per_pair  the whole `ops.registration_information` call per pair: stacking the
                         host clouds on the device, the overlap search (6 launches), the fit and the information kernel;
  optimize_ms_n60_all_pairs  `ops.pose_graph_optimize` on an N = 60 graph with every pair an edge (10 % wrong);
  optimize_ms_n256         on an N = 256 chain with loop closures to the next three nodes (10 % wrong).
All timings use CUDA events after one warm-up call.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests'))

import posegraph_oracle as PG  # noqa: E402
from regtr_b200 import lib  # noqa: E402
from regtr_b200 import multiway as M  # noqa: E402
from regtr_b200 import ops  # noqa: E402
from regtr_b200 import synthetic as S  # noqa: E402


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in q.split(',')]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=60)
    ap.add_argument('--batch_pairs', type=int, default=8)
    ap.add_argument('--reps', type=int, default=3)
    opt = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_multiway needs a GPU')
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.weights import random_state_dict
    cfg = get_config('3dmatch')
    model = RegTR(cfg).cuda().eval()
    model.load_state_dict(random_state_dict(cfg, 3), strict=True)
    sc = S.make_scene(0, opt.n, n_target=70000)       # ~20k points per fragment at N = 60
    frags = [f.astype(np.float64) for f in sc['fragments']]
    n_pairs = opt.n * (opt.n - 1) // 2
    reg_ms = timed(lambda: M.register_pairs(model, frags, opt.batch_pairs), 1)
    pairs = M.all_pairs(opt.n)
    T = np.stack([PG.rinv(sc['poses'][i]) @ sc['poses'][j] for i, j in pairs])[:, :3]

    def info_all():
        for a in range(0, n_pairs, 64):
            c = pairs[a:a + 64]
            ops.registration_information([frags[j] for _, j in c], [frags[i] for i, _ in c],
                                         torch.from_numpy(T[a:a + len(c)].copy()).cuda(), 0.0375, ops.new_status('cuda'))
    info_op_ms = timed(info_all, opt.reps)

    L = lib.load()
    status = ops.new_status('cuda')
    batches = []
    for a in range(0, n_pairs, 64):
        c = pairs[a:a + 64]
        xyz, offs, lens = ops._stack_pairs([frags[j] for _, j in c], [frags[i] for i, _ in c], 'bench')
        pose = torch.from_numpy(T[a:a + len(c)].copy()).cuda()
        nn = ops.overlap_nn(xyz, offs, len(c), pose, 0.0375, status)
        out = torch.empty((len(c), 6, 6), dtype=torch.float64, device='cuda')
        batches.append((xyz, offs, len(c), sum(lens), pose, nn, out))

    def info_kernels():
        for xyz, offs, B, n, pose, nn, out in batches:
            lib.check(L.regtr_registration_information(xyz.data_ptr(), offs.data_ptr(), B, n, pose.data_ptr(), 0.0375,
                                                       nn.data_ptr(), out.data_ptr(), status.data_ptr(), ops._stream()),
                      'regtr_registration_information')
    info_kernel_ms = timed(info_kernels, 10 * opt.reps)
    if int(status.item()):
        raise SystemExit(f'overlap search / information status {int(status.item()):#x}')
    out = {}
    for key, g in (('optimize_ms_n60_all_pairs', PG.noisy_graph(1, 60, all_pairs=True, wrong_frac=0.1, n_pts=60)),
                   ('optimize_ms_n256', PG.noisy_graph(2, 256, loop_span=3, wrong_frac=0.1, n_pts=60))):
        args = ([g['init']], [g['edges']], [g['X']], [g['info']], [g['uncertain']], 0.05)
        res = ops.pose_graph_optimize(*args)[3]
        out[key] = timed(lambda: ops.pose_graph_optimize(*args, status=ops.new_status('cuda')), opt.reps)
        out[key.replace('optimize_ms', 'iterations')] = res[0, :2].cpu().numpy().astype(int).tolist()
        out[key.replace('optimize_ms', 'edges')] = int(len(g['edges']))
    name, power = card()
    line = dict(gpu=name, power_limit=power, n_fragments=opt.n, pairs=n_pairs,
                mean_points=float(np.mean([len(f) for f in frags])),
                register_pairs_per_s=n_pairs / (reg_ms / 1e3),
                information_kernel_ms_per_pair=info_kernel_ms / n_pairs,
                registration_information_op_ms_per_pair=info_op_ms / n_pairs, **out)
    print(json.dumps(line))


if __name__ == '__main__':
    main()
