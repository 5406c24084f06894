"""Time the outlier filters (regtr_statistical_outlier, regtr_radius_outlier) and their compaction
(regtr_select_points) on the real 3DMatch fixture clouds (tests/golden/real/*_input.npz, 17-25k points each) at B = 1
and B = 8, and on a seeded synthetic scan of ~300k points with 1 % uniform outliers (tests/outlier_oracle.py).

    python scripts/bench_outliers.py [--k 20 --std 2.0] [--nb 16 --radius 0.05] [--blocks 7] [--reps 10]

Each C entry is called directly on device buffers (no host work in the window): CUDA events after warm-up, `--blocks`
blocks of `--reps` calls each, the median and the spread (min..max) of the per-call block means.  The whole
`ops.remove_statistical_outlier` / `ops.remove_radius_outlier` call (stacking, filter, compaction and the read of the
row counts) is timed with a host clock around synchronised calls.  On the synthetic scan it reports the fraction of
injected outliers removed and of inliers lost by each filter, and scipy's cKDTree on the host (`query(k)` and
`query_ball_point(return_length=True)`, then the same rule in numpy) as a CPU reference when scipy is present.  Prints
one JSON line with the card name and power limit read in the same run."""
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

from regtr_b200 import lib, ops

FIXTURES = ['real_3dmatch_redkitchen_0_5', 'real_3dmatch_sun3d_home_38_41', 'real_3dmatch_sun3d_hotel3_8_15']


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')[:2]]
    except Exception:                       # noqa: BLE001 -- no nvidia-smi: the name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def time_call(call, blocks, reps):
    """-> {'ms': median per-call ms, 'min', 'max'} over blocks of reps calls, after warm-up."""
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    per = []
    for _ in range(blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call()
        b.record()
        b.synchronize()
        per.append(a.elapsed_time(b) / reps)
    return {'ms': round(float(np.median(per)), 4), 'min': round(min(per), 4), 'max': round(max(per), 4)}


def time_host(call, blocks):
    for _ in range(2):
        call()
    per = []
    for _ in range(blocks):
        torch.cuda.synchronize()
        t = time.perf_counter()
        call()
        torch.cuda.synchronize()
        per.append((time.perf_counter() - t) * 1e3)
    return {'ms': round(float(np.median(per)), 4), 'min': round(min(per), 4), 'max': round(max(per), 4)}


def bench_set(clouds, opt):
    """Kernel times of the three C entries on one stack, and the whole ops calls."""
    L = lib.load()
    dev = torch.device('cuda:0')
    lens = [c.shape[0] for c in clouds]
    n, C = sum(lens), len(clouds)
    xyz = torch.from_numpy(np.concatenate(clouds)).to(dev)
    offs = ops.make_offsets(lens, dev)
    status = ops.new_status(dev)
    avg = torch.empty(n, dtype=torch.float64, device=dev)
    keep = torch.empty(n, dtype=torch.int32, device=dev)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    stats = torch.empty((C, 3), dtype=torch.float64, device=dev)
    ws = ops.workspace(L.regtr_outlier_ws_bytes(n, C), dev)
    state = ops.workspace(L.regtr_outlier_state_bytes(n), dev, 'scan_state', zero=True)
    cell = ops.knn_cell(xyz, max(lens), opt.k)
    st = torch.cuda.current_stream().cuda_stream

    def stat():
        lib.check(L.regtr_statistical_outlier(xyz.data_ptr(), offs.data_ptr(), C, n, opt.k, opt.std, cell,
                                              avg.data_ptr(), keep.data_ptr(), stats.data_ptr(), status.data_ptr(),
                                              ws.data_ptr(), ws.numel(), state.data_ptr(), state.numel(), st), 'stat')

    def rad():
        lib.check(L.regtr_radius_outlier(xyz.data_ptr(), offs.data_ptr(), C, n, opt.nb, opt.radius,
                                         ops.overlap_cell(opt.radius), counts.data_ptr(), keep.data_ptr(),
                                         status.data_ptr(), ws.data_ptr(), ws.numel(), state.data_ptr(),
                                         state.numel(), st), 'radius')

    out = torch.empty((n, 3), dtype=torch.float64, device=dev)
    index = torch.empty(n, dtype=torch.int32, device=dev)
    out_offs = torch.empty(C + 1, dtype=torch.int32, device=dev)
    sws = ops.workspace(L.regtr_select_points_ws_bytes(n), dev, 'select')
    sstate = ops.workspace(L.regtr_select_points_state_bytes(n), dev, 'scan_state', zero=True)

    def select():
        lib.check(L.regtr_select_points(xyz.data_ptr(), None, keep.data_ptr(), offs.data_ptr(), C, n, out.data_ptr(),
                                        None, index.data_ptr(), out_offs.data_ptr(), sws.data_ptr(), sws.numel(),
                                        sstate.data_ptr(), sstate.numel(), st), 'select')

    res = {'clouds': C, 'points': n, 'knn_cell': cell,
           'statistical': time_call(stat, opt.blocks, opt.reps),
           'radius': time_call(rad, opt.blocks, opt.reps),
           'select': time_call(select, opt.blocks, opt.reps),
           'ops_statistical': time_host(lambda: ops.remove_statistical_outlier(clouds, opt.k, opt.std), opt.blocks),
           'ops_radius': time_host(lambda: ops.remove_radius_outlier(clouds, opt.nb, opt.radius), opt.blocks)}
    torch.cuda.synchronize()
    if int(status.item()):
        raise RuntimeError(f'status {int(status.item()):#x}')
    return res


def cpu_reference(xyz, opt):
    """scipy cKDTree on the host: the kNN averages and the statistical rule, and the radius counts."""
    try:
        from scipy.spatial import cKDTree
    except ImportError:
        return None
    t = time.perf_counter()
    tree = cKDTree(xyz)
    dist, _ = tree.query(xyz, k=opt.k)
    avg = dist.mean(1)
    m, sd = avg.mean(), avg.std(ddof=1)
    keep_stat = avg < m + opt.std * sd
    t_stat = time.perf_counter() - t
    t = time.perf_counter()
    tree = cKDTree(xyz)
    keep_rad = tree.query_ball_point(xyz, opt.radius, return_length=True) >= opt.nb
    t_rad = time.perf_counter() - t
    return {'statistical_ms': round(t_stat * 1e3, 1), 'radius_ms': round(t_rad * 1e3, 1),
            'kept_statistical': int(keep_stat.sum()), 'kept_radius': int(keep_rad.sum())}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--k', type=int, default=20, help='statistical filter: nb_neighbors')
    ap.add_argument('--std', type=float, default=2.0, help='statistical filter: std_ratio')
    ap.add_argument('--nb', type=int, default=16, help='radius filter: nb_points')
    ap.add_argument('--radius', type=float, default=0.05, help='radius filter: radius')
    ap.add_argument('--blocks', type=int, default=7)
    ap.add_argument('--reps', type=int, default=10)
    opt = ap.parse_args(argv)
    import outlier_oracle as O
    if not torch.cuda.is_available():
        raise SystemExit('bench_outliers.py needs a CUDA device')
    name, power = card()
    real = []
    for f in FIXTURES:
        d = np.load(os.path.join(ROOT, 'tests', 'golden', 'real', f + '_input.npz'))
        real += [d['src_xyz'].astype(np.float64), d['tgt_xyz'].astype(np.float64)]
    out = {'card': name, 'power_limit': power, 'k': opt.k, 'std_ratio': opt.std, 'nb_points': opt.nb,
           'radius': opt.radius}
    out['real_B1'] = bench_set(real[:1], opt)
    out['real_B8'] = bench_set((real * 2)[:8], opt)
    xyz, mask = O.outlier_scan(2026)
    out['scan_300k'] = bench_set([xyz], opt)
    for what, fn, args in (('statistical', ops.remove_statistical_outlier, (opt.k, opt.std)),
                           ('radius', ops.remove_radius_outlier, (opt.nb, opt.radius))):
        kept = np.zeros(xyz.shape[0], bool)
        kept[fn([xyz], *args)[2][0].cpu().numpy()] = True
        out['scan_300k'][f'{what}_outliers_removed'] = round(float((~kept[mask]).mean()), 4)
        out['scan_300k'][f'{what}_inliers_lost'] = round(float((~kept[~mask]).mean()), 5)
    out['scan_300k']['cpu_ckdtree'] = cpu_reference(xyz, opt)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
