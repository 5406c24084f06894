"""Time ICP (`ops.icp`) on synthetic 3DMatch-shaped pairs (~20k points per cloud), starting from the ground truth
perturbed by a few degrees and centimetres, at B = 1 and B = 8; and the float64 CPU oracle (tests/icp_oracle.py,
tests/icp_plane_oracle.py, tests/gicp_oracle.py, tests/colored_icp_oracle.py) on the same inputs.

    python scripts/bench_icp.py [--method point_to_point|point_to_plane|generalized|colored] [--iters 30]
        [--radius 0.0375] [--normal_radius 2R] [--normal_max_nn 30] [--epsilon 1e-3] [--lambda_geometric 0.968]
        [--loss l2|huber|cauchy|gm|tukey --loss_k K] [--blocks 7] [--reps 10]

CUDA events after warm-up: `--blocks` blocks of `--reps` calls each; the median and the spread (min..max) of the
per-call block means.  With point_to_plane, the targets' normal estimation (`ops.estimate_normals`) and the ICP are
timed separately, and the iterations each pair needed are reported under both methods.  With generalized, the normal
estimation of both clouds of every pair (one call) and the ICP are timed separately, L2 point-to-plane ICP on the same
target normals is timed too, and the iterations each pair needed are reported under all three methods and for the
oracle.  With colored, the synthetic pairs (which have no colour) are coloured by the tests' procedural texture
(tests/colored_icp_oracle.py: a smooth function of world position, the source taken after its ground-truth pose); the
targets' normal estimation, their colour gradients (`ops.color_gradients`, radius 2 R, 30 neighbours, as
`eval.icp_refine` uses) and the colored ICP are timed separately, L2 point-to-plane ICP on the same target normals is
timed too, and the iterations are reported under both and for the oracle.  --loss applies to every method but
point_to_point.  Prints one JSON line with the card name and power limit read in the same run."""
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


def pair_colours(B, seed0=7000):
    """The procedural colours (src_rgb, tgt_rgb) of `perturbed_pairs(B, seed0)`, from each pair's ground truth."""
    import colored_icp_oracle as C
    out = []
    for b in range(B):
        p = make_3dmatch_pair(seed0 + b)
        out.append(C.colour_pair(p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), p['pose']))
    return out


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in q.split(',')[:2]]
    except Exception:                       # noqa: BLE001 -- no nvidia-smi: the name from torch, power unknown
        name, power = torch.cuda.get_device_name(0), 'unknown'
    return name, power


def time_calls(call, radius, what, blocks, reps):
    """call(status) -> result: (per-call ms of each block, launches of one call, the result of one call)."""
    dev = torch.device('cuda:0')
    status = ops.new_status(dev)
    for _ in range(3):
        call(status)
    torch.cuda.synchronize()
    ops.check_fit_status(status, radius, what)
    before = ops.LAUNCHES
    res = call(status)
    launches = ops.LAUNCHES - before
    per_call = []
    for _ in range(blocks):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call(status)
        b.record()
        b.synchronize()
        per_call.append(a.elapsed_time(b) / reps)
    ops.check_fit_status(status, radius, what)
    return per_call, launches, res


def time_device(pairs, iters, radius, blocks, reps, method='point_to_point', normal_radius=None, normal_max_nn=30,
                epsilon=1e-3, loss='l2', loss_k=None, colours=None, lambda_geometric=0.968):
    """-> dict of the timings of one batch (ms per call, launches) and the iterations each pair needed, the normals
    and the colour gradients (host arrays, None where the method takes none)."""
    dev = torch.device('cuda:0')
    src = [torch.from_numpy(s).to(dev) for s, _, _ in pairs]
    tgt = [torch.from_numpy(t).to(dev) for _, t, _ in pairs]
    init = torch.from_numpy(np.stack([p for _, _, p in pairs])).to(dev)
    B = len(pairs)
    out = {}
    normals = src_normals = None
    if method != 'point_to_point':
        clouds = src + tgt if method == 'generalized' else tgt
        ms, launches, normals = time_calls(lambda st: ops.estimate_normals(clouds, normal_radius, normal_max_nn, st),
                                           normal_radius, 'estimate_normals', blocks, reps)
        out.update(normals_ms_median=float(np.median(ms)), normals_ms_min=float(min(ms)),
                   normals_ms_max=float(max(ms)), normals_launches_per_call=launches)
        if method == 'generalized':
            src_normals, normals = normals[:B], normals[B:]
        _, p2p = ops.icp(src, tgt, init, radius, iters)
        out['iterations_needed_point_to_point'] = [int(v) for v in p2p[:, 3].cpu().numpy()]
    colour_kw = {}
    if method == 'colored':
        scol = [torch.from_numpy(s).to(dev) for s, _ in colours]
        tcol = [torch.from_numpy(t).to(dev) for _, t in colours]
        gr = 2.0 * radius
        ms, launches, grads = time_calls(lambda st: ops.color_gradients(tgt, normals, tcol, gr, 30, st), gr,
                                         'color_gradients', blocks, reps)
        out.update(gradients_ms_median=float(np.median(ms)), gradients_ms_min=float(min(ms)),
                   gradients_ms_max=float(max(ms)), gradients_launches_per_call=launches)
        colour_kw = dict(src_colors=scol, tgt_colors=tcol, tgt_color_gradients=grads, lambda_geometric=lambda_geometric)
    if method in ('generalized', 'colored'):      # L2 point-to-plane on the same target normals, for comparison
        ms, _, (_, res) = time_calls(
            lambda st: ops.icp(src, tgt, init, radius, iters, status=st, method='point_to_plane', tgt_normals=normals),
            radius, 'icp', blocks, reps)
        out.update(point_to_plane_ms_median=float(np.median(ms)), point_to_plane_ms_min=float(min(ms)),
                   point_to_plane_ms_max=float(max(ms)),
                   iterations_needed_point_to_plane=[int(v) for v in res[:, 3].cpu().numpy()])
    ms, launches, (_, res) = time_calls(
        lambda st: ops.icp(src, tgt, init, radius, iters, status=st, method=method, tgt_normals=normals,
                           src_normals=src_normals, epsilon=epsilon, loss=loss, loss_k=loss_k, **colour_kw), radius,
        'icp', blocks, reps)
    res = res.cpu().numpy()
    out.update(gpu_ms_median=float(np.median(ms)), gpu_ms_min=float(min(ms)), gpu_ms_max=float(max(ms)),
               launches_per_call=launches, iterations_needed=[int(v) for v in res[:, 3]],
               fitness=[round(float(v), 4) for v in res[:, 0]])
    host = lambda ns: [n.cpu().numpy() for n in ns] if ns is not None else None
    return out, host(normals), host(src_normals), host(colour_kw.get('tgt_color_gradients'))


def parser():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--radius', type=float, default=0.0375)
    ap.add_argument('--blocks', type=int, default=7)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--cpu-reps', type=int, default=1)
    ap.add_argument('--method', choices=ops.ICP_METHODS, default='point_to_point')
    ap.add_argument('--normal_radius', type=float, help='default: 2 * --radius')
    ap.add_argument('--normal_max_nn', type=int, default=30)
    ap.add_argument('--epsilon', type=float, default=1e-3, help='covariance epsilon of generalized ICP')
    ap.add_argument('--lambda_geometric', type=float, default=0.968, help='geometric weight of colored ICP')
    ap.add_argument('--loss', choices=ops.ICP_LOSSES, default='l2')
    ap.add_argument('--loss_k', type=float)
    return ap


def main():
    opt = parser().parse_args()
    import colored_icp_oracle as C
    import gicp_oracle as G
    import icp_oracle as I
    import icp_plane_oracle as N
    nr = 2.0 * opt.radius if opt.normal_radius is None else opt.normal_radius
    name, power = card()
    out = {'card': name, 'power_limit': power, 'method': opt.method, 'iters': opt.iters, 'radius': opt.radius}
    if opt.method != 'point_to_point':
        out.update(normal_radius=nr, normal_max_nn=opt.normal_max_nn, loss=opt.loss, loss_k=opt.loss_k)
    if opt.method == 'generalized':
        out['epsilon'] = opt.epsilon
    if opt.method == 'colored':
        out.update(lambda_geometric=opt.lambda_geometric, gradient_radius=2.0 * opt.radius, gradient_max_nn=30)
    for B in (1, 8):
        pairs = perturbed_pairs(B)
        colours = pair_colours(B) if opt.method == 'colored' else None
        row, normals, src_normals, _ = time_device(pairs, opt.iters, opt.radius, opt.blocks, opt.reps, opt.method,
                                                   nr, opt.normal_max_nn, opt.epsilon, opt.loss, opt.loss_k, colours,
                                                   opt.lambda_geometric)
        cpu = []
        for _ in range(opt.cpu_reps):
            t0 = time.perf_counter()
            if opt.method == 'generalized':           # the oracle's own normals and GICP
                nrm = [N.estimate_normals(c, nr, opt.normal_max_nn)[0] for c in
                       [s for s, _, _ in pairs] + [t for _, t, _ in pairs]]
                _, ores = G.icp_batch([s for s, _, _ in pairs], [t for _, t, _ in pairs], nrm[B:],
                                      np.stack([p for _, _, p in pairs]), opt.radius, opt.iters,
                                      src_normals_list=nrm[:B], epsilon=opt.epsilon, loss=opt.loss,
                                      loss_k=opt.loss_k)
                row['iterations_needed_oracle'] = [int(v) for v in ores[:, 3]]
            elif opt.method == 'colored':             # the oracle's own normals, gradients and colored ICP
                tgts = [t for _, t, _ in pairs]
                nrm = [N.estimate_normals(t, nr, opt.normal_max_nn)[0] for t in tgts]
                grd = [C.color_gradients(t, n, c[1], 2.0 * opt.radius, 30) for t, n, c in zip(tgts, nrm, colours)]
                _, ores = C.icp_batch([s for s, _, _ in pairs], tgts, nrm, [c[0] for c in colours],
                                      [c[1] for c in colours], grd, np.stack([p for _, _, p in pairs]), opt.radius,
                                      opt.iters, lambda_geometric=opt.lambda_geometric, loss=opt.loss,
                                      loss_k=opt.loss_k)
                row['iterations_needed_oracle'] = [int(v) for v in ores[:, 3]]
            elif opt.method == 'point_to_plane':      # the oracle's own normals and ICP
                nrm = [N.estimate_normals(t, nr, opt.normal_max_nn)[0] for _, t, _ in pairs]
                _, ores = G.icp_batch([s for s, _, _ in pairs], [t for _, t, _ in pairs], nrm,
                                      np.stack([p for _, _, p in pairs]), opt.radius, opt.iters,
                                      method='point_to_plane', loss=opt.loss, loss_k=opt.loss_k)
                row['iterations_needed_oracle'] = [int(v) for v in ores[:, 3]]
            else:
                I.icp_batch([s for s, _, _ in pairs], [t for _, t, _ in pairs], np.stack([p for _, _, p in pairs]),
                            opt.radius, opt.iters)
            cpu.append((time.perf_counter() - t0) * 1e3)
        out[f'B{B}'] = dict({'points_per_cloud': int(np.mean([len(s) for s, _, _ in pairs] +
                                                             [len(t) for _, t, _ in pairs]))}, **row,
                            cpu_oracle_ms_median=float(np.median(cpu)))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
