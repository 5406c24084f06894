"""Register a whole scan sequence: every pair of fragments, a robust pose graph, one scene (Open3D's multiway
registration after RegTR's pairwise poses).

    python -m regtr_b200.multiway FRAG_0 FRAG_1 ... --ckpt <logdir>/ckpt/model-best.pth [--config <yaml>] --out DIR
        [--icp R [--icp_iters 30] [--icp_method point_to_point|point_to_plane|generalized|colored
         [--normal_radius NR] [--normal_max_nn 30] [--icp_epsilon 1e-3] [--icp_lambda_geometric 0.968]
         [--icp_loss l2|huber|cauchy|gm|tukey --icp_loss_k K]]]
        [--ransac R [--ransac_iters 100000] [--ransac_confidence 0.999] [--ransac_n 3] [--ransac_edge 0.9]
         [--ransac_dist D] [--ransac_overlap 0.5] [--ransac_seed 0]]
        [--fgr [--fgr_dist 0.025] [--fgr_iters 64] [--fgr_tuple_test] [--fgr_overlap 0.5] ...]
        [--info_radius D] [--min_overlap 0.3] [--preference_loop_closure 1.0]
        [--voxel V] [--batch_pairs 8]

Fragments are given in sequence order, in any format `pointio` reads; fragment index = position in the list (3DMatch
scenes are numbered cloud_bin_0..N-1, so position is the benchmark index).  The config is found and the clouds are
cropped as `register` does.  Every pair i < j is registered with source j and target i (the 3DMatch benchmark's
direction) in eager forwards of --batch_pairs pairs, then refined by `ops.icp` with --icp as `register --icp` does
(generalized ICP uses each fragment's normals as source and as target normals; colored ICP reads every fragment's PLY
colours, a fragment without them being a usage error, and takes its target's gradients at radius 2 R, 30 neighbours).  With --ransac R each pair's pose
first comes from RANSAC over the network's correspondences (`ops.ransac`, as `register --ransac`), so that far loop
closures with little overlap survive the network's outlier correspondences; ICP then starts from it.  --fgr does the
same with Fast Global Registration over those correspondences (`ops.fgr`, as `register --fgr`) instead of RANSAC.
`ops.registration_information` at D (default: the config's overlap_radius) gives each pair its fit and information
matrix.  Edge (source j, target i, X = the pair's pose): j = i + 1 is a certain odometry edge; any other pair is an
uncertain loop-closure edge when Lambda[5,5] / min(n_j, n_i) >= --min_overlap (Open3D's reconstruction system's gate).
Initial poses follow the odometry chain (P_0 = I, P_j = P_{j-1} X_{j->j-1}); `ops.pose_graph_optimize` with
max_correspondence_distance D then optimises the graph.
Outputs in DIR:
  result.npz           poses (N,4,4), edges (E,2), transformation (E,4,4), information (E,6,6), uncertain, confidence,
                       kept, pairs (P,2) = (i, j) and fit (P,4) of every registered pair, edge or not;
  <scene>/est.log      per pair i < j the header `i j -1` and pose P_i^-1 P_j (eval.EstLogWriter), <scene> the first
                       fragment's parent directory name: `--out logs/3DMatch` is scored by
                       `scripts/evaluate_3dmatch.py --results_dir logs`;
  scene.ply            with --voxel V: every fragment moved by its pose, concatenated and grid-subsampled at V
                       (a barycentre per voxel).
One JSON line on stdout: fragments, pairs, edges (odometry, loop, kept), iterations of both passes, final objective.
"""
from __future__ import annotations

import argparse
import json
import os
from pathlib import Path
from typing import Dict, List, Sequence

import numpy as np
import torch

from .eval import (add_fgr_arguments, add_icp_arguments, add_ransac_arguments, check_fgr_arguments,
                   check_icp_arguments, check_ransac_arguments, fgr_kwargs, fgr_refine, icp_refine, ransac_kwargs,
                   ransac_refine)


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog='python -m regtr_b200.multiway',
                                 description='Register a sequence of fragments into one scene with a trained RegTR.')
    ap.add_argument('fragments', nargs='+', help='Fragments in sequence order (.ply, .pth, .bin or .npy)')
    ap.add_argument('--ckpt', required=True, help='Checkpoint ({"state_dict": ...}), e.g. <logdir>/ckpt/model-best.pth')
    ap.add_argument('--config', help='Config file (default: config.yaml one level above the checkpoint directory)')
    ap.add_argument('--out', required=True, help='Output directory')
    add_icp_arguments(ap, 'Refine every pair by ICP, max correspondence distance R')
    add_ransac_arguments(ap, 'Replace every pair\'s pose by RANSAC over the predicted correspondences, max '
                             'correspondence distance R (before ICP with --icp)')
    add_fgr_arguments(ap, 'Replace every pair\'s pose by Fast Global Registration over the predicted correspondences '
                          'instead of RANSAC (before ICP with --icp)')
    ap.add_argument('--info_radius', type=float, metavar='D',
                    help='Radius of the information matrices and the line process (default: overlap_radius)')
    ap.add_argument('--min_overlap', type=float, default=0.3,
                    help='Loop-closure gate: matches / min(fragment sizes) at D')
    ap.add_argument('--preference_loop_closure', type=float, default=1.0, help='Line-process preference')
    ap.add_argument('--voxel', type=float, metavar='V', help='Write scene.ply, grid-subsampled at V')
    ap.add_argument('--batch_pairs', type=int, default=8, help='Pairs per forward')
    return ap


def all_pairs(n: int):
    """(i, j) for every i < j, in the order of 3DMatch's gt.log."""
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def register_pairs(model, fragments: Sequence[np.ndarray], batch_pairs: int = 8, icp_radius: float = None,
                   icp_iters: int = 30, icp_method: str = 'point_to_point', normal_radius: float = None,
                   normal_max_nn: int = 30, icp_epsilon: float = 1e-3, icp_loss: str = 'l2',
                   icp_loss_k: float = None, ransac_radius: float = None, ransac_options: Dict = None,
                   fgr_options: Dict = None, colors: Sequence[np.ndarray] = None,
                   icp_lambda_geometric: float = 0.968) -> np.ndarray:
    """RegTR's final-layer pose of every pair (i, j) of `all_pairs`, source j -> target i, optionally refined by ICP
    (`eval.icp_refine` with icp_method, epsilon=icp_epsilon, loss=icp_loss, loss_k=icp_loss_k; the point-to-plane and
    generalized methods use every fragment's normals, estimated once).
    With ransac_radius, the network's pose is first replaced by `eval.ransac_refine` at that radius (ransac_options:
    its further keyword arguments), pair p of `all_pairs` drawing as pair p whatever batch_pairs; ICP then starts from
    the RANSAC pose.  fgr_options (a dict, possibly empty): the same with `eval.fgr_refine` and these keyword arguments
    instead, pair p drawing its tuples as pair p.  colors: every fragment's (n,3) rgb, for icp_method='colored' (with
    icp_lambda_geometric).
    fragments: (n,3) float64 host arrays (already cropped).  -> (P,3,4) float64."""
    from . import ops
    dev = model.device
    pairs = all_pairs(len(fragments))
    dev_frags = [torch.from_numpy(np.ascontiguousarray(f)).float().to(dev) for f in fragments]
    normals = None
    if icp_radius is not None and icp_method != 'point_to_point':
        nr = 2.0 * icp_radius if normal_radius is None else normal_radius
        normals = ops.estimate_normals(fragments, nr, normal_max_nn)
    out = []
    with torch.no_grad():
        for a in range(0, len(pairs), batch_pairs):
            chunk = pairs[a:a + batch_pairs]
            pred = model({'src_xyz': [dev_frags[j] for _, j in chunk], 'tgt_xyz': [dev_frags[i] for i, _ in chunk]})
            pose = pred['pose'][-1].double()
            if ransac_radius is not None:
                pose, _ = ransac_refine(pred, [fragments[j] for _, j in chunk], [fragments[i] for i, _ in chunk],
                                        ransac_radius, pair_base=a, **(ransac_options or {}))
            if fgr_options is not None:
                pose, _ = fgr_refine(pred, [fragments[j] for _, j in chunk], [fragments[i] for i, _ in chunk],
                                     pair_base=a, **fgr_options)
            if icp_radius is not None:
                pose, _ = icp_refine([fragments[j] for _, j in chunk], [fragments[i] for i, _ in chunk], pose,
                                     icp_radius, icp_iters, icp_method, epsilon=icp_epsilon, loss=icp_loss,
                                     loss_k=icp_loss_k, normals=None if normals is None else
                                     ([normals[j] for _, j in chunk], [normals[i] for i, _ in chunk]),
                                     colors=None if colors is None else
                                     ([colors[j] for _, j in chunk], [colors[i] for i, _ in chunk]),
                                     lambda_geometric=icp_lambda_geometric)
            out.append(pose.cpu().numpy())
    return np.concatenate(out, 0)


def odometry_chain(X: Dict) -> np.ndarray:
    """P_0 = I, P_j = P_{j-1} X_{j->j-1}; X maps (j-1, j) to the (4,4) pose of that pair."""
    n = len(X) + 1
    P = np.tile(np.eye(4), (n, 1, 1))
    for j in range(1, n):
        P[j] = P[j - 1] @ X[(j - 1, j)]
    return P


def optimize_scene(fragments: Sequence[np.ndarray], pair_poses, info_radius: float, min_overlap: float = 0.3,
                   preference_loop_closure: float = 1.0, batch_pairs: int = 64, **options) -> Dict:
    """Everything after the network: information matrices, gating, graph and optimisation.
    fragments: N (n,3) arrays; pair_poses: (P,3,4) or (P,4,4) poses of `all_pairs(N)`, source j -> target i.
    options: further `ops.pose_graph_optimize` arguments.  -> dict of host arrays (the result.npz keys, plus result
    (4,) and the counts)."""
    from . import ops
    N = len(fragments)
    if N < 2:
        raise ValueError('optimize_scene: expected at least two fragments')
    frags = [np.asarray(f, np.float64) for f in fragments]
    pairs = all_pairs(N)
    T = np.asarray(pair_poses, np.float64)
    if T.shape[0] != len(pairs):
        raise ValueError(f'optimize_scene: {T.shape[0]} pair poses for {len(pairs)} pairs')
    T44 = np.tile(np.eye(4), (len(pairs), 1, 1))
    T44[:, :3] = T[:, :3]
    fit, info = [], []
    for a in range(0, len(pairs), batch_pairs):
        chunk = pairs[a:a + batch_pairs]
        f, inf = ops.registration_information([frags[j] for _, j in chunk], [frags[i] for i, _ in chunk],
                                              torch.from_numpy(T44[a:a + len(chunk), :3].copy()).cuda(), info_radius)
        fit.append(f.cpu().numpy())
        info.append(inf.cpu().numpy())
    fit, info = np.concatenate(fit), np.concatenate(info)
    edges, unc, n_odo, n_loop = [], [], 0, 0
    for p, (i, j) in enumerate(pairs):
        if j == i + 1:
            edges.append(p); unc.append(False); n_odo += 1
        elif info[p, 5, 5] / min(len(frags[j]), len(frags[i])) >= min_overlap:
            edges.append(p); unc.append(True); n_loop += 1
    edges = np.asarray(edges, np.int64)
    e_st = np.array([[pairs[p][1], pairs[p][0]] for p in edges], np.int64).reshape(-1, 2)   # (source j, target i)
    P0 = odometry_chain({pairs[p]: T44[p] for p in edges if pairs[p][1] == pairs[p][0] + 1})
    poses, conf, kept, result = ops.pose_graph_optimize([P0], [e_st], [T44[edges]], [info[edges]],
                                                        [np.asarray(unc, bool)], info_radius,
                                                        preference_loop_closure=preference_loop_closure, **options)
    P = np.tile(np.eye(4), (N, 1, 1))
    P[:, :3] = poses[0].cpu().numpy()
    r = result[0].cpu().numpy()
    return dict(poses=P, edges=e_st, transformation=T44[edges], information=info[edges],
                uncertain=np.asarray(unc, bool), confidence=conf[0].cpu().numpy(), kept=kept[0].cpu().numpy(),
                pairs=np.asarray(pairs, np.int64), fit=fit, result=r, n_odometry=n_odo, n_loop=n_loop)


def relative_pose(P: np.ndarray, i: int, j: int) -> np.ndarray:
    """P_i^-1 P_j: fragment j into fragment i, est.log's pose of entry (i, j)."""
    Ri, ti = P[i, :3, :3], P[i, :3, 3]
    inv = np.eye(4)
    inv[:3, :3], inv[:3, 3] = Ri.T, -Ri.T @ ti
    return inv @ P[j]


def write_outputs(res: Dict, out_dir: str, scene: str, fragments: Sequence[np.ndarray] = None, voxel: float = None):
    """result.npz, <scene>/est.log and, with voxel, scene.ply (see the module docstring)."""
    from . import ops
    from .eval import EstLogWriter
    from .pointio import write_ply
    os.makedirs(out_dir, exist_ok=True)
    np.savez(os.path.join(out_dir, 'result.npz'),
             **{k: res[k] for k in ('poses', 'edges', 'transformation', 'information', 'uncertain', 'confidence',
                                    'kept', 'pairs', 'fit')})
    log = os.path.join(out_dir, scene, 'est.log')
    if os.path.exists(log):
        os.remove(log)
    writer = EstLogWriter(out_dir, '')
    for i, j in res['pairs']:
        writer.append(scene, int(j), int(i), relative_pose(res['poses'], int(i), int(j)))
    if voxel is not None:
        moved, _ = ops.transform_clouds(fragments, res['poses'])
        status = ops.new_status(moved.device)
        one = ops.make_offsets([moved.shape[0]], moved.device)
        out, offs = ops.grid_subsample(moved.contiguous(), one, 1, voxel, status, dense=False)
        if int(status.item()):
            raise RuntimeError(f'scene.ply: grid sub-sampling at {voxel} failed (status {int(status.item()):#x})')
        write_ply(os.path.join(out_dir, 'scene.ply'), out[:int(offs[1])].cpu().numpy())


def scene_name(path: str) -> str:
    return Path(os.path.abspath(path)).parent.name


def main(argv=None):
    ap = parser()
    opt = ap.parse_args(argv)
    check_fgr_arguments(ap, opt)
    check_icp_arguments(ap, opt, colors=True)
    check_ransac_arguments(ap, opt)
    from .config import load_config
    from .eval import load_icp_colors
    from .pointio import load_point_cloud
    from .register import config_path, crop, crop_colors, load_model
    if len(opt.fragments) < 2:
        raise SystemExit('expected at least two fragments')
    colors = load_icp_colors(ap, opt, opt.fragments)
    cfg_file = config_path(opt.ckpt, opt.config)
    if not cfg_file.exists():
        raise SystemExit(f'config not found: {cfg_file} (pass --config)')
    cfg = load_config(str(cfg_file))
    model = load_model(cfg, opt.ckpt)
    raw = [np.asarray(load_point_cloud(f), dtype=np.float64) for f in opt.fragments]
    frags = [crop(cfg, x) for x in raw]
    if colors is not None:
        colors = [crop_colors(cfg, x, c) for x, c in zip(raw, colors)]
    T = register_pairs(model, frags, opt.batch_pairs, opt.icp, opt.icp_iters, opt.icp_method, opt.normal_radius,
                       opt.normal_max_nn, opt.icp_epsilon, opt.icp_loss, opt.icp_loss_k, opt.ransac,
                       ransac_kwargs(opt) if opt.ransac is not None else None,
                       dict(fgr_kwargs(opt), overlap=opt.fgr_overlap) if opt.fgr else None, colors,
                       opt.icp_lambda_geometric)
    D = float(cfg['overlap_radius'] if opt.info_radius is None else opt.info_radius)
    res = optimize_scene(frags, T, D, opt.min_overlap, opt.preference_loop_closure)
    write_outputs(res, opt.out, scene_name(opt.fragments[0]), frags, opt.voxel)
    r = res['result']
    line = {'n_fragments': len(frags), 'pairs': int(len(res['pairs'])), 'edges_odometry': res['n_odometry'],
            'edges_loop': res['n_loop'], 'edges_kept': int(r[3]), 'iterations_pass1': int(r[0]),
            'iterations_pass2': int(r[1]), 'objective': float(r[2]), 'info_radius': D}
    print(json.dumps(line))
    return res


if __name__ == '__main__':
    main()
