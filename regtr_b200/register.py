"""Register two point-cloud files with a trained RegTR: the reference's `src/demo.py` on the library path.

    python -m regtr_b200.register SRC TGT --ckpt <logdir>/ckpt/model-best.pth [--config <yaml>] \\
        [--threshold 0.5] [--fit_radius R] [--out DIR]
        [--icp R [--icp_iters 30] [--icp_method point_to_point|point_to_plane|generalized|colored
         [--normal_radius NR] [--normal_max_nn 30] [--icp_epsilon 1e-3] [--icp_lambda_geometric 0.968]
         [--icp_loss l2|huber|cauchy|gm|tukey --icp_loss_k K]
         [--icp_voxels V1,V2,... [--icp_radii R1,...] [--icp_level_iters I1,...]]]]
        [--ransac R [--ransac_iters 100000] [--ransac_confidence 0.999] [--ransac_n 3] [--ransac_edge 0.9]
         [--ransac_dist D] [--ransac_overlap 0.5] [--ransac_seed 0]]
        [--fgr [--fgr_dist 0.025] [--fgr_iters 64] [--fgr_division 1.4] [--fgr_tuple_test [--fgr_tuple_scale 0.95]
         [--fgr_max_tuples 1000]] [--fgr_no_decrease_mu] [--fgr_absolute_scale] [--fgr_overlap 0.5] [--fgr_seed 0]]
    python -m regtr_b200.register SRC TGT --fpfh V [--fpfh_radius FR] [--fpfh_max_nn 100] [--fpfh_no_mutual]
        [--ransac R ... | --fgr [--fgr_dist D] [--fgr_no_tuple_test] ...] [--icp R ...] [--fit_radius R] [--out DIR]
    either form also takes [--remove_statistical_outlier K S] [--remove_radius_outlier N R]

SRC / TGT: .ply, .pth, .bin or .npy (regtr_b200.pointio).  The config is the config.yaml one level above the
checkpoint's directory, the layout `python -m regtr_b200.train` writes, unless --config names another.  Instead of the
demo's viewer, the result is judged by the fitness and inlier RMSE of the final pose on the full-resolution clouds
(Open3D's evaluate_registration definitions, computed on the device by `ops.registration_fit`), and written to --out:
  pose.txt             the final 4x4 pose in est.log's 12-decimal format;
  result.npz           pose (L,3,4) of every decoder layer, src_kp, src_kp_warped, src_overlap (sigmoid, final layer),
                       the same three for the target, fit (4,) = fitness_src, rmse_src, fitness_tgt, rmse_tgt;
  src_registered.ply   the source moved by the pose;
  src_kp.ply, src_kp_warped.ply   the source keypoints with predicted overlap > --threshold and their predicted
                       positions in the target, with an `overlap` property (the demo's two upper panels).
With --icp R the final decoder layer's pose is refined by ICP on the cropped full-resolution clouds (`ops.icp`,
Open3D's registration_icp with max_correspondence_distance R and --icp_iters iterations at most), point-to-point by
default; --icp_method point_to_plane first estimates the cropped target's normals (`ops.estimate_normals`, Open3D's
estimate_normals with KDTreeSearchParamHybrid(--normal_radius, default 2 R, --normal_max_nn)); --icp_method
generalized estimates the normals of both cropped clouds in one call and runs Open3D's registration_generalized_icp
(covariance epsilon --icp_epsilon); --icp_method colored reads both files' colours (PLY red / green / blue, a file
without them is a usage error), estimates the cropped target's normals as point_to_plane does and its intensity
gradients (`ops.color_gradients`, radius 2 R, 30 neighbours at most, Open3D's parameters), and runs Open3D's
registration_colored_icp (geometric weight --icp_lambda_geometric); --icp_loss with --icp_loss_k weights the
point-to-plane, generalized or colored residuals by Open3D's robust kernel of that name;
pose.txt, src_registered.ply and fit then use the refined pose, result.npz gains pose_coarse (the network's final
pose), pose_icp (the refined one) and icp (4,) = fitness, inlier_rmse, correspondences, iterations.  --icp_voxels
V1,V2,... runs multi-scale ICP (Open3D's colored-ICP tutorial): level l down-samples both clouds at V_l
(`ops.voxel_down_sample`, a grid anchored at each cloud's bounding box; a last 0 keeps the full clouds), estimates its
normals at 2 R_l and runs ICP at R_l (--icp_radii, default V_l, or R at a 0 voxel) for at most I_l iterations
(--icp_level_iters, default --icp_iters) from the previous level's pose; icp is then the last level's, and result.npz
and the JSON line gain icp_levels (L,4), the JSON line also icp_voxels, icp_radii and icp_level_iters.
With --ransac R the final decoder layer's pose is replaced by RANSAC over the network's two-way correspondences with
predicted overlap above --ransac_overlap (`ops.ransac`, Open3D's registration_ransac_based_on_correspondence with max
correspondence distance R on the cropped full-resolution clouds, --ransac_iters hypotheses at most, confidence
--ransac_confidence, --ransac_n correspondences per sample, the edge-length checker at --ransac_edge and the distance
checker at --ransac_dist); with --icp as well, ICP starts from the RANSAC pose (Open3D's global-then-local pipeline).
result.npz then gains pose_coarse, pose_ransac (3,4) float64 and ransac (5,) = fitness, inlier_rmse, hypotheses
walked, hypotheses validated, winning hypothesis.
With --fgr (instead of --ransac) the final decoder layer's pose is replaced by Fast Global Registration over the same
correspondences with predicted overlap above --fgr_overlap (`ops.fgr`, Open3D's registration_fgr_based_on_correspondence
with FastGlobalRegistrationOption: --fgr_dist the maximum correspondence distance, --fgr_iters iterations, --fgr_division,
--fgr_no_decrease_mu, --fgr_absolute_scale, and the tuple test only with --fgr_tuple_test); with --icp as well, ICP
starts from the FGR pose.  result.npz then gains pose_coarse, pose_fgr (3,4) float64 and fgr (4,) = correspondences of
the solve, tuples kept, trials walked, final GNC parameter.
One JSON line on stdout: the pose, the four fit numbers and the point counts (with --icp, also icp_fitness, icp_rmse,
icp_iterations, icp_radius and icp_method, and icp_loss, icp_loss_k, icp_epsilon and icp_lambda_geometric when they
are given; with --ransac,
ransac_fitness, ransac_rmse, ransac_iterations, ransac_validations and ransac_radius; with --fgr, fgr_correspondences,
fgr_tuples, fgr_trials, fgr_par and fgr_dist).
With --fpfh V there is no network and no --ckpt: Open3D's classical global registration (`eval.fpfh_register`) on the
device.  Both clouds are downsampled at voxel V (`ops.grid_subsample`, a grid anchored at the origin), their normals
estimated at 2 V with 30 neighbours at most, their FPFH features computed at --fpfh_radius (default 5 V) with
--fpfh_max_nn neighbours at most, and `ops.ransac_feature_matching` registers the downsampled clouds: mutual feature
matches (every match with --fpfh_no_mutual, or when fewer than 3 --ransac_n are mutual), --ransac radius (default
1.5 V), the distance checker at --ransac_dist (default: the --ransac radius); --ransac_overlap is ignored.  --icp then
refines the pose on the full clouds as above, and fit is taken at --fit_radius (default: the --ransac radius).
Written: pose.txt, src_registered.ply and result.npz with pose_fpfh (3,4) float64, ransac (5,), n_mutual, fit and,
with --icp, pose_icp and icp; no keypoint files.  The JSON line has the pose, the fit numbers, the point counts,
fpfh_voxel, n_src_down, n_tgt_down, n_mutual and the ransac_* (and icp_*) entries.
With --remove_statistical_outlier K S and / or --remove_radius_outlier N R, both clouds are first filtered as read
from the files, before the config's crop (`eval.remove_outliers`: Open3D's remove_statistical_outlier(K, S), then
remove_radius_outlier(N, R) on what is left, with the colours read for colored ICP filtered alike), which equals
reading the files in Open3D, filtering, saving and registering the saved clouds.  result.npz then gains src_index and
tgt_index (the surviving rows of each file) and the JSON line n_src_read, n_tgt_read, n_src_filtered and
n_tgt_filtered, on both paths.
With --fpfh V --fgr the mutual FPFH matches go to FGR instead (`ops.fgr_feature_matching`, the tuple test on unless
--fgr_no_tuple_test, --fgr_dist defaulting to 0.5 V as in Open3D's tutorial); --fpfh_no_mutual is then a usage error,
and fit is taken at --fit_radius (default 1.5 V).  result.npz holds pose_fpfh (the FGR pose) and fgr (4,) in place of
ransac, and the JSON line has the fgr_* entries in place of the ransac_* ones.
"""
from __future__ import annotations

import argparse
import json
import os
from pathlib import Path
from typing import Dict

import numpy as np
import torch

from .eval import (add_fgr_arguments, add_fpfh_arguments, add_icp_arguments, add_outlier_arguments,
                   add_ransac_arguments, check_fgr_arguments, check_fpfh_arguments, check_icp_arguments,
                   check_outlier_arguments, check_ransac_arguments, fgr_kwargs, fgr_refine, fpfh_kwargs, fpfh_register,
                   icp_kwargs, icp_levels, icp_refine, ransac_kwargs, ransac_refine, remove_outliers)


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog='python -m regtr_b200.register',
                                 description='Register a source point cloud to a target with a trained RegTR.')
    ap.add_argument('src', help='Source point cloud (.ply, .pth, .bin or .npy)')
    ap.add_argument('tgt', help='Target point cloud (.ply, .pth, .bin or .npy)')
    ap.add_argument('--ckpt', help='Checkpoint ({"state_dict": ...}), e.g. <logdir>/ckpt/model-best.pth (required '
                                   'unless --fpfh)')
    ap.add_argument('--config', help='Config file (default: config.yaml one level above the checkpoint directory)')
    ap.add_argument('--threshold', type=float, default=0.5,
                    help='Keypoints with predicted overlap above this go to src_kp.ply / src_kp_warped.ply')
    ap.add_argument('--fit_radius', type=float,
                    help='Inlier radius of the fitness / RMSE (default: overlap_radius; with --fpfh the RANSAC radius)')
    add_icp_arguments(ap, 'Refine the pose with point-to-point ICP, max correspondence distance R (default: no ICP)')
    add_ransac_arguments(ap, 'Replace the pose by RANSAC over the predicted correspondences, max correspondence '
                             'distance R (default: no RANSAC; before ICP with --icp; with --fpfh 1.5 V)')
    add_fgr_arguments(ap, 'Replace the pose by Fast Global Registration over the predicted correspondences (with '
                          '--fpfh: over the FPFH matches) instead of RANSAC; before ICP with --icp')
    add_fpfh_arguments(ap)
    add_outlier_arguments(ap)
    ap.add_argument('--out', default='.', help='Output directory')
    return ap


def parse_args(argv=None):
    """The parsed command line, its usage errors raised and the --fpfh defaults filled in."""
    ap = parser()
    opt = ap.parse_args(argv)
    check_fgr_arguments(ap, opt)
    check_fpfh_arguments(ap, opt)
    check_icp_arguments(ap, opt, colors=True)
    check_ransac_arguments(ap, opt)
    check_outlier_arguments(ap, opt)
    if opt.fpfh is not None and opt.fit_radius is None:
        opt.fit_radius = 1.5 * opt.fpfh if opt.fgr else opt.ransac
    return opt


def config_path(ckpt: str, config: str = None) -> Path:
    """--config, else demo.py's rule: Path(ckpt).parents[1] / 'config.yaml'."""
    return Path(config) if config is not None else Path(ckpt).parents[1] / 'config.yaml'


def crop(cfg, xyz: np.ndarray) -> np.ndarray:
    """demo.py: with `crop_radius` in the config, keep the points with ||x|| < crop_radius."""
    if 'crop_radius' in cfg:
        return xyz[np.linalg.norm(xyz, axis=1) < cfg['crop_radius'], :]
    return xyz


def crop_colors(cfg, xyz: np.ndarray, rgb: np.ndarray) -> np.ndarray:
    """The rows of rgb (N,3) that `crop(cfg, xyz)` keeps of xyz (N,3) float64."""
    if 'crop_radius' in cfg:
        return rgb[np.linalg.norm(xyz, axis=1) < cfg['crop_radius'], :]
    return rgb


def load_model(cfg, ckpt: str, device=None):
    """RegTR(cfg) on the device in eval mode with the checkpoint's state_dict loaded strictly (as the demo does)."""
    from .regtr import RegTR
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else device
    model = RegTR(cfg).to(device).eval()
    state = torch.load(ckpt, map_location='cpu', weights_only=True)
    model.load_state_dict(state['state_dict'])
    return model


def register(model, cfg, src_xyz: np.ndarray, tgt_xyz: np.ndarray, fit_radius: float = None,
             icp_radius: float = None, icp_iters: int = 30, icp_method: str = 'point_to_point',
             normal_radius: float = None, normal_max_nn: int = 30, icp_epsilon: float = 1e-3, icp_loss: str = 'l2',
             icp_loss_k: float = None, ransac_radius: float = None, ransac_options: Dict = None,
             fgr_options: Dict = None, colors=None, icp_lambda_geometric: float = 0.968, icp_voxels=None,
             icp_radii=None, icp_level_iters=None) -> Dict:
    """Crop, forward and fit one pair.  src_xyz / tgt_xyz (N,3) float64 host arrays; colors (src_rgb, tgt_rgb) (N,3)
    host arrays aligned with them, cropped alike, for icp_method='colored' (with icp_lambda_geometric).
    -> dict of host arrays: src_xyz / tgt_xyz (cropped, float64), pose (L,3,4) fp32, src_kp, src_kp_warped (final
    layer), src_overlap (sigmoid of the final layer's logit, (n,)), the same for tgt, fit (4,) float64.
    icp_radius: refine the final layer's pose by ICP on the cropped clouds (`eval.icp_refine` with icp_method, at most
    icp_iters iterations, and normal_radius, normal_max_nn, icp_epsilon, icp_loss and icp_loss_k); fit is then that of
    the refined pose, and the dict gains pose_coarse (3,4) fp32 (the network's final pose), pose_icp (3,4) float64 and
    icp (4,) float64 = fitness, inlier_rmse, correspondences, iterations.  icp_voxels (with icp_radii and
    icp_level_iters): multi-scale ICP (`eval.icp_refine`'s voxels, radii and level_iters); icp is then the last
    level's, and the dict gains icp_levels (L,4) float64, the four numbers of every level.
    ransac_radius: first replace the final layer's pose by `eval.ransac_refine` at that radius on the cropped clouds,
    with ransac_options its further keyword arguments (ICP then starts from it); the dict gains pose_coarse,
    pose_ransac (3,4) float64 and ransac (5,) float64 = fitness, inlier_rmse, walked, validated, winner.
    fgr_options: likewise, but `eval.fgr_refine` with these keyword arguments (overlap and `ops.fgr`'s options); the
    dict gains pose_coarse, pose_fgr (3,4) float64 and fgr (4,) float64 = correspondences, tuples, trials, par."""
    from . import ops
    src_xyz, tgt_xyz = np.asarray(src_xyz, dtype=np.float64), np.asarray(tgt_xyz, dtype=np.float64)
    if colors is not None:
        colors = [crop_colors(cfg, src_xyz, colors[0])], [crop_colors(cfg, tgt_xyz, colors[1])]
    src_xyz, tgt_xyz = crop(cfg, src_xyz), crop(cfg, tgt_xyz)
    dev = model.device
    batch = {'src_xyz': [torch.from_numpy(src_xyz).float().to(dev)],
             'tgt_xyz': [torch.from_numpy(tgt_xyz).float().to(dev)]}
    with torch.no_grad():
        out = model(batch)
        pose = out['pose'][:, 0]                                             # (L,3,4), pair 0
        radius = float(cfg['overlap_radius'] if fit_radius is None else fit_radius)
        status = ops.new_status(dev)
        final = pose[-1:]
        if ransac_radius is not None:
            final, ransac = ransac_refine(out, [src_xyz], [tgt_xyz], ransac_radius, **(ransac_options or {}))
            pose_ransac = final
        if fgr_options is not None:
            final, fgr = fgr_refine(out, [src_xyz], [tgt_xyz], **fgr_options)
            pose_fgr = final
        if icp_radius is not None:
            pyramid = {} if icp_voxels is None else dict(voxels=icp_voxels, radii=icp_radii,
                                                          level_iters=icp_level_iters, return_levels=True)
            final, icp, *levels = icp_refine([src_xyz], [tgt_xyz], final, icp_radius, icp_iters, icp_method,
                                             normal_radius, normal_max_nn, icp_epsilon, icp_loss, icp_loss_k,
                                             colors=colors, lambda_geometric=icp_lambda_geometric, **pyramid)
        fit = ops.registration_fit([src_xyz], [tgt_xyz], final, radius, status)
        res = {'src_xyz': src_xyz, 'tgt_xyz': tgt_xyz, 'pose': pose.cpu().numpy()}
        if icp_radius is not None:
            res.update(pose_coarse=res['pose'][-1], pose_icp=final[0].cpu().numpy(), icp=icp[0].cpu().numpy())
            if levels:
                res['icp_levels'] = levels[0][0].cpu().numpy()
        if ransac_radius is not None:
            res.update(pose_coarse=res['pose'][-1], pose_ransac=pose_ransac[0].cpu().numpy(),
                       ransac=ransac[0].cpu().numpy())
        if fgr_options is not None:
            res.update(pose_coarse=res['pose'][-1], pose_fgr=pose_fgr[0].cpu().numpy(), fgr=fgr[0].cpu().numpy())
        for side in ('src', 'tgt'):
            res[f'{side}_kp'] = out[f'{side}_kp'][0].cpu().numpy()
            res[f'{side}_kp_warped'] = out[f'{side}_kp_warped'][0][-1].cpu().numpy()
            res[f'{side}_overlap'] = torch.sigmoid(out[f'{side}_overlap'][0][-1][:, 0]).cpu().numpy()
        ops.check_fit_status(status, radius)
        res['fit'] = fit[0].cpu().numpy()
    return res


def register_fpfh(src_xyz: np.ndarray, tgt_xyz: np.ndarray, voxel: float, fit_radius: float,
                  icp_radius: float = None, icp_options: Dict = None, fpfh_options: Dict = None) -> Dict:
    """One pair without a network (`eval.fpfh_register` at voxel, fpfh_options its further keyword arguments, then ICP
    on the full clouds with icp_radius and icp_options).  -> dict of host arrays: src_xyz / tgt_xyz (float64),
    pose_fpfh (3,4) float64, ransac (5,) (fgr (4,) with method='fgr' in fpfh_options), n_mutual, n_src_down,
    n_tgt_down, fit (4,) of the final pose at fit_radius, and pose_icp / icp with icp_radius (and icp_levels with
    voxels in icp_options)."""
    from . import ops
    src_xyz = np.asarray(src_xyz, dtype=np.float64)
    tgt_xyz = np.asarray(tgt_xyz, dtype=np.float64)
    out = fpfh_register([src_xyz], [tgt_xyz], voxel, icp_radius=icp_radius, icp_kwargs=icp_options,
                        **(fpfh_options or {}))
    fit = ops.registration_fit([src_xyz], [tgt_xyz], out['pose'], fit_radius)
    glob = 'fgr' if 'fgr' in out else 'ransac'
    res = {'src_xyz': src_xyz, 'tgt_xyz': tgt_xyz, 'pose_fpfh': out['pose_fpfh'][0].cpu().numpy(),
           glob: out[glob][0].cpu().numpy(), 'n_mutual': int(out['n_mutual'][0]),
           'n_src_down': int(out['src_down'][0].shape[0]), 'n_tgt_down': int(out['tgt_down'][0].shape[0]),
           'fit': fit[0].cpu().numpy()}
    if icp_radius is not None:
        res.update(pose_icp=out['pose'][0].cpu().numpy(), icp=out['icp'][0].cpu().numpy())
    if 'icp_levels' in out:
        res['icp_levels'] = out['icp_levels'][0].cpu().numpy()
    return res


def pose44(pose34) -> np.ndarray:
    p = np.eye(4)
    p[:3] = np.asarray(pose34, dtype=np.float64)
    return p


def pose_text(pose34) -> str:
    """est.log's pose rows (eval.EstLogWriter): four lines of tab-separated 12-decimal numbers."""
    return ''.join('\t'.join(map('{0:.12f}'.format, row)) + '\n' for row in pose44(pose34))


def final_pose(res: Dict):
    """The pose `register` settles on: ICP's, else RANSAC's or FGR's (over network or FPFH matches), else the final
    decoder layer's."""
    for k in ('pose_icp', 'pose_ransac', 'pose_fgr', 'pose_fpfh'):
        if k in res:
            return res[k]
    return res['pose'][-1]


def write_outputs(res: Dict, out_dir: str, threshold: float = 0.5):
    from .pointio import write_ply
    os.makedirs(out_dir, exist_ok=True)
    final = final_pose(res)
    with open(os.path.join(out_dir, 'pose.txt'), 'w') as fh:
        fh.write(pose_text(final))
    p = final.astype(np.float64)
    write_ply(os.path.join(out_dir, 'src_registered.ply'), res['src_xyz'] @ p[:, :3].T + p[:, 3])
    if 'pose_fpfh' in res:
        keys = ('pose_fpfh', 'fgr' if 'fgr' in res else 'ransac', 'n_mutual', 'fit') + \
            (('pose_icp', 'icp') if 'pose_icp' in res else ()) + (('icp_levels',) if 'icp_levels' in res else ()) + \
            (('src_index', 'tgt_index') if 'src_index' in res else ())
        np.savez(os.path.join(out_dir, 'result.npz'), **{k: res[k] for k in keys})
        return 0
    keys = ('pose', 'src_kp', 'src_kp_warped', 'src_overlap', 'tgt_kp', 'tgt_kp_warped', 'tgt_overlap', 'fit')
    if 'pose_coarse' in res:
        keys += ('pose_coarse',)
    if 'pose_ransac' in res:
        keys += ('pose_ransac', 'ransac')
    if 'pose_fgr' in res:
        keys += ('pose_fgr', 'fgr')
    if 'pose_icp' in res:
        keys += ('pose_icp', 'icp')
    if 'icp_levels' in res:
        keys += ('icp_levels',)
    if 'src_index' in res:
        keys += ('src_index', 'tgt_index')
    np.savez(os.path.join(out_dir, 'result.npz'), **{k: res[k] for k in keys})
    m = res['src_overlap'] > threshold
    write_ply(os.path.join(out_dir, 'src_kp.ply'), res['src_kp'][m], {'overlap': res['src_overlap'][m]})
    write_ply(os.path.join(out_dir, 'src_kp_warped.ply'), res['src_kp_warped'][m], {'overlap': res['src_overlap'][m]})
    return int(m.sum())


def main(argv=None):
    opt = parse_args(argv)
    from .eval import load_icp_colors
    from .pointio import load_point_cloud
    colors = load_icp_colors(parser(), opt, [opt.src, opt.tgt])
    if opt.fpfh is not None:
        return main_fpfh(opt, *read_clouds(opt, load_point_cloud(opt.src), load_point_cloud(opt.tgt), colors))
    from .config import load_config
    cfg_file = config_path(opt.ckpt, opt.config)
    if not cfg_file.exists():
        raise SystemExit(f'config not found: {cfg_file} (pass --config)')
    cfg = load_config(str(cfg_file))
    model = load_model(cfg, opt.ckpt)
    src_xyz, tgt_xyz, colors, filtered = read_clouds(opt, load_point_cloud(opt.src), load_point_cloud(opt.tgt), colors)
    res = register(model, cfg, src_xyz, tgt_xyz, opt.fit_radius, opt.icp,
                   opt.icp_iters, opt.icp_method, opt.normal_radius, opt.normal_max_nn, opt.icp_epsilon,
                   opt.icp_loss, opt.icp_loss_k, opt.ransac, ransac_kwargs(opt) if opt.ransac is not None else None,
                   dict(fgr_kwargs(opt), overlap=opt.fgr_overlap) if opt.fgr else None, colors,
                   opt.icp_lambda_geometric, opt.icp_voxels, opt.icp_radii, opt.icp_level_iters)
    n_outlier = outlier_line(res, filtered)
    n_shown = write_outputs(res, opt.out, opt.threshold)
    f = [float(v) for v in res['fit']]
    line = {'pose': pose44(final_pose(res)).tolist(),
            'fitness_src': f[0], 'rmse_src': f[1],
            'fitness_tgt': f[2], 'rmse_tgt': f[3], 'n_src': int(res['src_xyz'].shape[0]),
            'n_tgt': int(res['tgt_xyz'].shape[0]), 'n_src_kp': int(res['src_kp'].shape[0]),
            'n_tgt_kp': int(res['tgt_kp'].shape[0]), 'n_src_kp_above_threshold': n_shown,
            'fit_radius': float(cfg['overlap_radius'] if opt.fit_radius is None else opt.fit_radius)}
    if opt.icp is not None:
        line.update(icp_line(opt, res))
    if opt.ransac is not None:
        rs = [float(v) for v in res['ransac']]
        line.update(ransac_fitness=rs[0], ransac_rmse=rs[1], ransac_iterations=int(rs[2]),
                    ransac_validations=int(rs[3]), ransac_radius=float(opt.ransac))
    if opt.fgr:
        line.update(fgr_line(opt, res['fgr']))
    line.update(n_outlier)
    print(json.dumps(line))
    return res


def read_clouds(opt, src_xyz, tgt_xyz, colors):
    """The clouds as read, filtered by the outlier flags when given (`eval.remove_outliers`, colours alike).
    -> (src_xyz, tgt_xyz, colors, filtered): filtered None without the flags, else ((n_src_read, n_tgt_read),
    [src_index, tgt_index])."""
    if opt.remove_statistical_outlier is None and opt.remove_radius_outlier is None:
        return src_xyz, tgt_xyz, colors, None
    read = (int(src_xyz.shape[0]), int(tgt_xyz.shape[0]))
    (src_xyz, tgt_xyz), colors, index = remove_outliers([src_xyz, tgt_xyz], colors, opt.remove_statistical_outlier,
                                                        opt.remove_radius_outlier)
    return src_xyz, tgt_xyz, colors, (read, index)


def outlier_line(res: Dict, filtered) -> Dict:
    """With the outlier flags (filtered = ((n_src_read, n_tgt_read), [src_index, tgt_index])): the surviving rows of
    each file into `register`'s dict as src_index / tgt_index, and -> the JSON line's point counts before and after
    the filters; else {}."""
    if filtered is None:
        return {}
    read, index = filtered
    res['src_index'], res['tgt_index'] = index
    return {'n_src_read': read[0], 'n_tgt_read': read[1], 'n_src_filtered': int(index[0].shape[0]),
            'n_tgt_filtered': int(index[1].shape[0])}


def fgr_line(opt, fgr) -> Dict:
    """The JSON line's fgr_* entries."""
    fgr = [float(v) for v in fgr]
    return dict(fgr_correspondences=int(fgr[0]), fgr_tuples=int(fgr[1]), fgr_trials=int(fgr[2]), fgr_par=fgr[3],
                fgr_dist=float(opt.fgr_dist))


def icp_line(opt, res: Dict) -> Dict:
    """The JSON line's icp_* entries from `register`'s dict (those of the last level with --icp_voxels, which adds
    icp_voxels, icp_radii and icp_level_iters as resolved and icp_levels, the four numbers of every level)."""
    icp = [float(v) for v in res['icp']]
    line = dict(icp_fitness=icp[0], icp_rmse=icp[1], icp_iterations=int(icp[3]), icp_radius=float(opt.icp),
                icp_method=opt.icp_method)
    if opt.icp_loss != 'l2':
        line.update(icp_loss=opt.icp_loss, icp_loss_k=float(opt.icp_loss_k))
    if opt.icp_method == 'generalized':
        line.update(icp_epsilon=float(opt.icp_epsilon))
    if opt.icp_method == 'colored':
        line.update(icp_lambda_geometric=float(opt.icp_lambda_geometric))
    if opt.icp_voxels is not None:
        plan = icp_levels(opt.icp_voxels, opt.icp_radii, opt.icp_level_iters, opt.icp, opt.icp_iters)
        line.update(icp_voxels=[v for v, _, _ in plan], icp_radii=[r for _, r, _ in plan],
                    icp_level_iters=[i for _, _, i in plan], icp_levels=res['icp_levels'].tolist())
    return line


def main_fpfh(opt, src_xyz, tgt_xyz, colors=None, filtered=None):
    """`main` with --fpfh: `register_fpfh`, its files and its JSON line (colors: the files' rgb for colored ICP;
    filtered: what the outlier filters kept, as `outlier_line` takes it)."""
    icp_options = None
    if opt.icp is not None:
        icp_options = dict(icp_kwargs(opt), **({} if colors is None else {'colors': ([colors[0]], [colors[1]])}))
    res = register_fpfh(src_xyz, tgt_xyz, opt.fpfh, opt.fit_radius, opt.icp, icp_options, fpfh_kwargs(opt))
    n_outlier = outlier_line(res, filtered)
    write_outputs(res, opt.out)
    f = [float(v) for v in res['fit']]
    line = {'pose': pose44(final_pose(res)).tolist(), 'fitness_src': f[0], 'rmse_src': f[1], 'fitness_tgt': f[2],
            'rmse_tgt': f[3], 'n_src': int(res['src_xyz'].shape[0]), 'n_tgt': int(res['tgt_xyz'].shape[0]),
            'fit_radius': float(opt.fit_radius), 'fpfh_voxel': float(opt.fpfh), 'n_src_down': res['n_src_down'],
            'n_tgt_down': res['n_tgt_down'], 'n_mutual': res['n_mutual']}
    if opt.fgr:
        line.update(fgr_line(opt, res['fgr']))
    else:
        rs = [float(v) for v in res['ransac']]
        line.update(ransac_fitness=rs[0], ransac_rmse=rs[1], ransac_iterations=int(rs[2]),
                    ransac_validations=int(rs[3]), ransac_radius=float(opt.ransac))
    if opt.icp is not None:
        line.update(icp_line(opt, res))
    line.update(n_outlier)
    print(json.dumps(line))
    return res


if __name__ == '__main__':
    main()
