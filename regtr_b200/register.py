"""Register two point-cloud files with a trained RegTR: the reference's `src/demo.py` on the library path.

    python -m regtr_b200.register SRC TGT --ckpt <logdir>/ckpt/model-best.pth [--config <yaml>] \\
        [--threshold 0.5] [--fit_radius R] [--out DIR]

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
One JSON line on stdout: the pose, the four fit numbers and the point counts.
"""
from __future__ import annotations

import argparse
import json
import os
from pathlib import Path
from typing import Dict

import numpy as np
import torch


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog='python -m regtr_b200.register',
                                 description='Register a source point cloud to a target with a trained RegTR.')
    ap.add_argument('src', help='Source point cloud (.ply, .pth, .bin or .npy)')
    ap.add_argument('tgt', help='Target point cloud (.ply, .pth, .bin or .npy)')
    ap.add_argument('--ckpt', required=True, help='Checkpoint ({"state_dict": ...}), e.g. <logdir>/ckpt/model-best.pth')
    ap.add_argument('--config', help='Config file (default: config.yaml one level above the checkpoint directory)')
    ap.add_argument('--threshold', type=float, default=0.5,
                    help='Keypoints with predicted overlap above this go to src_kp.ply / src_kp_warped.ply')
    ap.add_argument('--fit_radius', type=float, help='Inlier radius of the fitness / RMSE (default: overlap_radius)')
    ap.add_argument('--out', default='.', help='Output directory')
    return ap


def config_path(ckpt: str, config: str = None) -> Path:
    """--config, else demo.py's rule: Path(ckpt).parents[1] / 'config.yaml'."""
    return Path(config) if config is not None else Path(ckpt).parents[1] / 'config.yaml'


def crop(cfg, xyz: np.ndarray) -> np.ndarray:
    """demo.py: with `crop_radius` in the config, keep the points with ||x|| < crop_radius."""
    if 'crop_radius' in cfg:
        return xyz[np.linalg.norm(xyz, axis=1) < cfg['crop_radius'], :]
    return xyz


def load_model(cfg, ckpt: str, device=None):
    """RegTR(cfg) on the device in eval mode with the checkpoint's state_dict loaded strictly (as the demo does)."""
    from .regtr import RegTR
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else device
    model = RegTR(cfg).to(device).eval()
    state = torch.load(ckpt, map_location='cpu', weights_only=True)
    model.load_state_dict(state['state_dict'])
    return model


def register(model, cfg, src_xyz: np.ndarray, tgt_xyz: np.ndarray, fit_radius: float = None) -> Dict:
    """Crop, forward and fit one pair.  src_xyz / tgt_xyz (N,3) float64 host arrays.
    -> dict of host arrays: src_xyz / tgt_xyz (cropped, float64), pose (L,3,4) fp32, src_kp, src_kp_warped (final
    layer), src_overlap (sigmoid of the final layer's logit, (n,)), the same for tgt, fit (4,) float64."""
    from . import ops
    src_xyz = crop(cfg, np.asarray(src_xyz, dtype=np.float64))
    tgt_xyz = crop(cfg, np.asarray(tgt_xyz, dtype=np.float64))
    dev = model.device
    batch = {'src_xyz': [torch.from_numpy(src_xyz).float().to(dev)],
             'tgt_xyz': [torch.from_numpy(tgt_xyz).float().to(dev)]}
    with torch.no_grad():
        out = model(batch)
        pose = out['pose'][:, 0]                                             # (L,3,4), pair 0
        radius = float(cfg['overlap_radius'] if fit_radius is None else fit_radius)
        status = ops.new_status(dev)
        fit = ops.registration_fit([src_xyz], [tgt_xyz], pose[-1:], radius, status)
        res = {'src_xyz': src_xyz, 'tgt_xyz': tgt_xyz, 'pose': pose.cpu().numpy()}
        for side in ('src', 'tgt'):
            res[f'{side}_kp'] = out[f'{side}_kp'][0].cpu().numpy()
            res[f'{side}_kp_warped'] = out[f'{side}_kp_warped'][0][-1].cpu().numpy()
            res[f'{side}_overlap'] = torch.sigmoid(out[f'{side}_overlap'][0][-1][:, 0]).cpu().numpy()
        ops.check_fit_status(status, radius)
        res['fit'] = fit[0].cpu().numpy()
    return res


def pose44(pose34) -> np.ndarray:
    p = np.eye(4)
    p[:3] = np.asarray(pose34, dtype=np.float64)
    return p


def pose_text(pose34) -> str:
    """est.log's pose rows (eval.EstLogWriter): four lines of tab-separated 12-decimal numbers."""
    return ''.join('\t'.join(map('{0:.12f}'.format, row)) + '\n' for row in pose44(pose34))


def write_outputs(res: Dict, out_dir: str, threshold: float = 0.5):
    from .pointio import write_ply
    os.makedirs(out_dir, exist_ok=True)
    final = res['pose'][-1]
    with open(os.path.join(out_dir, 'pose.txt'), 'w') as fh:
        fh.write(pose_text(final))
    np.savez(os.path.join(out_dir, 'result.npz'), **{k: res[k] for k in (
        'pose', 'src_kp', 'src_kp_warped', 'src_overlap', 'tgt_kp', 'tgt_kp_warped', 'tgt_overlap', 'fit')})
    p = final.astype(np.float64)
    write_ply(os.path.join(out_dir, 'src_registered.ply'), res['src_xyz'] @ p[:, :3].T + p[:, 3])
    m = res['src_overlap'] > threshold
    write_ply(os.path.join(out_dir, 'src_kp.ply'), res['src_kp'][m], {'overlap': res['src_overlap'][m]})
    write_ply(os.path.join(out_dir, 'src_kp_warped.ply'), res['src_kp_warped'][m], {'overlap': res['src_overlap'][m]})
    return int(m.sum())


def main(argv=None):
    opt = parser().parse_args(argv)
    from .config import load_config
    from .pointio import load_point_cloud
    cfg_file = config_path(opt.ckpt, opt.config)
    if not cfg_file.exists():
        raise SystemExit(f'config not found: {cfg_file} (pass --config)')
    cfg = load_config(str(cfg_file))
    model = load_model(cfg, opt.ckpt)
    res = register(model, cfg, load_point_cloud(opt.src), load_point_cloud(opt.tgt), opt.fit_radius)
    n_shown = write_outputs(res, opt.out, opt.threshold)
    f = [float(v) for v in res['fit']]
    print(json.dumps({'pose': pose44(res['pose'][-1]).tolist(), 'fitness_src': f[0], 'rmse_src': f[1],
                      'fitness_tgt': f[2], 'rmse_tgt': f[3], 'n_src': int(res['src_xyz'].shape[0]),
                      'n_tgt': int(res['tgt_xyz'].shape[0]), 'n_src_kp': int(res['src_kp'].shape[0]),
                      'n_tgt_kp': int(res['tgt_kp'].shape[0]), 'n_src_kp_above_threshold': n_shown,
                      'fit_radius': float(cfg['overlap_radius'] if opt.fit_radius is None else opt.fit_radius)}))
    return res


if __name__ == '__main__':
    main()
