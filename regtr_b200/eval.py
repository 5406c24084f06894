"""Registration metrics around the forward pass (SURVEY.md 8f N1): the callers that turn poses into
the numbers the paper reports.

Host-side mirror of
  * `GenericRegModel._compute_metrics / _aggregate_metrics / _save_3DMatch_log`
    (/root/reference/src/models/generic_reg_model.py:175-229, 260-281),
  * the 3DMatch / 3DLoMatch registration-recall benchmark of Predator
    (/root/reference/src/benchmark/benchmark_predator.py:17-375),
  * the 3DMatch success rate of Deep Global Registration (benchmark/benchmark_3dmatch.py:benchmark_dgr),
  * the ModelNet metrics of RPMNet (/root/reference/src/benchmark/benchmark_modelnet.py:33-97).
Same file formats (Redwood `gt.log` / `gt.info` / `est.log`), same definitions, same summary strings,
so a run of this package can be scored with either implementation.  Pure numpy / torch: none of this is
on the GPU hot path.  Pinned against the reference's own functions by tests/golden/eval.npz.
"""
from __future__ import annotations

import argparse
import math
import os
from typing import Dict, Iterable, List

import numpy as np
import torch

# ------------------------------------------------------------------------------- SE(3) helpers


def _as44(pose):
    pose = np.asarray(pose, dtype=np.float64)
    if pose.shape[-2] == 3:
        pad = np.broadcast_to(np.array([0.0, 0.0, 0.0, 1.0]), pose.shape[:-2] + (1, 4))
        pose = np.concatenate([pose, pad], axis=-2)
    return pose


def se3_compare(a: torch.Tensor, b: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Residual rotation (degrees) and translation of a * b^-1 (utils/se3_torch.py:93-105); ([*,]3,4) inputs."""
    ra, ta = a[..., :3, :3], a[..., :3, 3:4]
    rb, tb = b[..., :3, :3], b[..., :3, 3:4]
    rbi = rb.transpose(-1, -2)
    rot = ra @ rbi
    trans = ta - rot @ tb
    trace = rot[..., 0, 0] + rot[..., 1, 1] + rot[..., 2, 2]
    rot_deg = torch.acos(torch.clamp(0.5 * (trace - 1), -1.0, 1.0)) * 180 / math.pi
    return {'rot_deg': rot_deg, 'trans': torch.norm(trans[..., 0], dim=-1)}


def compute_metrics(pred: Dict, gt_pose: torch.Tensor) -> Dict[str, torch.Tensor]:
    """generic_reg_model.py:175-187: rot/trans error of every `pose*` entry, (n_pred, B) each."""
    out = {}
    with torch.no_grad():
        for k in [k for k in pred if k.startswith('pose')]:
            err = se3_compare(pred[k], gt_pose[None, :])
            out[f'rot_err_deg{k[4:]}'] = err['rot_deg']
            out[f'trans_err{k[4:]}'] = err['trans']
    return out


def aggregate_metrics(metrics: List[Dict[str, torch.Tensor]], thresh_rot=10.0, thresh_trans=0.1):
    """generic_reg_model.py:189-229: means, histograms and registration success per decoder layer."""
    if len(metrics) == 0 or len(metrics[0]) == 0:
        return {}
    keys = set(metrics[0].keys())
    cat = {k: torch.cat([m[k] for m in metrics], dim=1) for k in keys}
    rot_keys = [k for k in cat if k.startswith('rot_err_deg')]
    num_pred = cat[rot_keys[0]].shape[0]
    avg = {}
    for p in range(num_pred):
        suffix = f'{p}' if p < num_pred - 1 else 'final'
        for rk in rot_keys:
            ps = rk[11:]
            tk = 'trans_err' + ps
            avg[f'rot_err_deg{ps}_{suffix}'] = torch.mean(cat[rk][p])
            avg[f'rot_err{ps}_{suffix}_hist'] = cat[rk][p]
            avg[f'{tk}_{suffix}'] = torch.mean(cat[tk][p])
            avg[f'{tk}_{suffix}_hist'] = cat[tk][p]
            ok = torch.logical_and(cat[rk][p, :] < thresh_rot, cat[tk][p, :] < thresh_trans)
            avg[f'reg_success{ps}_{suffix}'] = ok.float().mean()
    return avg


# ---------------------------------------------------------------------- Redwood trajectory files


def read_trajectory(filename, dim=4):
    """`gt.log` / `est.log` -> (keys (n,3) str, traj (n,dim,dim))  (benchmark_predator.py:80-117)."""
    with open(filename) as f:
        lines = f.readlines()
    keys = [[c.strip() for c in ln.split('\t')[0:3]] for ln in lines[0::dim + 1]]
    rows = [ln.split('\t')[0:dim] for i, ln in enumerate(lines) if i % (dim + 1) != 0]
    traj = np.asarray(rows, dtype=np.float64).reshape(-1, dim, dim)
    return np.asarray(keys), traj


def read_trajectory_info(filename, dim=6):
    """`gt.info` -> (n_fragments, information matrices (n,6,6))  (benchmark_predator.py:120-151)."""
    with open(filename) as fid:
        contents = fid.readlines()
    n_pairs = len(contents) // 7
    assert len(contents) == 7 * n_pairs
    info, n_frame = [], 0
    for i in range(n_pairs):
        _, _, n_frame = [int(v) for v in contents[i * 7].strip().split()]
        info.append(np.stack([np.array(ln.split(), dtype=np.float64) for ln in contents[i * 7 + 1:i * 7 + 7]]))
    return n_frame, np.asarray(info, dtype=np.float64).reshape(-1, dim, dim)


def write_trajectory(traj, metadata, filename, dim=4):
    """benchmark_predator.py:176-195 (entries whose third metadata field is falsy are skipped)."""
    with open(filename, 'w') as f:
        for idx in range(traj.shape[0]):
            if metadata[idx][2]:
                p = traj[idx].tolist()
                f.write('\t'.join(map(str, metadata[idx])) + '\n')
                f.write('\n'.join('\t'.join(map('{0:.12f}'.format, p[i])) for i in range(dim)))
                f.write('\n')


class EstLogWriter:
    """Appends predicted poses to `<log_path>/<benchmark>/<scene>/est.log` exactly like
    `GenericRegModel._save_3DMatch_log` (generic_reg_model.py:260-281): header `tgt_idx src_idx -1`,
    four rows of 12-decimal numbers."""

    def __init__(self, log_path: str, benchmark: str):
        self.root = os.path.join(log_path, benchmark)

    @staticmethod
    def parse_path(path: str):
        """('.../<scene>/cloud_bin_<i>.pth') -> (scene, i); the scene is the SECOND path component, as in the
        reference (`src_path.split(os.path.sep)[1]`)."""
        scene = path.split(os.path.sep)[1]
        idx = int(os.path.basename(path).split('_')[-1].replace('.pth', ''))
        return scene, idx

    def append(self, scene: str, src_idx: int, tgt_idx: int, pose):
        pose = _as44(pose.detach().cpu().numpy() if torch.is_tensor(pose) else pose)
        folder = os.path.join(self.root, scene)
        os.makedirs(folder, exist_ok=True)
        with open(os.path.join(folder, 'est.log'), 'a') as fid:
            fid.write('{}\t{}\t{}\n'.format(tgt_idx, src_idx, -1))
            for i in range(4):
                fid.write('\t'.join(map('{0:.12f}'.format, pose[i])) + '\n')

    def append_batch(self, batch: Dict, pred: Dict):
        poses = pred['pose'][-1] if pred['pose'].ndim == 4 else pred['pose']
        for b in range(len(batch['src_xyz'])):
            scene, si = self.parse_path(batch['src_path'][b])
            _, ti = self.parse_path(batch['tgt_path'][b])
            self.append(scene, si, ti, poses[b])


# --------------------------------------------------------------- 3DMatch registration recall


def mat2quat(M):
    """Rotation matrix -> unit quaternion (w, x, y, z), w >= 0: eigenvector of Bar-Itzhack's K matrix for
    the largest eigenvalue (the method nibabel.quaternions.mat2quat documents).  The benchmark only uses
    the vector part inside a quadratic form, which is invariant to the quaternion's sign."""
    Qxx, Qyx, Qzx, Qxy, Qyy, Qzy, Qxz, Qyz, Qzz = np.asarray(M, dtype=np.float64).flat
    K = np.array([[Qxx - Qyy - Qzz, 0, 0, 0],
                  [Qyx + Qxy, Qyy - Qxx - Qzz, 0, 0],
                  [Qzx + Qxz, Qzy + Qyz, Qzz - Qxx - Qyy, 0],
                  [Qyz - Qzy, Qzx - Qxz, Qxy - Qyx, Qxx + Qyy + Qzz]]) / 3.0
    vals, vecs = np.linalg.eigh(K)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    return q * -1 if q[0] < 0 else q


def transformation_error(trans, info):
    """Redwood transformation error: approximate squared RMSE of the ground-truth correspondences
    (benchmark_predator.py:59-77)."""
    er = np.concatenate([trans[:3, 3], mat2quat(trans[:3, :3])[1:]], axis=0)
    return (er.reshape(1, 6) @ info @ er.reshape(6, 1) / info[0, 0]).item()


def rotation_error(R1, R2):
    """Degrees, (b,1)  (benchmark_predator.py:17-40)."""
    R_ = np.matmul(np.transpose(R1, (0, 2, 1)), R2)
    e = np.clip((np.trace(R_, axis1=1, axis2=2) - 1) / 2, -1, 1)
    return (180.0 * np.arccos(e) / math.pi)[:, None]


def translation_error(t1, t2):
    """Metres, (b,)  (benchmark_predator.py:43-56)."""
    return np.linalg.norm((t1 - t2).reshape(t1.shape[0], -1), axis=1)


def evaluate_registration(num_fragment, result, result_pairs, gt_pairs, gt, gt_info, err2=0.2):
    """benchmark_predator.py:223-281: precision, recall, per-result flags (0 good, 1 bad, 2 not in gt) and errors.
    Only non-consecutive ground-truth pairs count."""
    err2 = err2 ** 2
    gt_mask = np.zeros((num_fragment, num_fragment), dtype=np.int64)
    for idx in range(gt_pairs.shape[0]):
        i, j = int(gt_pairs[idx, 0]), int(gt_pairs[idx, 1])
        if j - i > 1:
            gt_mask[i, j] = idx
    n_gt = np.sum(gt_mask > 0)
    errors = np.full(result_pairs.shape[0], np.nan)
    flags, good, n_res = [], 0, 0
    for idx in range(result_pairs.shape[0]):
        i, j = int(result_pairs[idx, 0]), int(result_pairs[idx, 1])
        if gt_mask[i, j] > 0:
            n_res += 1
            g = gt_mask[i, j]
            p = transformation_error(np.linalg.inv(gt[g]) @ result[idx], gt_info[g])
            errors[idx] = p
            good += p <= err2
            flags.append(0 if p <= err2 else 1)
        else:
            flags.append(2)
    if n_res == 0:
        n_res += 1e6
    return good * 1.0 / n_res, good * 1.0 / n_gt, flags, errors


def extract_corresponding_trajectors(est_pairs, gt_pairs, gt_traj):
    """benchmark_predator.py:154-173."""
    ext = np.zeros((len(est_pairs), 4, 4))
    for k, pair in enumerate(est_pairs):
        pair[2] = gt_pairs[0][2]
        ext[k] = gt_traj[np.where((gt_pairs == pair).all(axis=1))[0]]
    return ext


SHORT_NAMES = ['Kitchen', 'Home 1', 'Home 2', 'Hotel 1', 'Hotel 2', 'Hotel 3', 'Study', 'MIT Lab']


def benchmark_3dmatch(est_folder, gt_folder, save_flags=False):
    """Registration recall over the scenes of `gt_folder` (benchmark_predator.py:284-375).
    -> (summary string identical to the reference's, mean recall, per-scene dict)."""
    scenes = sorted(os.listdir(gt_folder))
    re_med, te_med, precision, recall, n_valids = [], [], [], [], []
    out = "Scene\t¦ prec.\t¦ rec.\t¦ re\t¦ te\t¦ samples\t¦\n"
    per_scene = {}
    for idx, scene in enumerate(scenes):
        gt_pairs, gt_traj = read_trajectory(os.path.join(gt_folder, scene, 'gt.log'))
        n_valid = int(sum(abs(int(e[0]) - int(e[1])) > 1 for e in gt_pairs))
        n_valids.append(n_valid)
        n_frag, gt_info = read_trajectory_info(os.path.join(gt_folder, scene, 'gt.info'))
        est_pairs, est_traj = read_trajectory(os.path.join(est_folder, scene, 'est.log'))
        prec, rec, flags, errors = evaluate_registration(n_frag, est_traj, est_pairs, gt_pairs, gt_traj, gt_info)
        ext = extract_corresponding_trajectors(est_pairs, gt_pairs, gt_traj)
        good = np.array(flags) == 0
        re = rotation_error(ext[:, :3, :3], est_traj[:, :3, :3])[good]
        te = translation_error(ext[:, :3, 3:4], est_traj[:, :3, 3:4])[good]
        re_med.append(np.median(re)); te_med.append(np.median(te))
        precision.append(prec); recall.append(rec)
        name = SHORT_NAMES[idx] if idx < len(SHORT_NAMES) else scene
        out += "{}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:3d}¦\n".format(name, prec, rec, np.median(re),
                                                                            np.median(te), n_valid)
        per_scene[scene] = dict(precision=prec, recall=rec, flags=np.array(flags), errors=errors,
                                re_median=float(np.median(re)), te_median=float(np.median(te)), n_valid=n_valid)
        if save_flags:
            np.save(f'{est_folder}/{scene}/flag.npy', flags)
            np.save(f'{est_folder}/{scene}/errors.npy', errors)
    weighted = (np.array(n_valids) * np.array(precision)).sum() / np.sum(n_valids)
    out += "Mean precision: {:.3f}: +- {:.3f}\n".format(np.mean(precision), np.std(precision))
    out += "Weighted precision: {:.3f}\n".format(weighted)
    out += "Mean median RRE: {:.3f}: +- {:.3f}\n".format(np.mean(re_med), np.std(re_med))
    out += "Mean median RTE: {:.3F}: +- {:.3f}\n".format(np.mean(te_med), np.std(te_med))
    return out, float(np.mean(recall)), per_scene


# ------------------------------------------------------ 3DMatch success rate of Deep Global Registration


def compute_rre(R_est, R):
    """Degrees; the cosine is clipped to [-1 + 1e-16, 1 - 1e-16] (benchmark_3dmatch.py:compute_rre)."""
    eps = 1e-16
    return np.arccos(np.clip((np.trace(R_est.T @ R) - 1) / 2, -1 + eps, 1 - eps)) * 180. / np.pi


def compute_rte(t, t_est):
    return np.linalg.norm(t - t_est)


def benchmark_dgr(est_folder, gt_folder, re_thres=15, te_thres=0.3):
    """DGR success rate (RRE < re_thres degrees and RTE < te_thres) over the scenes of `gt_folder`
    (benchmark/benchmark_3dmatch.py:benchmark_dgr), with the reference's rules: the i-th est.log entry is scored
    against the i-th gt.log entry whatever their keys, and the errors are those of the inverted poses.
    -> (summary string identical to the reference's, {scene: dict(rre, rte, success) arrays per est.log entry})."""
    import warnings
    scenes = sorted(os.listdir(gt_folder))
    out = "Scene\t¦ success.\t¦ rre\t¦ rte\t¦ rre_all\t¦ rte_all\t¦\n"
    success, rre_ok, rte_ok, rre_all, rte_all = [], [], [], [], []
    per_scene = {}

    def row(name, s, ro, to, ra, ta):
        with warnings.catch_warnings():            # np.mean([]) of a scene without a success is nan, as in the reference
            warnings.simplefilter('ignore', RuntimeWarning)
            return "{}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:.3f}\t¦ {:.3f}¦\n".format(
                name, np.mean(s), np.mean(ro), np.mean(to), np.mean(ra), np.mean(ta))

    for idx, scene in enumerate(scenes):
        _, gt_traj = read_trajectory(os.path.join(gt_folder, scene, 'gt.log'))
        _, est_traj = read_trajectory(os.path.join(est_folder, scene, 'est.log'))
        s_flag, s_ro, s_to, s_ra, s_ta = [], [], [], [], []
        for i in range(len(est_traj)):
            est_inv, gt_inv = np.linalg.inv(est_traj[i]), np.linalg.inv(gt_traj[i])
            rot_error = compute_rre(est_inv[:3, :3], gt_inv[:3, :3])
            trans_error = compute_rte(est_inv[:3, 3], gt_inv[:3, 3])
            s_ra.append(rot_error)
            s_ta.append(trans_error)
            ok = bool(rot_error < re_thres and trans_error < te_thres)
            s_flag.append(ok)
            if ok:
                s_ro.append(rot_error)
                s_to.append(trans_error)
        out += row(SHORT_NAMES[idx] if idx < len(SHORT_NAMES) else scene, s_flag, s_ro, s_to, s_ra, s_ta)
        per_scene[scene] = dict(rre=np.array(s_ra, dtype=np.float64), rte=np.array(s_ta, dtype=np.float64),
                                success=np.array(s_flag, dtype=bool))
        success += s_flag; rre_ok += s_ro; rte_ok += s_to; rre_all += s_ra; rte_all += s_ta
    out += row('Avg', success, rre_ok, rte_ok, rre_all, rte_all)
    return out, per_scene


# ------------------------------------------------------------------------------ ModelNet metrics


def _se3_inv(p):
    r = p[..., :3, :3].transpose(-1, -2)
    return torch.cat([r, -(r @ p[..., :3, 3:4])], dim=-1)


def _se3_cat(a, b):
    return torch.cat([a[..., :3, :3] @ b[..., :3, :3], a[..., :3, :3] @ b[..., :3, 3:4] + a[..., :3, 3:4]], dim=-1)


def _se3_transform(p, xyz):
    return xyz @ p[..., :3, :3].transpose(-1, -2) + p[..., :3, 3:4].transpose(-1, -2)


def compute_modelnet_metrics(data: Dict, pred_transforms: torch.Tensor) -> Dict[str, np.ndarray]:
    """benchmark_modelnet.py:33-82: DCP-style Euler/translation errors, isotropic errors, modified Chamfer
    distance.  data: points_src/points_ref/points_raw (B,N,>=3), transform_gt (B,3,4)."""
    from scipy.spatial.transform import Rotation

    def euler(m):
        return np.stack([Rotation.from_matrix(r).as_euler('xyz', degrees=True) for r in m])

    def sqdist(a, b):
        return torch.sum((a[:, :, None, :] - b[:, None, :, :]) ** 2, dim=-1)

    with torch.no_grad():
        gt = data['transform_gt']
        src, ref, raw = (data[k][..., :3] for k in ('points_src', 'points_ref', 'points_raw'))
        e_gt = euler(gt[:, :3, :3].detach().cpu().numpy())
        e_pr = euler(pred_transforms[:, :3, :3].detach().cpu().numpy())
        t_gt, t_pr = gt[:, :3, 3], pred_transforms[:, :3, 3]
        cat = _se3_cat(_se3_inv(gt), pred_transforms)
        trace = cat[:, 0, 0] + cat[:, 1, 1] + cat[:, 2, 2]
        rot_deg = torch.acos(torch.clamp(0.5 * (trace - 1), min=-1.0, max=1.0)) * 180.0 / np.pi
        src_t = _se3_transform(pred_transforms, src)
        src_clean = _se3_transform(_se3_cat(pred_transforms, _se3_inv(gt)), raw)
        chamfer = torch.mean(torch.min(sqdist(src_t, raw), dim=-1)[0], dim=1) + \
            torch.mean(torch.min(sqdist(ref, src_clean), dim=-1)[0], dim=1)
        npy = lambda t: t.detach().cpu().numpy()
        return {'r_mse': np.mean((e_gt - e_pr) ** 2, axis=1), 'r_mae': np.mean(np.abs(e_gt - e_pr), axis=1),
                't_mse': npy(torch.mean((t_gt - t_pr) ** 2, dim=1)), 't_mae': npy(torch.mean(torch.abs(t_gt - t_pr), dim=1)),
                'err_r_deg': npy(rot_deg), 'err_t': npy(cat[:, :, 3].norm(dim=-1)), 'chamfer_dist': npy(chamfer)}


def summarize_modelnet_metrics(metrics: Dict[str, np.ndarray]) -> Dict[str, float]:
    """benchmark_modelnet.py:85-97."""
    out = {}
    for k, v in metrics.items():
        if k.endswith('mse'):
            out[k[:-3] + 'rmse'] = np.sqrt(np.mean(v))
        elif k.startswith('err'):
            out[k + '_mean'] = np.mean(v)
            out[k + '_rmse'] = np.sqrt(np.mean(v ** 2))
        else:
            out[k] = np.mean(v)
    return out


# ------------------------------------------------------------------- test loop (reference: test.py)


def icp_levels(voxels, radii=None, level_iters=None, radius: float = None, max_iteration: int = 30):
    """The multi-scale ICP pyramid as [(V_l, R_l, I_l)], or ValueError naming what is wrong.  voxels: L > 0 values,
    strictly decreasing, all > 0 except that the last may be 0 (the full clouds, not down-sampled).  radii: the
    levels' max correspondence distances, each finite and > 0 (default: V_l, Open3D's colored-ICP tutorial's rule; the
    positional radius at V = 0).  level_iters: iterations at most per level, each >= 0 (default: max_iteration)."""
    vox = [float(v) for v in voxels]
    L = len(vox)
    if L == 0:
        raise ValueError('icp voxels: expected at least one level')
    for name, vals in (('radii', radii), ('level_iters', level_iters)):
        if vals is not None and len(vals) != L:
            raise ValueError(f'icp {name}: {len(vals)} values for {L} voxels')
    if not all(math.isfinite(v) for v in vox) or any(b >= a for a, b in zip(vox, vox[1:])) or \
            any(v <= 0.0 for v in vox[:-1]) or vox[-1] < 0.0:
        raise ValueError(f'icp voxels {vox}: must be finite and strictly decreasing, all > 0 except a last 0')
    rad = [float(r) for r in radii] if radii is not None else [v if v > 0.0 else radius for v in vox]
    if not all(r is not None and math.isfinite(r) and r > 0.0 for r in rad):
        raise ValueError(f'icp radii {rad}: must be finite and > 0')
    its = [int(i) for i in level_iters] if level_iters is not None else [int(max_iteration)] * L
    if any(i < 0 for i in its):
        raise ValueError(f'icp level_iters {its}: must be >= 0')
    return list(zip(vox, rad, its))


def _stack_levels(results):
    """Per-level (B,4) results -> (B,L,4), torch or numpy as they come."""
    if torch.is_tensor(results[0]):
        return torch.stack(results, 1)
    return np.stack([np.asarray(r) for r in results], 1)


def icp_refine(src_list, tgt_list, init, radius: float, max_iteration: int = 30, method: str = 'point_to_point',
               normal_radius: float = None, normal_max_nn: int = 30, epsilon: float = 1e-3, loss: str = 'l2',
               loss_k: float = None, normals=None, icp=None, estimate_normals=None, colors=None,
               lambda_geometric: float = 0.968, color_gradients=None, voxels=None, radii=None, level_iters=None,
               return_levels: bool = False, voxel_down_sample=None):
    """Refine B poses init (B,3,4) by ICP of src_list onto tgt_list: the normals each method needs, then one icp call.
    -> icp's (pose (B,3,4), result).
    icp(src_list, tgt_list, init, radius, max_iteration, ...) defaults to `ops.icp`; point-to-point passes nothing
    more.  method='point_to_plane': the targets' normals come from estimate_normals(tgt_list, normal_radius (default
    2 * radius), normal_max_nn) (default `ops.estimate_normals`), and icp gets method=method, tgt_normals=.
    method='generalized': the normals of src_list + tgt_list come from one estimate_normals call, and icp also gets
    src_normals=.  normals=(src_normals, tgt_normals) skips the estimation (only the ones the method needs are
    passed on).  epsilon, loss and loss_k (see `ops.icp`) are passed on only when they differ from their defaults.
    method='colored' (Open3D's registration_colored_icp): colors=(src_colors, tgt_colors), B (n,3) rgb arrays each;
    the targets' normals are estimated as for point_to_plane, then their intensity gradients by
    color_gradients(tgt_list, normals, tgt_colors, 2 * radius, 30) (default `ops.color_gradients`; Open3D's own
    parameters), and icp also gets src_colors=, tgt_colors=, tgt_color_gradients= and lambda_geometric=.
    Multi-scale ICP (Open3D's colored-ICP tutorial, the tensor API's multi_scale_icp): voxels, radii and level_iters as
    `icp_levels` takes them.  Level l down-samples src_list + tgt_list (and their colours, for 'colored') in one
    voxel_down_sample(clouds, V_l, colors=) call (default `ops.voxel_down_sample`; none at V = 0), then runs the
    single-level refinement above at R_l for at most I_l iterations from the previous level's pose (level 0 from
    init): normals at 2 R_l with normal_max_nn, gradients at 2 R_l with 30.  normals= and normal_radius= are refused
    with voxels.  -> the last level's (pose, result); return_levels adds the (B,L,4) results of every level (L = 1
    without voxels)."""
    if voxels is None:
        pose, res = _icp_level(src_list, tgt_list, init, radius, max_iteration, method, normal_radius, normal_max_nn,
                               epsilon, loss, loss_k, normals, icp, estimate_normals, colors, lambda_geometric,
                               color_gradients)
        return (pose, res, _stack_levels([res])) if return_levels else (pose, res)
    if normals is not None or normal_radius is not None:
        raise ValueError('icp_refine: normals= and normal_radius= do not go with voxels (each level estimates its own '
                         'normals at 2 R_l)')
    plan = icp_levels(voxels, radii, level_iters, radius, max_iteration)
    if method == 'colored' and colors is None:
        raise ValueError('icp_refine: colored ICP needs colors=(src_colors, tgt_colors)')
    if voxel_down_sample is None:
        from .ops import voxel_down_sample
    B = len(src_list)
    colors = colors if method == 'colored' else None
    pose, results = init, []
    for v, r, it in plan:
        src, tgt, col = src_list, tgt_list, colors
        if v > 0.0:
            down, dc = voxel_down_sample(list(src_list) + list(tgt_list), v,
                                         colors=None if colors is None else list(colors[0]) + list(colors[1]))
            src, tgt = down[:B], down[B:]
            col = None if dc is None else (dc[:B], dc[B:])
        pose, res = _icp_level(src, tgt, pose, r, it, method, None, normal_max_nn, epsilon, loss, loss_k, None, icp,
                               estimate_normals, col, lambda_geometric, color_gradients)
        results.append(res)
    return (pose, res, _stack_levels(results)) if return_levels else (pose, res)


def _icp_level(src_list, tgt_list, init, radius, max_iteration, method, normal_radius, normal_max_nn, epsilon, loss,
               loss_k, normals, icp, estimate_normals, colors, lambda_geometric, color_gradients):
    """`icp_refine` at one scale: the normals and gradients the method needs, then one icp call."""
    if icp is None:
        from .ops import icp
    if method == 'colored' and colors is None:
        raise ValueError('icp_refine: colored ICP needs colors=(src_colors, tgt_colors)')
    kw = {}
    if method != 'point_to_point':
        if normals is None:
            if estimate_normals is None:
                from .ops import estimate_normals
            nr = 2.0 * radius if normal_radius is None else normal_radius
            if method == 'generalized':
                B = len(src_list)
                est = estimate_normals(list(src_list) + list(tgt_list), nr, normal_max_nn)
                normals = est[:B], est[B:]
            else:
                normals = None, estimate_normals(tgt_list, nr, normal_max_nn)
        kw.update(method=method, tgt_normals=normals[1])
        if method == 'generalized':
            kw['src_normals'] = normals[0]
    if method == 'colored':
        if color_gradients is None:
            from .ops import color_gradients
        grads = color_gradients(tgt_list, normals[1], colors[1], 2.0 * radius, 30)
        kw.update(src_colors=colors[0], tgt_colors=colors[1], tgt_color_gradients=grads,
                  lambda_geometric=lambda_geometric)
    if epsilon != 1e-3:
        kw['epsilon'] = epsilon
    if loss != 'l2':
        kw['loss'] = loss
    if loss_k is not None:
        kw['loss_k'] = loss_k
    return icp(src_list, tgt_list, init, radius, max_iteration, **kw)



def add_icp_arguments(ap, icp_help: str):
    """The ICP refinement flags of a command line, for `icp_refine`: --icp R (help text icp_help), --icp_iters,
    --icp_method, --normal_radius, --normal_max_nn, --icp_epsilon, --icp_loss, --icp_loss_k,
    --icp_lambda_geometric, and the multi-scale pyramid's --icp_voxels, --icp_radii and --icp_level_iters."""
    from .ops import ICP_LOSSES, ICP_METHODS
    ap.add_argument('--icp', type=float, metavar='R', help=icp_help)
    ap.add_argument('--icp_iters', type=int, default=30, help='ICP iterations at most (with --icp)')
    ap.add_argument('--icp_method', choices=ICP_METHODS, default='point_to_point',
                    help='ICP error metric (with --icp); point_to_plane estimates the target normals first, '
                         'generalized those of both clouds, colored the target normals and colour gradients '
                         '(needs .ply inputs with red, green and blue)')
    ap.add_argument('--normal_radius', type=float, metavar='NR',
                    help='Normal estimation radius of point_to_plane / generalized ICP (default: 2 * the --icp radius)')
    ap.add_argument('--normal_max_nn', type=int, default=30,
                    help='Neighbours at most of the normal estimation (with point_to_plane / generalized ICP)')
    ap.add_argument('--icp_epsilon', type=float, default=1e-3,
                    help='Covariance epsilon of generalized ICP, in (0, 1]')
    ap.add_argument('--icp_loss', choices=ICP_LOSSES, default='l2',
                    help='Robust kernel of point_to_plane / generalized ICP (needs --icp_loss_k unless l2)')
    ap.add_argument('--icp_loss_k', type=float, metavar='K', help='The robust kernel\'s parameter k')
    ap.add_argument('--icp_lambda_geometric', type=float, default=0.968, metavar='L',
                    help='Weight of the geometric residual of colored ICP, in [0, 1]')
    ap.add_argument('--icp_voxels', type=_number_list(float), metavar='V1,V2,...',
                    help='Multi-scale ICP (with --icp): voxel sizes, strictly decreasing, a last 0 meaning the full '
                         'clouds; every level down-samples both clouds, estimates its own normals at 2 R_l and starts '
                         'from the previous level\'s pose')
    ap.add_argument('--icp_radii', type=_number_list(float), metavar='R1,...',
                    help='Max correspondence distance per level (with --icp_voxels; default: the voxel sizes, the '
                         '--icp radius at a 0 voxel)')
    ap.add_argument('--icp_level_iters', type=_number_list(int), metavar='I1,...',
                    help='ICP iterations at most per level (with --icp_voxels; default: --icp_iters at every level)')


def _number_list(kind):
    """argparse type: 'a,b,c' -> [kind(a), kind(b), kind(c)]."""
    def parse(text):
        try:
            return [kind(v) for v in text.split(',')]
        except ValueError:
            raise argparse.ArgumentTypeError(f'expected comma-separated {kind.__name__} values, got {text!r}')
    return parse


def check_icp_arguments(ap, opt, colors: bool = False):
    """Reject, as usage errors and before any model is loaded, a robust --icp_loss without its --icp_loss_k, an
    --icp_lambda_geometric outside [0, 1], --icp_method colored on a command line whose inputs carry no colour
    (colors=False), and a pyramid that `icp_levels` refuses, --icp_voxels / --icp_radii / --icp_level_iters without
    --icp, the last two without --icp_voxels, or --normal_radius with --icp_voxels."""
    if opt.icp_loss != 'l2' and opt.icp_loss_k is None:
        ap.error(f'--icp_loss {opt.icp_loss} needs --icp_loss_k')
    if not 0.0 <= opt.icp_lambda_geometric <= 1.0:
        ap.error(f'--icp_lambda_geometric {opt.icp_lambda_geometric} must be in [0, 1]')
    if opt.icp_method == 'colored' and not colors:
        ap.error('--icp_method colored needs coloured clouds, and this command line reads none')
    given = [f for f in ('icp_voxels', 'icp_radii', 'icp_level_iters') if getattr(opt, f) is not None]
    if given and opt.icp is None:
        ap.error(f'--{given[0]} needs --icp')
    if given and opt.icp_voxels is None:
        ap.error(f'--{given[0]} needs --icp_voxels')
    if opt.icp_voxels is not None:
        if opt.normal_radius is not None:
            ap.error('--normal_radius does not go with --icp_voxels: every level estimates its normals at 2 R_l')
        try:
            icp_levels(opt.icp_voxels, opt.icp_radii, opt.icp_level_iters, opt.icp, opt.icp_iters)
        except ValueError as e:
            ap.error(f'--icp_voxels / --icp_radii / --icp_level_iters: {e}')


def add_outlier_arguments(ap):
    """The outlier-removal flags of a command line, for `remove_outliers`: --remove_statistical_outlier K S and
    --remove_radius_outlier N R."""
    ap.add_argument('--remove_statistical_outlier', nargs=2, metavar=('K', 'S'),
                    help='Drop the points whose mean distance to their K nearest neighbours is at least S standard '
                         'deviations above their cloud\'s mean (Open3D\'s remove_statistical_outlier), on the clouds as '
                         'read, before the crop')
    ap.add_argument('--remove_radius_outlier', nargs=2, metavar=('N', 'R'),
                    help='Drop the points with fewer than N points within radius R (Open3D\'s remove_radius_outlier), '
                         'on the clouds as read, after --remove_statistical_outlier and before the crop')


def check_outlier_arguments(ap, opt):
    """Reject, as usage errors, outlier options the filters would refuse, before any model is loaded, and turn the
    flags' values into (nb_neighbors int, std_ratio float) and (nb_points int, radius float)."""
    from .ops import OUTLIER_MAX_NEIGHBORS
    for flag, first, second in (('statistical', 'K', 'S'), ('radius', 'N', 'R')):
        name = f'remove_{flag}_outlier'
        vals = getattr(opt, name)
        if vals is None:
            continue
        try:
            n, v = int(vals[0]), float(vals[1])
        except ValueError:
            ap.error(f'--{name} {" ".join(vals)}: expected an integer {first} and a number {second}')
        if flag == 'statistical' and not (1 <= n <= OUTLIER_MAX_NEIGHBORS and math.isfinite(v) and v > 0.0):
            ap.error(f'--{name} {n} {v}: K must be in 1..{OUTLIER_MAX_NEIGHBORS} and S finite and > 0')
        if flag == 'radius' and not (n >= 1 and math.isfinite(v) and v > 0.0):
            ap.error(f'--{name} {n} {v}: N must be >= 1 and R finite and > 0')
        setattr(opt, name, (n, v))


def remove_outliers(clouds, colors=None, statistical=None, radius=None, remove_statistical_outlier=None,
                    remove_radius_outlier=None):
    """The clouds (and colours) of a command line filtered as its outlier flags ask: `ops.remove_statistical_outlier`
    with statistical = (nb_neighbors, std_ratio), then `ops.remove_radius_outlier` with radius = (nb_points, radius)
    on what is left, every cloud in one call each (either function injectable).
    clouds / colors: lists of (n,3) host arrays.  -> (clouds, colours or None, indices): lists of host float64 arrays
    and of int64 arrays, the rows of each input cloud that survive, ascending."""
    if remove_statistical_outlier is None or remove_radius_outlier is None:
        from . import ops
        remove_statistical_outlier = remove_statistical_outlier or ops.remove_statistical_outlier
        remove_radius_outlier = remove_radius_outlier or ops.remove_radius_outlier
    index = [np.arange(np.asarray(c).shape[0], dtype=np.int64) for c in clouds]
    for fn, args in ((remove_statistical_outlier, statistical), (remove_radius_outlier, radius)):
        if args is None:
            continue
        kept, kc, ki = fn(clouds, args[0], args[1], colors=colors)
        clouds = [np.asarray(torch.as_tensor(c).cpu(), dtype=np.float64) for c in kept]
        colors = None if kc is None else [np.asarray(torch.as_tensor(c).cpu(), dtype=np.float64) for c in kc]
        index = [ix[np.asarray(torch.as_tensor(k).cpu(), dtype=np.int64)] for ix, k in zip(index, ki)]
    return clouds, colors, index


def load_icp_colors(ap, opt, paths):
    """With --icp and --icp_method colored: the rgb (N,3) of every file of `paths` (`pointio.load_point_cloud_colors`),
    a file without colours being a usage error that names it; else None."""
    if opt.icp is None or opt.icp_method != 'colored':
        return None
    from .pointio import load_point_cloud_colors
    out = []
    for path in paths:
        try:
            out.append(load_point_cloud_colors(path)[1])
        except ValueError as e:
            ap.error(f'--icp_method colored: {e}')
    return out


def icp_forward(forward_fn, radius: float, max_iteration: int = 30, icp=None, method: str = 'point_to_point',
                normal_radius: float = None, normal_max_nn: int = 30, estimate_normals=None, epsilon: float = 1e-3,
                loss: str = 'l2', loss_k: float = None, lambda_geometric: float = 0.968, color_gradients=None,
                voxels=None, radii=None, level_iters=None):
    """Wrap `forward_fn(batch) -> pred` so that the final pose of every pair is refined by ICP on the batch's full
    clouds: -> a NEW dict with pred's entries, pose (1,B,3,4) float64 the refined poses and pose_coarse
    (1,B,3,4) float64 the network's final poses (so that `compute_metrics` reports both, and EstLogWriter writes the
    refined ones).  pred's own tensors are not written to (a graphed forward owns them).
    The refinement is `icp_refine` with these arguments, icp, estimate_normals, color_gradients and the pyramid's
    voxels, radii and level_iters included; with
    method='colored' the colours are the batch's src_colors / tgt_colors (a batch without them raises ValueError)."""
    from .ops import ICP_METHODS
    if method not in ICP_METHODS:
        raise ValueError(f'icp_forward: unknown method {method!r}')
    def run(batch):
        pred = forward_fn(batch)
        coarse = pred['pose'][-1].to(torch.float64)                     # (B,3,4), a new tensor
        kw = {} if voxels is None else dict(voxels=voxels, radii=radii, level_iters=level_iters)
        if method == 'colored':
            if 'src_colors' not in batch or 'tgt_colors' not in batch:
                raise ValueError('icp_forward: colored ICP needs the batch\'s src_colors and tgt_colors')
            kw.update(colors=(batch['src_colors'], batch['tgt_colors']), lambda_geometric=lambda_geometric,
                      color_gradients=color_gradients)
        pose, _ = icp_refine(batch['src_xyz'], batch['tgt_xyz'], coarse, radius, max_iteration, method,
                             normal_radius, normal_max_nn, epsilon, loss, loss_k, icp=icp,
                             estimate_normals=estimate_normals, **kw)
        out = dict(pred)
        out['pose'] = torch.as_tensor(pose, dtype=torch.float64, device=coarse.device).reshape(coarse.shape)[None]
        out['pose_coarse'] = coarse[None]
        return out
    return run


def ransac_refine(pred, src_list, tgt_list, radius: float, max_iteration: int = 100000, confidence: float = 0.999,
                  ransac_n: int = 3, edge_length: float = 0.9, distance: float = None, overlap: float = 0.5,
                  seed: int = 0, pair_base: int = 0, ransac=None, correspondences=None):
    """A robust pose for every pair of a forward's output `pred`: RANSAC (`ops.ransac`, max correspondence distance
    `radius`, validated on src_list / tgt_list) over RegTR's two-way correspondences with predicted overlap above
    `overlap` (`ops.regtr_correspondences`).  -> ransac's (pose (B,3,4), result (B,5)).
    ransac(src_list, tgt_list, corr_src, corr_tgt, radius, max_iteration, ...) and correspondences(pred, overlap)
    default to the `ops` functions."""
    if ransac is None:
        from .ops import ransac
    if correspondences is None:
        from .ops import regtr_correspondences as correspondences
    corr_src, corr_tgt, corr_mask = correspondences(pred, overlap)
    return ransac(src_list, tgt_list, corr_src, corr_tgt, radius, max_iteration, confidence=confidence,
                  ransac_n=ransac_n, edge_length=edge_length, distance=distance, corr_mask=corr_mask, seed=seed,
                  pair_base=pair_base)


def add_ransac_arguments(ap, ransac_help: str):
    """The RANSAC flags of a command line, for `ransac_refine`: --ransac R (help text ransac_help), --ransac_iters,
    --ransac_confidence, --ransac_n, --ransac_edge, --ransac_dist, --ransac_overlap and --ransac_seed."""
    ap.add_argument('--ransac', type=float, metavar='R', help=ransac_help)
    ap.add_argument('--ransac_iters', type=int, default=100000, help='RANSAC hypotheses at most (with --ransac)')
    ap.add_argument('--ransac_confidence', type=float, default=0.999,
                    help='RANSAC stops early once this confidence is reached, in [0, 1]')
    ap.add_argument('--ransac_n', type=int, default=3, help='Correspondences per RANSAC sample, 3..16')
    ap.add_argument('--ransac_edge', type=float, default=0.9,
                    help='Edge-length checker\'s similarity threshold (0: off)')
    ap.add_argument('--ransac_dist', type=float, metavar='D',
                    help='Distance checker\'s threshold (default: off)')
    ap.add_argument('--ransac_overlap', type=float, default=0.5,
                    help='Correspondences whose predicted overlap is above this take part in RANSAC')
    ap.add_argument('--ransac_seed', type=int, default=0, help='Seed of the RANSAC samples')


def check_ransac_arguments(ap, opt):
    """Reject, as a usage error, RANSAC options `ops.ransac` would refuse, before any model is loaded."""
    from .ops import RANSAC_MAX_N
    if opt.ransac is None:
        return
    if not opt.ransac > 0.0:
        ap.error(f'--ransac {opt.ransac} must be > 0')
    if not 3 <= opt.ransac_n <= RANSAC_MAX_N:
        ap.error(f'--ransac_n {opt.ransac_n} must be in 3..{RANSAC_MAX_N}')
    if not 0 <= opt.ransac_iters < 2 ** 31:
        ap.error(f'--ransac_iters {opt.ransac_iters} must be >= 0')
    if not 0.0 <= opt.ransac_confidence <= 1.0:
        ap.error(f'--ransac_confidence {opt.ransac_confidence} must be in [0, 1]')
    for flag, v in (('--ransac_edge', opt.ransac_edge), ('--ransac_dist', opt.ransac_dist)):
        if v is not None and not (math.isfinite(v) and v >= 0.0):
            ap.error(f'{flag} {v} must be a finite value >= 0')
    if not 0 <= opt.ransac_seed < 2 ** 64:
        ap.error(f'--ransac_seed {opt.ransac_seed} must be in [0, 2^64)')


def ransac_kwargs(opt) -> Dict:
    """`ransac_refine`'s keyword arguments from the parsed --ransac_* flags."""
    return dict(max_iteration=opt.ransac_iters, confidence=opt.ransac_confidence, ransac_n=opt.ransac_n,
                edge_length=opt.ransac_edge, distance=opt.ransac_dist, overlap=opt.ransac_overlap,
                seed=opt.ransac_seed)


def ransac_forward(forward_fn, radius: float, max_iteration: int = 100000, confidence: float = 0.999,
                   ransac_n: int = 3, edge_length: float = 0.9, distance: float = None, overlap: float = 0.5,
                   seed: int = 0, ransac=None, correspondences=None, icp_radius: float = None, icp_kwargs=None,
                   icp=None, estimate_normals=None):
    """Wrap `forward_fn(batch) -> pred` so that every pair's pose comes from RANSAC over the network's
    correspondences (`ransac_refine` with these arguments, validated on the batch's full clouds): -> a NEW dict with
    pred's entries, pose (1,B,3,4) float64 the RANSAC poses and pose_coarse (1,B,3,4) float64 the network's final
    poses.  With icp_radius, ICP then starts from the RANSAC poses (Open3D's global-then-local pipeline:
    `icp_refine` with icp_radius, icp_kwargs (its keyword arguments), icp and estimate_normals): pose is the refined
    pose and pose_ransac the RANSAC one.  pred's own tensors are not written to."""
    def run(batch):
        pred = forward_fn(batch)
        coarse = pred['pose'][-1].to(torch.float64)                     # (B,3,4), a new tensor
        pose, _ = ransac_refine(pred, batch['src_xyz'], batch['tgt_xyz'], radius, max_iteration, confidence,
                                ransac_n, edge_length, distance, overlap, seed, ransac=ransac,
                                correspondences=correspondences)
        pose = torch.as_tensor(pose, dtype=torch.float64, device=coarse.device).reshape(coarse.shape)
        out = dict(pred)
        out['pose_coarse'] = coarse[None]
        if icp_radius is not None:
            out['pose_ransac'] = pose[None]
            pose, _ = icp_refine(batch['src_xyz'], batch['tgt_xyz'], pose, icp_radius, icp=icp,
                                 estimate_normals=estimate_normals, **(icp_kwargs or {}))
            pose = torch.as_tensor(pose, dtype=torch.float64, device=coarse.device).reshape(coarse.shape)
        out['pose'] = pose[None]
        return out
    return run


def fgr_refine(pred, src_list, tgt_list, overlap: float = 0.5, pair_base: int = 0, fgr=None, correspondences=None,
               **fgr_kwargs):
    """A global pose for every pair of a forward's output `pred`: Fast Global Registration (`ops.fgr`, normalised by
    src_list / tgt_list, fgr_kwargs its options) over RegTR's two-way correspondences with predicted overlap above
    `overlap` (`ops.regtr_correspondences`).  -> fgr's (pose (B,3,4), result (B,4)).
    fgr(src_list, tgt_list, corr_src, corr_tgt, corr_mask, pair_base=, ...) and correspondences(pred, overlap) default
    to the `ops` functions."""
    if fgr is None:
        from .ops import fgr
    if correspondences is None:
        from .ops import regtr_correspondences as correspondences
    corr_src, corr_tgt, corr_mask = correspondences(pred, overlap)
    return fgr(src_list, tgt_list, corr_src, corr_tgt, corr_mask, pair_base=pair_base, **fgr_kwargs)


def add_fgr_arguments(ap, fgr_help: str):
    """The FGR flags of a command line, for `fgr_refine` and `fpfh_register`: --fgr (help text fgr_help), --fgr_dist,
    --fgr_iters, --fgr_division, --fgr_tuple_scale, --fgr_max_tuples, --fgr_tuple_test, --fgr_no_tuple_test,
    --fgr_no_decrease_mu, --fgr_absolute_scale, --fgr_seed and --fgr_overlap."""
    ap.add_argument('--fgr', action='store_true', help=fgr_help)
    ap.add_argument('--fgr_dist', type=float, metavar='D',
                    help='FGR maximum correspondence distance, the end of its GNC schedule (default: 0.025; with '
                         '--fpfh 0.5 V)')
    ap.add_argument('--fgr_iters', type=int, default=64, help='FGR iterations')
    ap.add_argument('--fgr_division', type=float, default=1.4, help='FGR divisor of the GNC parameter, > 0')
    ap.add_argument('--fgr_tuple_scale', type=float, default=0.95, help='FGR tuple test similarity, in (0, 1]')
    ap.add_argument('--fgr_max_tuples', type=int, default=1000, help='FGR tuples kept at most by the tuple test')
    ap.add_argument('--fgr_tuple_test', action='store_true',
                    help='Run the tuple test on the predicted correspondences (the feature path always does, unless '
                         '--fgr_no_tuple_test)')
    ap.add_argument('--fgr_no_tuple_test', action='store_true', help='Skip the tuple test on FPFH matches (--fpfh)')
    ap.add_argument('--fgr_no_decrease_mu', action='store_true', help='Keep FGR\'s GNC parameter fixed')
    ap.add_argument('--fgr_absolute_scale', action='store_true',
                    help='Do not rescale the clouds to unit size before the FGR solve')
    ap.add_argument('--fgr_seed', type=int, default=0, help='Seed of the FGR tuple draws')
    ap.add_argument('--fgr_overlap', type=float, default=0.5,
                    help='Correspondences whose predicted overlap is above this take part in FGR')


def check_fgr_arguments(ap, opt):
    """Reject, as usage errors, FGR options `ops.fgr` would refuse and flag combinations that make no sense, before
    any model is loaded, and fill in --fgr_dist (0.5 V with --fpfh V, else 0.025).  Call before
    `check_fpfh_arguments`, which then leaves --ransac unset."""
    from .ops import FGR_MAX_TUPLES
    if not opt.fgr:
        return
    fpfh = getattr(opt, 'fpfh', None)
    if opt.ransac is not None:
        ap.error('--fgr and --ransac are exclusive: choose one global registration')
    if fpfh is not None and opt.fpfh_no_mutual:
        ap.error('--fpfh_no_mutual cannot be used with --fgr: FGR always keeps the mutual matches only')
    if fpfh is None and opt.fgr_no_tuple_test:
        ap.error('--fgr_no_tuple_test applies to --fpfh; on predicted correspondences the tuple test is off unless '
                 '--fgr_tuple_test')
    if opt.fgr_dist is None:
        opt.fgr_dist = 0.5 * fpfh if fpfh is not None and fpfh > 0.0 else 0.025
    for flag, v in (('--fgr_dist', opt.fgr_dist), ('--fgr_division', opt.fgr_division)):
        if not (math.isfinite(v) and v > 0.0):
            ap.error(f'{flag} {v} must be a finite value > 0')
    if not 0 <= opt.fgr_iters < 2 ** 31:
        ap.error(f'--fgr_iters {opt.fgr_iters} must be >= 0')
    if not 0.0 < opt.fgr_tuple_scale <= 1.0:
        ap.error(f'--fgr_tuple_scale {opt.fgr_tuple_scale} must be in (0, 1]')
    if not 1 <= opt.fgr_max_tuples <= FGR_MAX_TUPLES:
        ap.error(f'--fgr_max_tuples {opt.fgr_max_tuples} must be in 1..{FGR_MAX_TUPLES}')
    if not 0 <= opt.fgr_seed < 2 ** 64:
        ap.error(f'--fgr_seed {opt.fgr_seed} must be in [0, 2^64)')


def fgr_kwargs(opt) -> Dict:
    """`ops.fgr`'s keyword arguments from the parsed --fgr_* flags (without --fgr_overlap).  The tuple test runs on FPFH
    matches (--fpfh) unless --fgr_no_tuple_test, and on predicted correspondences only with --fgr_tuple_test."""
    tuple_test = not opt.fgr_no_tuple_test if getattr(opt, 'fpfh', None) is not None else opt.fgr_tuple_test
    return dict(maximum_correspondence_distance=opt.fgr_dist, iteration_number=opt.fgr_iters,
                division_factor=opt.fgr_division, decrease_mu=not opt.fgr_no_decrease_mu,
                use_absolute_scale=opt.fgr_absolute_scale, tuple_test=tuple_test, tuple_scale=opt.fgr_tuple_scale,
                maximum_tuple_count=opt.fgr_max_tuples, seed=opt.fgr_seed)


def fgr_forward(forward_fn, overlap: float = 0.5, fgr=None, correspondences=None, icp_radius: float = None,
                icp_kwargs=None, icp=None, estimate_normals=None, **fgr_kwargs):
    """Wrap `forward_fn(batch) -> pred` so that every pair's pose comes from FGR over the network's correspondences
    (`fgr_refine` with overlap and fgr_kwargs, normalised by the batch's full clouds): -> a NEW dict with pred's
    entries, pose (1,B,3,4) float64 the FGR poses and pose_coarse (1,B,3,4) float64 the network's final poses.  With
    icp_radius, ICP then starts from the FGR poses (`icp_refine` with icp_radius, icp_kwargs, icp and
    estimate_normals): pose is the refined pose and pose_fgr the FGR one.  pred's own tensors are not written to."""
    def run(batch):
        pred = forward_fn(batch)
        coarse = pred['pose'][-1].to(torch.float64)                     # (B,3,4), a new tensor
        pose, _ = fgr_refine(pred, batch['src_xyz'], batch['tgt_xyz'], overlap, fgr=fgr,
                             correspondences=correspondences, **fgr_kwargs)
        pose = torch.as_tensor(pose, dtype=torch.float64, device=coarse.device).reshape(coarse.shape)
        out = dict(pred)
        out['pose_coarse'] = coarse[None]
        if icp_radius is not None:
            out['pose_fgr'] = pose[None]
            pose, _ = icp_refine(batch['src_xyz'], batch['tgt_xyz'], pose, icp_radius, icp=icp,
                                 estimate_normals=estimate_normals, **(icp_kwargs or {}))
            pose = torch.as_tensor(pose, dtype=torch.float64, device=coarse.device).reshape(coarse.shape)
        out['pose'] = pose[None]
        return out
    return run


def fpfh_downsample(clouds, voxel: float):
    """`ops.grid_subsample(dense=False)` of C clouds at `voxel` in one call: the mean of every occupied voxel of a grid
    anchored at the origin (Open3D's voxel_down_sample anchors its grid at the bounding box's minimum corner).
    -> list of C (m,3) float32 device tensors."""
    from . import ops
    dev = torch.device('cuda', torch.cuda.current_device())
    ts = [torch.as_tensor(c).to(dev, torch.float32) for c in clouds]
    xyz = torch.cat(ts, 0).contiguous()
    status = ops.new_status(dev)
    out, offs = ops.grid_subsample(xyz, ops.make_offsets([t.shape[0] for t in ts], dev), len(ts), voxel, status,
                                   dense=False)
    word = int(status.item())
    if word:
        raise RuntimeError(f'fpfh: grid sub-sampling at {voxel} failed (status {word:#x})')
    o = offs.tolist()
    return [out[o[k]:o[k + 1]] for k in range(len(ts))]


def fpfh_register(src_list, tgt_list, voxel: float, normal_radius: float = None, normal_max_nn: int = 30,
                  fpfh_radius: float = None, fpfh_max_nn: int = 100, mutual_filter: bool = True,
                  ransac_radius: float = None, max_iteration: int = 100000, confidence: float = 0.999,
                  ransac_n: int = 3, edge_length: float = 0.9, distance: float = None, seed: int = 0,
                  pair_base: int = 0, icp_radius: float = None, icp_kwargs=None, method: str = 'ransac',
                  fgr_kwargs=None) -> Dict:
    """Classical global registration of B pairs without a network, Open3D's tutorial pipeline on the device:
    `fpfh_downsample` at voxel V, `ops.estimate_normals` (normal_radius, default 2 V, normal_max_nn), `ops.fpfh`
    (fpfh_radius, default 5 V, fpfh_max_nn), then `ops.ransac_feature_matching` at ransac_radius (default 1.5 V) with the
    distance checker at `distance` (default: ransac_radius; 0: off), validated on the downsampled clouds.
    method='fgr' replaces RANSAC by `ops.fgr_feature_matching` on the downsampled clouds with fgr_kwargs (its options;
    maximum_correspondence_distance defaults to 0.5 V as in Open3D's tutorial) and needs mutual_filter; the RANSAC
    arguments are then unused.  With icp_radius, `icp_refine` (icp_kwargs) then starts from the global poses on the
    full clouds.
    -> dict: pose (B,3,4) float64 (the final poses), pose_fpfh (B,3,4) the RANSAC (or FGR) poses, ransac (B,5) (or
    fgr (B,4)), n_mutual (B,), src_down / tgt_down (B downsampled clouds), and icp (B,4) with icp_radius (and
    icp_levels (B,L,4) with voxels in icp_kwargs); device tensors."""
    from . import ops
    if method not in ('ransac', 'fgr'):
        raise ValueError(f'fpfh_register: unknown method {method!r}')
    if method == 'fgr' and not mutual_filter:
        raise ValueError('fpfh_register: FGR keeps the mutual matches only (mutual_filter=False is not supported)')
    B = len(src_list)
    down = fpfh_downsample(list(src_list) + list(tgt_list), voxel)
    normals = ops.estimate_normals(down, 2.0 * voxel if normal_radius is None else normal_radius, normal_max_nn)
    feats = ops.fpfh(down, normals, 5.0 * voxel if fpfh_radius is None else fpfh_radius, fpfh_max_nn)
    if method == 'fgr':
        kw = dict(fgr_kwargs or {})
        kw.setdefault('maximum_correspondence_distance', 0.5 * voxel)
        pose, res, n_mutual = ops.fgr_feature_matching(down[:B], down[B:], feats[:B], feats[B:], pair_base=pair_base,
                                                       **kw)
        out = dict(pose=pose, pose_fpfh=pose, fgr=res, n_mutual=n_mutual, src_down=down[:B], tgt_down=down[B:])
        _fpfh_icp(out, src_list, tgt_list, icp_radius, icp_kwargs)
        return out
    r = 1.5 * voxel if ransac_radius is None else ransac_radius
    pose, res, n_mutual = ops.ransac_feature_matching(
        down[:B], down[B:], feats[:B], feats[B:], mutual_filter, r, ransac_n, max_iteration=max_iteration,
        confidence=confidence, edge_length=edge_length, distance=r if distance is None else distance, seed=seed,
        pair_base=pair_base)
    out = dict(pose=pose, pose_fpfh=pose, ransac=res, n_mutual=n_mutual, src_down=down[:B], tgt_down=down[B:])
    _fpfh_icp(out, src_list, tgt_list, icp_radius, icp_kwargs)
    return out


def _fpfh_icp(out, src_list, tgt_list, icp_radius, icp_kwargs):
    """`fpfh_register`'s ICP from out['pose'] (with icp_radius): sets pose and icp, and icp_levels (B,L,4) when
    icp_kwargs has voxels."""
    if icp_radius is None:
        return
    kw = dict(icp_kwargs or {})
    levels = kw.get('voxels') is not None
    out['pose'], out['icp'], *lv = icp_refine(src_list, tgt_list, out['pose'], icp_radius, return_levels=levels, **kw)
    if levels:
        out['icp_levels'] = lv[0]


def fpfh_forward(voxel: float, icp_radius: float = None, icp_kwargs=None, **fpfh_kwargs):
    """A network-free `forward_fn(batch) -> pred` for `run_3dmatch_benchmark`: `fpfh_register` of the batch's full
    clouds (voxel, fpfh_kwargs (method='fgr' and fgr_kwargs included), and ICP after it with icp_radius / icp_kwargs)
    -> dict with pose (1,B,3,4) float64, and pose_fpfh (1,B,3,4) (the RANSAC or FGR poses) when ICP follows."""
    def run(batch):
        res = fpfh_register(batch['src_xyz'], batch['tgt_xyz'], voxel, icp_radius=icp_radius, icp_kwargs=icp_kwargs,
                            **fpfh_kwargs)
        out = {'pose': torch.as_tensor(res['pose'], dtype=torch.float64)[None]}
        if icp_radius is not None:
            out['pose_fpfh'] = res['pose_fpfh'][None]
        return out
    return run


def add_fpfh_arguments(ap):
    """The FPFH flags of a command line, for `fpfh_register`: --fpfh V, --fpfh_radius, --fpfh_max_nn and
    --fpfh_no_mutual."""
    ap.add_argument('--fpfh', type=float, metavar='V',
                    help='Register without a network: FPFH features of the clouds downsampled at voxel V, matched in '
                         'feature space, then RANSAC, or FGR with --fgr (Open3D\'s global registration); no --ckpt')
    ap.add_argument('--fpfh_radius', type=float, metavar='FR', help='FPFH feature radius (default: 5 V)')
    ap.add_argument('--fpfh_max_nn', type=int, default=100, help='Neighbours at most of the FPFH feature, 1..128')
    ap.add_argument('--fpfh_no_mutual', action='store_true',
                    help='Use every forward feature match, not only the mutual ones')


def check_fpfh_arguments(ap, opt):
    """With --fpfh: reject --ckpt and bad FPFH values as usage errors, and fill in the defaults that depend on V
    (--fpfh_radius 5 V, --ransac 1.5 V, --ransac_dist the --ransac radius; with --fgr, --ransac stays unset).
    Without it, --ckpt is required.  Call before `check_ransac_arguments`."""
    from .ops import FPFH_MAX_NN
    if opt.fpfh is None:
        if opt.ckpt is None:
            ap.error('the following arguments are required: --ckpt')
        return
    if opt.ckpt is not None:
        ap.error('--fpfh registers without a network: --ckpt is not allowed')
    if not opt.fpfh > 0.0:
        ap.error(f'--fpfh {opt.fpfh} must be > 0')
    if not 1 <= opt.fpfh_max_nn <= FPFH_MAX_NN:
        ap.error(f'--fpfh_max_nn {opt.fpfh_max_nn} must be in 1..{FPFH_MAX_NN}')
    if opt.fpfh_radius is None:
        opt.fpfh_radius = 5.0 * opt.fpfh
    if not opt.fpfh_radius > 0.0:
        ap.error(f'--fpfh_radius {opt.fpfh_radius} must be > 0')
    if getattr(opt, 'fgr', False):
        return
    if opt.ransac is None:
        opt.ransac = 1.5 * opt.fpfh
    if opt.ransac_dist is None:
        opt.ransac_dist = opt.ransac


def fpfh_kwargs(opt) -> Dict:
    """`fpfh_register`'s keyword arguments from the parsed --fpfh_* / --ransac_* flags (without V and ICP, and without
    --ransac_overlap, which has no meaning without a network; the normals are always estimated at 2 V, 30, and
    --normal_* stays ICP's).  With --fgr: the features, method='fgr' and fgr_kwargs from the --fgr_* flags."""
    if getattr(opt, 'fgr', False):
        return dict(fpfh_radius=opt.fpfh_radius, fpfh_max_nn=opt.fpfh_max_nn, method='fgr', fgr_kwargs=fgr_kwargs(opt))
    return dict(fpfh_radius=opt.fpfh_radius,
                fpfh_max_nn=opt.fpfh_max_nn, mutual_filter=not opt.fpfh_no_mutual, ransac_radius=opt.ransac,
                max_iteration=opt.ransac_iters, confidence=opt.ransac_confidence, ransac_n=opt.ransac_n,
                edge_length=opt.ransac_edge, distance=opt.ransac_dist, seed=opt.ransac_seed)


def icp_kwargs(opt) -> Dict:
    """`icp_refine`'s keyword arguments from the parsed --icp_* / --normal_* flags (without the radius); voxels, radii
    and level_iters only with --icp_voxels."""
    kw = dict(max_iteration=opt.icp_iters, method=opt.icp_method, normal_radius=opt.normal_radius,
              normal_max_nn=opt.normal_max_nn, epsilon=opt.icp_epsilon, loss=opt.icp_loss, loss_k=opt.icp_loss_k)
    if opt.icp_method == 'colored':
        kw['lambda_geometric'] = opt.icp_lambda_geometric
    if opt.icp_voxels is not None:
        kw.update(voxels=opt.icp_voxels, radii=opt.icp_radii, level_iters=opt.icp_level_iters)
    return kw


def run_3dmatch_benchmark(batches: Iterable[Dict], forward_fn, log_path: str, benchmark: str, gt_folder: str,
                          thresh_rot=10.0, thresh_trans=0.1):
    """`Trainer.test` + `GenericRegModel.test_step/test_epoch_end` for the 3DMatch benchmarks
    (trainer.py:195-207, generic_reg_model.py:130-175): run `forward_fn(batch) -> pred` over collated batches
    (regtr_b200.data.PairStream), append every final pose to est.log, aggregate the pose errors against
    `batch['pose']`, then score the logs with the registration-recall benchmark.
    -> dict(summary=str, recall=float, metrics={...}, per_scene={...})."""
    writer = EstLogWriter(log_path, benchmark)
    per_batch = []
    for batch in batches:
        pred = forward_fn(batch)
        writer.append_batch(batch, pred)
        gt = batch['pose'].to(pred['pose'].device, pred['pose'].dtype)
        per_batch.append({k: v.detach().cpu() for k, v in compute_metrics(pred, gt).items()})
    summary, recall, per_scene = benchmark_3dmatch(writer.root, gt_folder)
    return dict(summary=summary, recall=recall, per_scene=per_scene,
                metrics=aggregate_metrics(per_batch, thresh_rot, thresh_trans))
