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
        gt = batch['pose'].to(pred['pose'].device)
        per_batch.append({k: v.detach().cpu() for k, v in compute_metrics(pred, gt).items()})
    summary, recall, per_scene = benchmark_3dmatch(writer.root, gt_folder)
    return dict(summary=summary, recall=recall, per_scene=per_scene,
                metrics=aggregate_metrics(per_batch, thresh_rot, thresh_trans))
