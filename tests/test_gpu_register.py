"""Registration of two point-cloud files on the device: `ops.registration_fit` (regtr_registration_fit on the
matches of regtr_overlap_nn) against a float64 restatement on cKDTree, on the real 3DMatch and ModelNet clouds,
and `python -m regtr_b200.register` end to end against a direct forward."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import train_data_oracle as O
from conftest import GOLDEN, ROOT
from regtr_b200 import data as D
from regtr_b200 import eval as E
from regtr_b200 import lib, ops
from regtr_b200 import pointio as P
from regtr_b200 import register as R

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')


def gt_log_pair(fixture, scene):
    """(src, tgt, pose (3,4)) of a real 3DMatch pair with the benchmark's gt.log pose: the pose of entry (i, j)
    maps cloud_bin_j onto cloud_bin_i, so cloud_bin_j is the source."""
    keys, traj = E.read_trajectory(os.path.join(REAL, 'benchmarks', '3DMatch', scene, 'gt.log'))
    inp = np.load(os.path.join(REAL, fixture + '_input.npz'))
    src_is_file_src = os.path.basename(str(inp['src_file'])) == f'cloud_bin_{int(keys[0][1])}.pth'
    a, b = inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)
    return (a, b, traj[0][:3]) if src_is_file_src else (b, a, traj[0][:3])


def modelnet_pair():
    s = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_0.ply'))
    t = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_1.ply'))
    pose = np.eye(3, 4)
    pose[:, :3] = O.axis_angle(np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8]), np.deg2rad(2.0))
    pose[:, 3] = [0.01, -0.005, 0.003]
    return s, t, pose


def oracle_fit(s, t, pose, r):
    """Float64 restatement: counts from data.compute_overlap on the source moved in the kernel's operation order,
    squared distances from cKDTree."""
    sa = O.align(s, pose)
    sm, tm, _ = D.compute_overlap(sa, t, r)
    out = []
    for q, ref, m in ((sa, t, sm), (t, sa, tm)):
        k = int(m.sum())
        if len(ref) and len(q):
            d, _ = cKDTree(ref).query(q, k=1, distance_upper_bound=r)
            ssum = float(np.sum(d[m] ** 2))
        else:
            ssum = 0.0
        out += [k / len(q) if len(q) else 0.0, np.sqrt(ssum / k) if k else 0.0, k]
    return out          # fitness_src, rmse_src, k_src, fitness_tgt, rmse_tgt, k_tgt


def check_against_oracle(fit, pairs, r):
    for b, (s, t, p) in enumerate(pairs):
        fs, rs, ks, ft, rt, kt = oracle_fit(s, t, p, r)
        assert ks > 0 and kt > 0, b
        assert round(fit[b, 0] * len(s)) == ks and fit[b, 0] == ks / len(s), b          # exact inlier counts
        assert round(fit[b, 2] * len(t)) == kt and fit[b, 2] == kt / len(t), b
        assert abs(fit[b, 1] - rs) <= 1e-12 * rs and abs(fit[b, 3] - rt) <= 1e-12 * rt, (b, fit[b], rs, rt)


def test_fit_on_the_real_3dmatch_pairs_batched():
    pairs = [gt_log_pair('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
             gt_log_pair('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3')]
    r = 0.0375
    pose = torch.from_numpy(np.stack([p for _, _, p in pairs])).cuda()
    fit = ops.registration_fit([s for s, _, _ in pairs], [t for _, t, _ in pairs], pose, r)
    again = ops.registration_fit([s for s, _, _ in pairs], [t for _, t, _ in pairs], pose, r)
    assert fit.shape == (2, 4) and fit.dtype == torch.float64 and fit.is_cuda
    assert torch.equal(fit, again)                                                     # bit-identical rerun
    f = fit.cpu().numpy()
    check_against_oracle(f, pairs, r)
    assert (f[:, [0, 2]] > 0.2).all() and (f[:, [1, 3]] < r).all()
    # the same pairs one at a time give the same bits
    for b, (s, t, p) in enumerate(pairs):
        one = ops.registration_fit([s], [t], torch.from_numpy(p[None]).cuda(), r)
        assert torch.equal(one[0], fit[b])


def test_fit_on_the_modelnet_pair_and_edge_cases():
    s, t, pose = modelnet_pair()
    fit = ops.registration_fit([s], [t], torch.from_numpy(pose[None]), 0.04).cpu().numpy()
    check_against_oracle(fit, [(s, t, pose)], 0.04)
    far = pose.copy()
    far[:, 3] += 50.0
    eye = np.eye(3, 4)
    fit = ops.registration_fit([s, s, np.zeros((0, 3))], [t, np.zeros((0, 3)), t],
                               torch.from_numpy(np.stack([far, eye, eye])), 0.04).cpu().numpy()
    assert np.array_equal(fit, np.zeros((3, 4)))                    # no inliers; empty clouds give 0, not nan


def test_fit_beyond_the_coordinate_bound_raises():
    r = 0.04
    bound = ops.overlap_coord_bound(r)
    src = np.array([[0.0, 0.0, 0.0], [bound * 1.001, 0.0, 0.0]])
    tgt = np.array([[0.01, 0.0, 0.0]])
    with pytest.raises(lib.RegtrLibError, match=re.escape(f'{bound:.3f}')):
        ops.registration_fit([src], [tgt], torch.from_numpy(np.eye(3, 4)[None]), r)
    # with the caller's status word nothing is raised until the caller checks it
    status = ops.new_status(torch.device('cuda'))
    ops.registration_fit([src], [tgt], torch.from_numpy(np.eye(3, 4)[None]), r, status)
    with pytest.raises(lib.RegtrLibError, match='overlap_coord_bound'):
        ops.check_fit_status(status, r)
    # the moved source counts, not the raw one
    pose = np.eye(3, 4)
    pose[0, 3] = bound * 1.001
    with pytest.raises(lib.RegtrLibError):
        ops.registration_fit([tgt], [tgt], torch.from_numpy(pose[None]), r)


def test_fit_flags_matches_that_the_overlap_search_cannot_produce():
    """nn indices outside the partner cloud are not counted (memory-safe) and raise REGTR_STATUS_INPUT."""
    L = lib.load()
    xyz = torch.tensor([[0.0, 0, 0], [0.01, 0, 0], [0.02, 0, 0]], dtype=torch.float64, device='cuda')
    offs = ops.make_offsets([2, 1], xyz.device)
    pose = torch.from_numpy(np.eye(3, 4)[None]).cuda()
    nn = torch.tensor([0, 7, 0], dtype=torch.int32, device='cuda')          # 7: no such target
    out = torch.full((1, 4), -1.0, dtype=torch.float64, device='cuda')
    status = ops.new_status(xyz.device)
    lib.check(L.regtr_registration_fit(xyz.data_ptr(), offs.data_ptr(), 1, 3, pose.data_ptr(), 0.04, nn.data_ptr(),
                                       out.data_ptr(), status.data_ptr(), ops._stream()), 'regtr_registration_fit')
    assert int(status.item()) & ops.STATUS_INPUT
    o = out.cpu().numpy()[0]
    d = np.sqrt(np.float64(0.02) * np.float64(0.02))
    assert o.tolist() == [0.5, d, 1.0, d]


def test_register_cli_end_to_end(tmp_path):
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('modelnet')
    sd = random_state_dict(cfg, 41)
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': sd, 'step': 123}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, 'modelnet', str(run / 'config.yaml'))
    src_file = os.path.join(REAL, 'modelnet_test_2_0.ply')
    s = P.load_point_cloud(src_file)
    t = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_1.ply'))
    torch.save(t, str(tmp_path / 'tgt.pth'))
    out_dir = tmp_path / 'out'
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.register', src_file, str(tmp_path / 'tgt.pth'),
                        '--ckpt', str(run / 'ckpt' / 'model-best.pth'), '--out', str(out_dir), '--threshold', '0.3'],
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])

    model = RegTR(cfg).cuda().eval()
    model.load_state_dict(sd, strict=True)
    pred = model({'src_xyz': [torch.from_numpy(s).float().cuda()], 'tgt_xyz': [torch.from_numpy(t).float().cuda()]})
    pose = pred['pose'][:, 0].cpu().numpy()
    res = np.load(str(out_dir / 'result.npz'))
    assert res['pose'].dtype == np.float32 and np.array_equal(res['pose'], pose)
    assert open(out_dir / 'pose.txt').read() == R.pose_text(pose[-1])
    assert np.array_equal(np.array(line['pose']), R.pose44(pose[-1]))
    p = pose[-1].astype(np.float64)
    np.testing.assert_allclose(P.load_point_cloud(str(out_dir / 'src_registered.ply')), s @ p[:, :3].T + p[:, 3],
                               rtol=0, atol=1e-6)
    fit = ops.registration_fit([s], [t], torch.from_numpy(pose[-1:]).cuda(), cfg.overlap_radius).cpu().numpy()[0]
    assert np.array_equal(res['fit'], fit)
    assert [line[k] for k in ('fitness_src', 'rmse_src', 'fitness_tgt', 'rmse_tgt')] == fit.tolist()
    assert line['n_src'] == len(s) and line['n_tgt'] == len(t)
    # keypoint panels: the keypoints with predicted overlap above the threshold
    ov = torch.sigmoid(pred['src_overlap'][0][-1][:, 0]).cpu().numpy()
    assert np.array_equal(res['src_overlap'], ov)
    m = ov > 0.3
    assert line['n_src_kp_above_threshold'] == int(m.sum())
    assert np.array_equal(P.load_point_cloud(str(out_dir / 'src_kp.ply')), pred['src_kp'][0].cpu().numpy()[m])
    assert np.array_equal(P.load_point_cloud(str(out_dir / 'src_kp_warped.ply')),
                          pred['src_kp_warped'][0][-1].cpu().numpy()[m])


def test_fit_kernel_does_not_spill(tmp_path):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c',
                                                    os.path.join(build.CSRC, 'traindata.cu'), '-o',
                                                    str(tmp_path / 'traindata.o')],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    block = text[text.index('k_registration_fit'):]
    stats = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', block)
    assert stats and stats.groups()[1:] == ('0', '0'), block[:400]
