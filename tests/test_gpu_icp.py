"""Point-to-point ICP on the device (`ops.icp`, regtr_icp) against the float64 oracle (tests/icp_oracle.py) on the real
3DMatch fixtures and on synthetic 3DMatch-shaped pairs: final pose, iteration count, correspondences and RMSE, the
state after 0..3 iterations, batching, reruns, the launch count, agreement with `ops.registration_fit`, the range
check, and `python -m regtr_b200.register --icp` end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import icp_oracle as I
import train_data_oracle as O
from conftest import GOLDEN, ROOT
from regtr_b200 import lib, ops
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from regtr_b200.synthetic import make_3dmatch_pair
from test_gpu_register import gt_log_pair

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')
RADIUS = 0.0375
K_DIFF = []                    # |k_device - k_oracle| seen, reported by test_report_largest_k_difference


def perturb(pose, seed, deg=3.0, metres=0.03):
    rng = np.random.default_rng(seed)
    axis = rng.normal(size=3)
    d = np.eye(3, 4)
    d[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
    d[:, 3] = rng.normal(size=3) * metres / np.sqrt(3.0)
    return I.compose(d, np.asarray(pose, np.float64))


def real_pairs():
    """(src, tgt, init) of the three real fixtures; the two with a benchmark gt.log pose start from it perturbed,
    the third (no ground truth in the fixtures) from the identity."""
    out = []
    for i, (fx, scene) in enumerate((('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
                                     ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3'))):
        s, t, p = gt_log_pair(fx, scene)
        out.append((s, t, perturb(p, 100 + i)))
    inp = np.load(os.path.join(REAL, 'real_3dmatch_sun3d_home_38_41_input.npz'))
    out.append((inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64), np.eye(3, 4)))
    return out


def synthetic_pairs(seeds=(4001, 4002)):
    out = []
    for s in seeds:
        p = make_3dmatch_pair(s)
        out.append((p['src_xyz'].astype(np.float64), p['tgt_xyz'].astype(np.float64), perturb(p['pose'], s)))
    return out


def device_icp(pairs, max_iteration=30, **kw):
    pose, res = ops.icp([s for s, _, _ in pairs], [t for _, t, _ in pairs],
                        torch.from_numpy(np.stack([p for _, _, p in pairs])).cuda(), RADIUS, max_iteration, **kw)
    return pose, res


def check_against_oracle(pose, res, pairs, max_iteration=30):
    pose, res = pose.cpu().numpy(), res.cpu().numpy()
    for b, (s, t, p) in enumerate(pairs):
        o = I.icp(s, t, p, RADIUS, max_iteration)
        rot_err = np.linalg.norm(pose[b, :, :3] - o['pose'][:, :3])
        trans_err = np.linalg.norm(pose[b, :, 3] - o['pose'][:, 3])
        assert rot_err <= 1e-9 and trans_err <= 1e-9, (b, rot_err, trans_err)
        assert int(res[b, 3]) == o['iterations'], (b, res[b], o['iterations'])
        K_DIFF.append(abs(int(res[b, 2]) - o['k']))
        assert abs(int(res[b, 2]) - o['k']) <= 2, (b, res[b, 2], o['k'])
        assert abs(res[b, 1] - o['rmse']) <= 1e-12 * o['rmse'], (b, res[b, 1], o['rmse'])
        assert res[b, 0] == res[b, 2] / len(s)
    return res


def test_real_pairs_against_the_oracle():
    pairs = real_pairs()
    pose, res = device_icp(pairs)
    assert pose.shape == (3, 3, 4) and pose.dtype == torch.float64 and res.shape == (3, 4)
    r = check_against_oracle(pose, res, pairs)
    assert (r[:2, 0] > 0.2).all()                           # the ground-truth pairs overlap


def test_synthetic_pairs_against_the_oracle():
    pairs = synthetic_pairs()
    pose, res = device_icp(pairs)
    check_against_oracle(pose, res, pairs)


def test_state_after_each_of_the_first_iterations():
    pairs = real_pairs()[:1] + synthetic_pairs((4003,))
    for it in range(4):
        pose, res = device_icp(pairs, it)
        r = check_against_oracle(pose, res, pairs, it)
        assert (r[:, 3] == it).all()
        if it == 0:
            assert np.array_equal(pose.cpu().numpy(), np.stack([p for _, _, p in pairs]))


def test_batch_equals_one_call_per_pair_and_reruns_are_identical():
    real = real_pairs()
    syn = synthetic_pairs((4004,))[0]
    far = (syn[0][:3000], syn[1][:5000] + 40.0, syn[2])              # no correspondences at all
    pairs = [real[0], far, (real[1][0][:7001], real[1][1], real[1][2]), syn]
    pose, res = device_icp(pairs)
    again = device_icp(pairs)
    assert torch.equal(pose, again[0]) and torch.equal(res, again[1])
    for b, pr in enumerate(pairs):
        p1, r1 = device_icp([pr])
        assert torch.equal(p1[0], pose[b]) and torch.equal(r1[0], res[b]), b
    r = res.cpu().numpy()
    assert r[1].tolist() == [0.0, 0.0, 0.0, 1.0]
    assert np.array_equal(pose[1].cpu().numpy(), far[2])


def test_launch_count_does_not_depend_on_batch_or_convergence():
    syn = synthetic_pairs((4005,))
    counts = []
    loose = dict(relative_fitness=1e-2, relative_rmse=1e-2)                  # converges within a few iterations
    never = dict(relative_fitness=0.0, relative_rmse=0.0)                    # |d| < 0 never holds
    for pairs, kw, done_early in (([syn[0]], loose, True), ([syn[0]] * 8, loose, True), ([syn[0]], never, False),
                                  ([syn[0]] * 8, never, False)):
        before = ops.LAUNCHES
        _, res = device_icp(pairs, 30, **kw)
        torch.cuda.synchronize()
        counts.append(ops.LAUNCHES - before)
        iters = res[:, 3].cpu().numpy()
        assert (iters < 30).all() if done_early else (iters == 30).all(), iters
    assert counts == [ops.icp_launches(30)] * 4, counts


def test_final_fitness_agrees_with_the_registration_fit():
    pairs = real_pairs()[:2] + synthetic_pairs((4006,))
    pose, res = device_icp(pairs)
    fit = ops.registration_fit([s for s, _, _ in pairs], [t for _, t, _ in pairs], pose, RADIUS).cpu().numpy()
    r = res.cpu().numpy()
    for b, (s, _, _) in enumerate(pairs):
        k_fit = round(fit[b, 0] * len(s))
        k = int(r[b, 2])
        K_DIFF.append(abs(k_fit - k))
        assert abs(k_fit - k) <= 2, (b, k_fit, k)
        # a correspondence flipping at the radius moves the RMSE by at most ~ (r^2 / rmse^2) / k relative
        tol = 1e-9 if k_fit == k else 3.0 * (RADIUS / r[b, 1]) ** 2 / k
        assert abs(fit[b, 1] - r[b, 1]) <= tol * r[b, 1], (b, fit[b], r[b])


def test_coordinate_beyond_the_bound_raises():
    bound = ops.overlap_coord_bound(RADIUS)
    src = np.array([[0.0, 0.0, 0.0], [bound * 1.001, 0.0, 0.0]])
    tgt = np.array([[0.01, 0.0, 0.0]])
    eye = torch.from_numpy(np.eye(3, 4)[None])
    with pytest.raises(lib.RegtrLibError, match='icp: a coordinate'):
        ops.icp([src], [tgt], eye, RADIUS)
    with pytest.raises(lib.RegtrLibError, match='overlap_coord_bound'):
        ops.icp([tgt], [src], eye, RADIUS)                          # a target coordinate
    far = np.eye(3, 4)
    far[0, 3] = bound * 1.001
    with pytest.raises(lib.RegtrLibError):
        ops.icp([tgt], [tgt], torch.from_numpy(far[None]), RADIUS)  # the moved source counts, not the raw one
    status = ops.new_status(torch.device('cuda'))
    ops.icp([src], [tgt], eye, RADIUS, status=status)               # the caller's word: raised where it is read
    with pytest.raises(lib.RegtrLibError):
        ops.check_fit_status(status, RADIUS, 'icp')
    ok, _ = ops.icp([src[:1]], [tgt], eye, RADIUS)
    assert torch.isfinite(ok).all()


def test_report_largest_k_difference():
    print(f'largest |k_device - k_oracle| (and vs. the fit): {max(K_DIFF) if K_DIFF else "n/a"}')
    assert not K_DIFF or max(K_DIFF) <= 2


def _run_register(tmp_path, run, src_file, tgt_file, out_dir, extra):
    env = dict(os.environ, PYTHONNOUSERSITE='1')
    r = subprocess.run([sys.executable, '-m', 'regtr_b200.register', src_file, tgt_file,
                        '--ckpt', str(run / 'ckpt' / 'model-best.pth'), '--out', str(out_dir)] + extra,
                       capture_output=True, text=True, cwd=ROOT, env=env, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_register_cli_with_icp(tmp_path):
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('modelnet')
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, 43), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, 'modelnet', str(run / 'config.yaml'))
    src_file = os.path.join(REAL, 'modelnet_test_2_0.ply')
    tgt_file = os.path.join(REAL, 'modelnet_test_2_1.ply')
    s, t = P.load_point_cloud(src_file), P.load_point_cloud(tgt_file)
    plain = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'plain', [])
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'icp', ['--icp', str(RADIUS)])

    # without --icp: the files and the line of the plain registration
    res0 = np.load(str(tmp_path / 'plain' / 'result.npz'))
    assert sorted(res0.files) == sorted(['pose', 'src_kp', 'src_kp_warped', 'src_overlap', 'tgt_kp', 'tgt_kp_warped',
                                         'tgt_overlap', 'fit'])
    coarse = res0['pose'][-1]
    assert open(tmp_path / 'plain' / 'pose.txt').read() == R.pose_text(coarse)
    assert not any(k.startswith('icp') for k in plain)

    res = np.load(str(tmp_path / 'icp' / 'result.npz'))
    assert np.array_equal(res['pose'], res0['pose']) and np.array_equal(res['pose_coarse'], coarse)
    pose, out = ops.icp([s], [t], torch.from_numpy(coarse[None]).cuda(), RADIUS, 30)
    pose, out = pose[0].cpu().numpy(), out[0].cpu().numpy()
    assert np.array_equal(res['pose_icp'], pose) and np.array_equal(res['icp'], out)
    assert open(tmp_path / 'icp' / 'pose.txt').read() == R.pose_text(pose)
    assert np.array_equal(np.array(line['pose']), R.pose44(pose))
    assert (line['icp_fitness'], line['icp_rmse'], line['icp_iterations'], line['icp_radius']) == \
        (float(out[0]), float(out[1]), int(out[3]), RADIUS)
    fit = ops.registration_fit([s], [t], torch.from_numpy(pose[None]).cuda(), cfg.overlap_radius).cpu().numpy()[0]
    assert np.array_equal(res['fit'], fit)
    np.testing.assert_allclose(P.load_point_cloud(str(tmp_path / 'icp' / 'src_registered.ply')),
                               s @ pose[:, :3].T + pose[:, 3], rtol=0, atol=1e-6)

