"""Normal estimation (`ops.estimate_normals`, regtr_estimate_normals) and point-to-plane ICP (`ops.icp` with
method='point_to_plane') on the device against the float64 oracle (tests/icp_plane_oracle.py) on the real 3DMatch and
ModelNet fixtures and on synthetic 3DMatch-shaped pairs: neighbour counts, normal directions and signs, the final pose,
iteration count, correspondences and RMSE, the state after 0..3 iterations, batching, reruns, the launch count, the
errors, and `python -m regtr_b200.register --icp R --icp_method point_to_plane` end to end."""
import os

import numpy as np
import pytest
import torch

import icp_plane_oracle as N
from conftest import GOLDEN
from regtr_b200 import lib, ops
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from test_gpu_icp import RADIUS, _run_register, real_pairs, synthetic_pairs

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')
NR = 2.0 * RADIUS              # the normal radius register uses by default
K_DIFF = []                    # |k_device - k_oracle| seen, reported by test_report_largest_k_difference
RATIO = []                     # worst sin(theta) / (lambda_max / (lambda_mid - lambda_min)) per cloud


def real_clouds():
    """(clouds, radius) sets: the three real 3DMatch inputs at NR, the ModelNet .ply pair at 0.1."""
    c3 = []
    for fx in ('real_3dmatch_redkitchen_0_5', 'real_3dmatch_sun3d_hotel3_8_15', 'real_3dmatch_sun3d_home_38_41'):
        inp = np.load(os.path.join(REAL, fx + '_input.npz'))
        c3 += [inp['src_xyz'].astype(np.float64), inp['tgt_xyz'].astype(np.float64)]
    mn = [P.load_point_cloud(os.path.join(REAL, f'modelnet_test_2_{i}.ply')).astype(np.float64) for i in (0, 1)]
    return [(c3, NR), (mn, 0.1)]


def check_normals(dev_n, dev_c, xyz, r, max_nn=30):
    want, cnt, lam = N.estimate_normals(xyz, r, max_nn, return_eigvals=True)
    assert np.array_equal(dev_c, cnt)
    zero = cnt < 3
    assert not dev_n[zero].any()
    assert np.abs(np.linalg.norm(dev_n[~zero], axis=1) - 1.0).max() <= 1e-15
    s = (dev_n[:, 0] * xyz[:, 0] + dev_n[:, 1] * xyz[:, 1]) + dev_n[:, 2] * xyz[:, 2]
    assert (s <= 0.0).all()
    sin = np.linalg.norm(np.cross(dev_n[~zero], want[~zero]), axis=1)
    lam = lam[~zero]
    gap = lam[:, 1] - lam[:, 0]
    ok = gap > 0
    scale = lam[ok, 2] / gap[ok]
    ratio = sin[ok] / scale
    RATIO.append(float(ratio.max()) if ratio.size else 0.0)
    worst = int(np.argmax(ratio)) if ratio.size else 0
    assert (ratio <= 1e-12).all(), (ratio.max(), sin[ok][worst], scale[worst])
    return zero.mean()


def test_normals_against_the_oracle():
    for clouds, r in real_clouds():
        out, cnt = ops.estimate_normals(clouds, r, 30, return_counts=True)
        assert len(out) == len(clouds)
        for c, n, k in zip(clouds, out, cnt):
            assert n.shape == c.shape and n.dtype == torch.float64 and k.dtype == torch.int32
            check_normals(n.cpu().numpy(), k.cpu().numpy(), c, r)
    print(f'worst sin(theta) / (lambda_max / (lambda_mid - lambda_min)) per cloud: '
          f'{", ".join(f"{v:.2e}" for v in RATIO)}')


def test_normals_other_max_nn_and_stacking():
    (c3, r), (mn, _) = real_clouds()
    clouds = [c3[0], mn[1], c3[3][:5001], mn[0]]
    radii = r
    for max_nn in (1, 3, 17, 64):
        out, cnt = ops.estimate_normals(clouds, radii, max_nn, return_counts=True)
        again = ops.estimate_normals(clouds, radii, max_nn)
        for b, c in enumerate(clouds):
            assert torch.equal(again[b], out[b])
            alone, ca = ops.estimate_normals([c], radii, max_nn, return_counts=True)
            assert torch.equal(alone[0], out[b]) and torch.equal(ca[0], cnt[b]), (max_nn, b)
            if max_nn in (3, 64) and b < 2:
                check_normals(out[b].cpu().numpy(), cnt[b].cpu().numpy(), c, radii, max_nn)
        if max_nn < 3:
            assert all(not o.any() for o in out)


def plane_pairs(pairs, max_nn=30):
    normals = ops.estimate_normals([t for _, t, _ in pairs], NR, max_nn)
    return [(s, t, p, n.cpu().numpy()) for (s, t, p), n in zip(pairs, normals)], normals


def device_plane_icp(pairs4, max_iteration=30, **kw):
    return ops.icp([s for s, _, _, _ in pairs4], [t for _, t, _, _ in pairs4],
                   torch.from_numpy(np.stack([p for _, _, p, _ in pairs4])).cuda(), RADIUS, max_iteration,
                   method='point_to_plane', tgt_normals=[n for _, _, _, n in pairs4], **kw)


def check_against_oracle(pose, res, pairs4, max_iteration=30):
    pose, res = pose.cpu().numpy(), res.cpu().numpy()
    for b, (s, t, p, n) in enumerate(pairs4):
        o = N.icp(s, t, n, p, RADIUS, max_iteration)
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
    pairs4, _ = plane_pairs(real_pairs())
    pose, res = device_plane_icp(pairs4)
    assert pose.shape == (3, 3, 4) and pose.dtype == torch.float64 and res.shape == (3, 4)
    r = check_against_oracle(pose, res, pairs4)
    assert (r[:2, 0] > 0.2).all()
    print(f'point-to-plane iterations (real pairs): {r[:, 3].astype(int).tolist()}')


def test_synthetic_pairs_against_the_oracle():
    pairs4, _ = plane_pairs(synthetic_pairs())
    pose, res = device_plane_icp(pairs4)
    r = check_against_oracle(pose, res, pairs4)
    print(f'point-to-plane iterations (synthetic pairs): {r[:, 3].astype(int).tolist()}')


def test_state_after_each_of_the_first_iterations():
    pairs4, _ = plane_pairs(real_pairs()[:1] + synthetic_pairs((4003,)))
    for it in range(4):
        pose, res = device_plane_icp(pairs4, it)
        r = check_against_oracle(pose, res, pairs4, it)
        assert (r[:, 3] == it).all()
        if it == 0:
            assert np.array_equal(pose.cpu().numpy(), np.stack([p for _, _, p, _ in pairs4]))


def test_batch_equals_one_call_per_pair_and_reruns_are_identical():
    real = real_pairs()
    syn = synthetic_pairs((4004,))[0]
    far = (syn[0][:3000], syn[1][:5000] + 40.0, syn[2])              # no correspondences at all
    pairs4, _ = plane_pairs([real[0], far, (real[1][0][:7001], real[1][1], real[1][2]), syn])
    pose, res = device_plane_icp(pairs4)
    again = device_plane_icp(pairs4)
    assert torch.equal(pose, again[0]) and torch.equal(res, again[1])
    for b, pr in enumerate(pairs4):
        p1, r1 = device_plane_icp([pr])
        assert torch.equal(p1[0], pose[b]) and torch.equal(r1[0], res[b]), b
    r = res.cpu().numpy()
    assert r[1].tolist() == [0.0, 0.0, 0.0, 1.0]
    assert np.array_equal(pose[1].cpu().numpy(), far[2])


def test_launch_count_and_the_default_method():
    syn = synthetic_pairs((4005,))
    pairs4, normals = plane_pairs(syn)
    before = ops.LAUNCHES
    ops.estimate_normals([syn[0][1]] * 5, NR)
    assert ops.LAUNCHES - before == ops.normals_launches()
    counts = []
    loose = dict(relative_fitness=1e-2, relative_rmse=1e-2)
    never = dict(relative_fitness=0.0, relative_rmse=0.0)
    for batch, kw, done_early in ((pairs4, loose, True), (pairs4 * 8, loose, True), (pairs4, never, False),
                                  (pairs4 * 8, never, False)):
        before = ops.LAUNCHES
        _, res = device_plane_icp(batch, 30, **kw)
        torch.cuda.synchronize()
        counts.append(ops.LAUNCHES - before)
        iters = res[:, 3].cpu().numpy()
        assert (iters < 30).all() if done_early else (iters == 30).all(), iters
    assert counts == [ops.icp_launches(30)] * 4, counts
    s, t, p = syn[0]
    init = torch.from_numpy(p[None]).cuda()
    a = ops.icp([s], [t], init, RADIUS)
    b = ops.icp([s], [t], init, RADIUS, method='point_to_point', tgt_normals=None)
    c = ops.icp([s], [t], init, RADIUS, method='point_to_point', tgt_normals=normals)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and all(torch.equal(x, y) for x, y in zip(a, c))
    d = ops.icp([s], [t], init, RADIUS, method='point_to_plane', tgt_normals=normals)
    assert not torch.equal(a[0], d[0])


def test_errors():
    bound = ops.overlap_coord_bound(NR)
    cloud = np.array([[0.0, 0.0, 0.0], [0.01, 0.0, 0.0], [0.0, 0.01, 0.0], [bound * 1.001, 0.0, 0.0]])
    with pytest.raises(lib.RegtrLibError, match='estimate_normals: a coordinate'):
        ops.estimate_normals([cloud[:3], cloud], NR)
    nan = cloud[:3].copy()
    nan[1, 2] = np.nan
    with pytest.raises(lib.RegtrLibError):
        ops.estimate_normals([nan], NR)
    ok = ops.estimate_normals([cloud[:3]], NR)[0].cpu().numpy()
    assert np.array_equal(np.abs(ok), np.tile([0.0, 0.0, 1.0], (3, 1)))       # the plane z = 0
    rb = ops.overlap_coord_bound(RADIUS)
    src = np.array([[0.0, 0.0, 0.0], [rb * 1.001, 0.0, 0.0]])
    tgt = np.array([[0.01, 0.0, 0.0]])
    eye = torch.from_numpy(np.eye(3, 4)[None])
    nrm = [np.array([[0.0, 0.0, 1.0]])]
    with pytest.raises(lib.RegtrLibError, match='icp: a coordinate'):
        ops.icp([src], [tgt], eye, RADIUS, method='point_to_plane', tgt_normals=nrm)
    with pytest.raises(lib.RegtrLibError, match='overlap_coord_bound'):
        ops.icp([tgt], [src], eye, RADIUS, method='point_to_plane', tgt_normals=[np.zeros((2, 3))])
    with pytest.raises(ValueError, match='target normals'):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='point_to_plane')
    with pytest.raises(ValueError):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='point_to_plane', tgt_normals=[np.zeros((2, 3))])
    with pytest.raises(ValueError):
        ops.icp([src[:1]], [tgt], eye, RADIUS, method='plane')
    with pytest.raises(ValueError):
        ops.estimate_normals([cloud[:3]], NR, max_nn=65)
    pose, _ = ops.icp([src[:1]], [tgt], eye, RADIUS, method='point_to_plane', tgt_normals=nrm)
    assert torch.isfinite(pose).all()


def test_report_largest_k_difference():
    print(f'largest |k_device - k_oracle|: {max(K_DIFF) if K_DIFF else "n/a"}')
    assert not K_DIFF or max(K_DIFF) <= 2


def test_register_cli_with_point_to_plane_icp(tmp_path):
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
    radius = 0.05
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'plane',
                         ['--icp', str(radius), '--icp_method', 'point_to_plane'])
    res = np.load(str(tmp_path / 'plane' / 'result.npz'))
    coarse = res['pose'][-1]
    assert np.array_equal(res['pose_coarse'], coarse)
    normals = ops.estimate_normals([t], 2.0 * radius, 30)
    pose, out = ops.icp([s], [t], torch.from_numpy(coarse[None]).cuda(), radius, 30, method='point_to_plane',
                        tgt_normals=normals)
    pose, out = pose[0].cpu().numpy(), out[0].cpu().numpy()
    assert np.array_equal(res['pose_icp'], pose) and np.array_equal(res['icp'], out)
    assert open(tmp_path / 'plane' / 'pose.txt').read() == R.pose_text(pose)
    assert np.array_equal(np.array(line['pose']), R.pose44(pose))
    assert (line['icp_fitness'], line['icp_rmse'], line['icp_iterations'], line['icp_radius'], line['icp_method']) == \
        (float(out[0]), float(out[1]), int(out[3]), radius, 'point_to_plane')
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'plane_nr',
                         ['--icp', str(radius), '--icp_method', 'point_to_plane', '--normal_radius', '0.08',
                          '--normal_max_nn', '12'])
    normals = ops.estimate_normals([t], 0.08, 12)
    pose, out = ops.icp([s], [t], torch.from_numpy(coarse[None]).cuda(), radius, 30, method='point_to_plane',
                        tgt_normals=normals)
    assert np.array_equal(np.load(str(tmp_path / 'plane_nr' / 'result.npz'))['pose_icp'], pose[0].cpu().numpy())
