"""Multiway registration on the host: the float64 pose-graph and information oracle (tests/posegraph_oracle.py) on its
own, the CLI of `python -m regtr_b200.multiway`, the est.log layout, and the new kernels' register budgets."""
import os
import re
import subprocess

import numpy as np
from scipy.spatial import cKDTree

import posegraph_oracle as PG
from regtr_b200 import eval as E
from regtr_b200 import multiway as M


def test_jacobians_match_central_differences():
    rng = np.random.default_rng(1)
    P = np.stack([PG.random_pose(rng, 60.0, 2.0) for _ in range(2)])
    X = PG.rinv(P[1]) @ P[0] @ PG.random_pose(rng, 5.0, 0.1)
    zeta, Js, Jt = PG.residual_and_jacobian(P, 0, 1, X)
    h = 1e-6
    for node, J in ((0, Js), (1, Jt)):
        for k in range(6):
            d = np.zeros(6)
            d[k] = h
            Pp, Pm = P.copy(), P.copy()
            Pp[node] = PG.rt_exp(d) @ P[node]
            Pm[node] = PG.rt_exp(-d) @ P[node]
            fd = (PG.residual_and_jacobian(Pp, 0, 1, X)[0] - PG.residual_and_jacobian(Pm, 0, 1, X)[0]) / (2 * h)
            assert np.abs(fd - J[:, k]).max() < 1e-6, (node, k, fd, J[:, k])


def test_consistent_graph_has_zero_objective_and_comes_back_unchanged():
    g = PG.noisy_graph(2, 6, loop_span=3, noise_deg=0.0, noise_t=0.0)
    out = PG.optimize(g['truth'], g['edges'], g['X'], g['info'], g['uncertain'], 0.05)
    assert out['result'][2] < 1e-18
    assert np.array_equal(out['poses'], g['truth'][:, :3])
    assert out['result'][:2].tolist() == [0, 0] and out['kept'].all()


def test_wrong_loop_closures_are_pruned_and_poses_improve():
    g = PG.noisy_graph(3, 12, loop_span=4, wrong_frac=0.2)
    assert g['wrong'].sum() >= 2
    out = PG.optimize(g['init'], g['edges'], g['X'], g['info'], g['uncertain'], 0.05)
    assert np.array_equal(~out['kept'], g['wrong'])
    assert PG.pose_error(out['poses'], g['truth']) < 0.5 * PG.pose_error(g['init'], g['truth'])
    assert out['result'][3] == (~g['wrong']).sum()


def test_information_restatement_uses_the_lowest_index_tie_rule():
    rng = np.random.default_rng(4)
    tgt = rng.uniform(-1, 1, (300, 3))
    tgt[:30] = tgt[30:60]                                  # duplicated targets: ties go to the lowest index
    src = tgt[rng.permutation(300)[:200]] + rng.normal(scale=0.01, size=(200, 3))
    pose = np.eye(3, 4)
    r = 0.05
    got = PG.information(src, tgt, pose, r)
    # brute force
    want = np.zeros((6, 6))
    for q in src:
        d2 = ((q - tgt) ** 2).sum(1)
        j = int(np.argmin(np.where(d2 < r * r, d2, np.inf)))
        if d2[j] < r * r:
            want += PG.info_of_points(tgt[j:j + 1])
    assert np.allclose(got, want, rtol=1e-12, atol=1e-12)
    d, _ = cKDTree(tgt).query(src, distance_upper_bound=r)
    assert got[5, 5] == np.isfinite(d).sum()


def test_cli_parsing():
    ap = M.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', 'c.ply', '--ckpt', 'r/ckpt/m.pth', '--out', 'o'])
    assert opt.fragments == ['a.ply', 'b.ply', 'c.ply'] and opt.icp is None and opt.voxel is None
    assert opt.min_overlap == 0.3 and opt.preference_loop_closure == 1.0 and opt.info_radius is None
    opt = ap.parse_args(['a', 'b', '--ckpt', 'k', '--out', 'o', '--icp', '0.05', '--icp_method', 'point_to_plane',
                         '--info_radius', '0.04', '--min_overlap', '0.2', '--preference_loop_closure', '2',
                         '--voxel', '0.01', '--batch_pairs', '3'])
    assert (opt.icp, opt.icp_method, opt.info_radius, opt.min_overlap, opt.preference_loop_closure, opt.voxel,
            opt.batch_pairs) == (0.05, 'point_to_plane', 0.04, 0.2, 2.0, 0.01, 3)
    assert M.all_pairs(4) == [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]


def test_est_log_layout_round_trips(tmp_path):
    rng = np.random.default_rng(6)
    P = np.stack([PG.random_pose(rng, 90.0, 2.0) for _ in range(4)])
    res = {'pairs': np.asarray(M.all_pairs(4)), 'poses': P}
    for k in ('edges', 'transformation', 'information', 'uncertain', 'confidence', 'kept', 'fit'):
        res[k] = np.zeros(1)
    M.write_outputs(res, str(tmp_path), 'scene-a')
    M.write_outputs(res, str(tmp_path), 'scene-a')             # rewritten, not appended
    keys, traj = E.read_trajectory(str(tmp_path / 'scene-a' / 'est.log'))
    assert [tuple(int(v) for v in k) for k in keys] == [(i, j, -1) for i, j in M.all_pairs(4)]
    for (i, j), T in zip(M.all_pairs(4), traj):
        assert np.abs(T - np.linalg.inv(P[i]) @ P[j]).max() < 1e-11
    assert M.scene_name('/data/3DMatch/7-scenes-redkitchen/cloud_bin_0.ply') == '7-scenes-redkitchen'


def test_multiway_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    for src, kernels in (('posegraph.cu', ('k_pose_graph',)),
                         ('traindata.cu', ('k_registration_information', 'k_transform_clouds'))):
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, src),
                                                        '-o', str(tmp_path / (src + '.o'))],
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr
        text = r.stdout + r.stderr
        for k in kernels:
            block = text[text.index(k):]
            stats = re.search(r'(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads', block)
            assert stats and stats.groups()[1:] == ('0', '0'), (k, block[:400])
