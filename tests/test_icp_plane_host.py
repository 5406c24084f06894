"""Normal estimation and point-to-plane ICP on the host: the float64 oracle (tests/icp_plane_oracle.py) against
analytic normals, brute-force neighbour sets and known transforms, its singular and 6-vector rules, the CLI flags of
`python -m regtr_b200.register`, the 3DMatch benchmark wrapper's point-to-plane layout, and that the normal kernels
do not spill (the ICP kernels' check is in test_icp_host.py)."""
import os
import re
import subprocess

import numpy as np
import torch
from scipy.spatial.transform import Rotation

import icp_oracle as I
import icp_plane_oracle as N
import train_data_oracle as O
from regtr_b200 import eval as E
from regtr_b200 import register as R


def pose34(axis, deg, t):
    axis = np.asarray(axis, np.float64)
    p = np.eye(3, 4)
    p[:, :3] = O.axis_angle(axis / np.linalg.norm(axis), np.deg2rad(deg))
    p[:, 3] = t
    return p


def inverse(p):
    inv = np.eye(3, 4)
    inv[:, :3] = p[:, :3].T
    inv[:, 3] = -p[:, :3].T @ p[:, 3]
    return inv


def oriented(n, p):
    """n flipped towards the origin, per row."""
    s = (n * p).sum(axis=1)
    return np.where(s[:, None] > 0, -n, n)


def test_normals_of_planes_match_the_analytic_normal():
    rng = np.random.default_rng(1)
    for k in range(3):
        rot = pose34(rng.normal(size=3), rng.uniform(0, 180), rng.uniform(-2, 2, 3))
        uv = rng.uniform(-0.5, 0.5, (1500, 2))
        pts = I.transform(rot, np.concatenate([uv, np.zeros((1500, 1))], axis=1))
        nrm, cnt = N.estimate_normals(pts, 0.08, 30)
        assert (cnt >= 3).all()
        want = oriented(np.tile(rot[:, 2], (1500, 1)), pts)
        assert np.abs(nrm - want).max() < 1e-12, np.abs(nrm - want).max()
        s = (nrm[:, 0] * pts[:, 0] + nrm[:, 1] * pts[:, 1]) + nrm[:, 2] * pts[:, 2]
        assert (s <= 0).all()


def test_normals_of_a_sphere_match_the_radial_direction():
    """Symmetric caps of a unit sphere: a pole point and rings of 6 points at equal polar angles, so that the
    neighbourhood's covariance has the radial axis as an exact eigenvector; the normal points to the centre."""
    rng = np.random.default_rng(2)
    caps, poles = [], []
    for k in range(40):
        axis = rng.normal(size=3)
        axis /= np.linalg.norm(axis)
        rot = Rotation.align_vectors([axis], [[0.0, 0.0, 1.0]])[0].as_matrix()
        pts = [[0.0, 0.0, 1.0]]
        for theta in (0.02, 0.04):
            for a in np.arange(6) * np.pi / 3 + theta:
                pts.append([np.sin(theta) * np.cos(a), np.sin(theta) * np.sin(a), np.cos(theta)])
        cap = np.asarray(pts) @ rot.T
        if any(np.linalg.norm(cap[0] - c[0]) < 0.3 for c in caps):
            continue
        poles.append(sum(len(c) for c in caps))
        caps.append(cap)
    xyz = np.concatenate(caps)
    nrm, cnt = N.estimate_normals(xyz, 0.05, 30)
    assert (cnt[poles] == 13).all()
    want = -xyz[poles] / np.linalg.norm(xyz[poles], axis=1, keepdims=True)
    assert np.abs(nrm[poles] - want).max() < 1e-12, np.abs(nrm[poles] - want).max()


def test_neighbour_sets_equal_brute_force():
    rng = np.random.default_rng(3)
    for n, r, max_nn in ((400, 0.2, 30), (300, 0.5, 7), (50, 0.05, 64)):
        xyz = rng.uniform(-1, 1, (n, 3))
        xyz[: n // 10] = xyz[n // 10: 2 * (n // 10)]                  # duplicates: ties go to the lower index
        q, j, dd = N.neighbours(xyz, r, max_nn)
        for i in range(n):
            d = xyz[i] - xyz
            d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
            inside = np.nonzero(d2 < r * r)[0]
            want = inside[np.lexsort((inside, d2[inside]))][:max_nn]
            assert np.array_equal(j[q == i], want), i
            assert np.array_equal(dd[q == i], d2[want])
        _, cnt = N.estimate_normals(xyz, r, max_nn)
        assert np.array_equal(cnt, np.bincount(q, minlength=n))
    # a lone point and a pair have no normal
    nrm, cnt = N.estimate_normals(np.array([[0.0, 0.0, 0.0], [5.0, 0.0, 0.0], [5.01, 0.0, 0.0]]), 0.1, 30)
    assert cnt.tolist() == [1, 2, 2] and not nrm.any()
    # exactly on the radius is not a neighbour (strict)
    _, cnt = N.estimate_normals(np.array([[0.0, 0.0, 0.0], [0.5, 0.0, 0.0]]), 0.5, 30)
    assert cnt.tolist() == [1, 1]


def room(rng, n_face=1500):
    """Points on the inside faces of a 4 x 3 x 2.5 m box with a 1 x 0.8 x 0.9 m table in it."""
    out = []
    for lo, hi, m in (((-2.0, -1.5, 0.0), (2.0, 1.5, 2.5), n_face), ((-0.5, -0.4, 0.0), (0.5, 0.4, 0.9), n_face // 3)):
        lo, hi = np.asarray(lo), np.asarray(hi)
        for axis in range(3):
            for side in (lo, hi):
                p = rng.uniform(lo, hi, (m, 3))
                p[:, axis] = side[axis]
                out.append(p)
    return np.concatenate(out)


def test_point_to_plane_recovers_a_rigid_transform_on_a_noiseless_pair():
    rng = np.random.default_rng(5)
    tgt = room(rng)
    gt = pose34([0.2, -0.4, 0.9], 3.0, [0.03, -0.02, 0.01])
    src = I.transform(inverse(gt), tgt)                            # gt maps src exactly onto tgt
    nrm, cnt = N.estimate_normals(tgt, 0.15, 30)
    assert (cnt >= 3).mean() > 0.99
    out = N.icp(src, tgt, nrm, np.eye(3, 4), 0.2, max_iteration=100, relative_fitness=1e-12, relative_rmse=1e-12)
    assert np.abs(out['pose'] - gt).max() < 1e-10, np.abs(out['pose'] - gt).max()
    assert out['fitness'] == 1.0 and out['rmse'] < 1e-10 and out['k'] == len(src)
    assert 0 < out['iterations'] < 100
    pose, res = N.icp_batch([src], [tgt], [nrm], np.eye(3, 4)[None], 0.2, 100, 1e-12, 1e-12)
    assert np.array_equal(pose[0], out['pose']) and res[0].tolist() == [1.0, out['rmse'], len(src),
                                                                        out['iterations']]


def test_correspondences_on_one_plane_give_the_identity_and_stop():
    rng = np.random.default_rng(7)
    uv = rng.uniform(-1, 1, (500, 2))
    tgt = np.concatenate([uv, np.zeros((500, 1))], axis=1)
    src = tgt + [0.01, -0.02, 0.0]                                 # slid along the plane
    nrm = np.tile([0.0, 0.0, -1.0], (500, 1))
    jtj, _ = N.plane_system(src, tgt, nrm)
    assert abs(np.linalg.det(jtj)) < 1e-6
    assert np.array_equal(N.plane_update(src, tgt, nrm), np.eye(3, 4))
    init = pose34([0, 0, 1], 0.0, [0.0, 0.0, 0.0])
    out = N.icp(src, tgt, nrm, init, 0.1)
    assert np.array_equal(out['pose'], init) and out['iterations'] == 1 and out['k'] == 500
    # without correspondences: the identity too
    far = N.icp(src + 50.0, tgt, nrm, init, 0.1)
    assert np.array_equal(far['pose'], init) and far['k'] == 0 and far['iterations'] == 1
    # zero normals drop out of the update but not out of k
    zero = N.icp(src, tgt, np.zeros_like(nrm), init, 0.1)
    assert np.array_equal(zero['pose'], init) and zero['k'] == 500


def test_six_vector_rule_matches_an_independent_construction():
    rng = np.random.default_rng(9)
    for _ in range(20):
        x = rng.normal(size=6) * [0.5, 0.5, 0.5, 1.0, 1.0, 1.0]
        got = N.vec6_to_pose(x)
        want = Rotation.from_euler('ZYX', [x[2], x[1], x[0]]).as_matrix()          # intrinsic z, y', x''
        assert np.abs(got[:, :3] - want).max() < 1e-15
        assert np.array_equal(got[:, 3], x[3:])


def test_register_parser_accepts_the_point_to_plane_flags():
    ap = R.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.0375', '--icp_method',
                         'point_to_plane', '--normal_radius', '0.08', '--normal_max_nn', '20'])
    assert (opt.icp, opt.icp_method, opt.normal_radius, opt.normal_max_nn) == (0.0375, 'point_to_plane', 0.08, 20)
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.0375'])
    assert (opt.icp_method, opt.normal_radius, opt.normal_max_nn) == ('point_to_point', None, 30)
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth', '--icp', '0.0375', '--icp_iters', '12'])
    assert opt.icp == 0.0375 and opt.icp_iters == 12
    opt = ap.parse_args(['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth'])
    assert opt.icp is None and opt.icp_iters == 30


def test_benchmark_wrapper_point_to_plane_layout_on_cpu():
    rng = np.random.default_rng(11)
    B, L = 2, 3
    tgts = [room(rng, 300) * 0.5 for _ in range(B)]
    gts = [pose34([0, 0, 1], 2.0, [0.01, 0, 0]), pose34([1, 0, 0], -1.5, [0, 0.02, 0])]
    srcs = [torch.from_numpy(I.transform(inverse(g), t)).float() for t, g in zip(tgts, gts)]
    net = torch.from_numpy(np.stack([np.stack(gts)] * L)).float()
    net_before = net.clone()
    batch = {'src_xyz': srcs, 'tgt_xyz': [torch.from_numpy(t).float() for t in tgts],
             'pose': torch.from_numpy(np.stack(gts)).float()}
    calls = []

    def oracle_normals(clouds, radius, max_nn):
        calls.append(('normals', radius, max_nn))
        return [N.estimate_normals(c.numpy(), radius, max_nn)[0] for c in clouds]

    def oracle_icp(src_list, tgt_list, init, radius, max_iteration, method, tgt_normals):
        calls.append(('icp', radius, max_iteration, method))
        return N.icp_batch([s.numpy() for s in src_list], [t.numpy() for t in tgt_list], tgt_normals, init.numpy(),
                           radius, max_iteration)

    run = E.icp_forward(lambda b: {'pose': net, 'src_kp': 'kept'}, 0.05, 7, icp=oracle_icp, method='point_to_plane',
                        normal_max_nn=20, estimate_normals=oracle_normals)
    pred = run(batch)
    assert calls == [('normals', 0.1, 20), ('icp', 0.05, 7, 'point_to_plane')]   # normal radius 2 R by default
    assert pred['pose'].shape == (1, B, 3, 4) and pred['pose'].dtype == torch.float64
    assert torch.equal(pred['pose_coarse'][0], net[-1].double())
    assert pred['src_kp'] == 'kept' and torch.equal(net, net_before)
    normals = oracle_normals(batch['tgt_xyz'], 0.1, 20)
    want, _ = oracle_icp(batch['src_xyz'], batch['tgt_xyz'], net[-1].double(), 0.05, 7, 'point_to_plane', normals)
    assert np.array_equal(pred['pose'][0].numpy(), want)
    calls.clear()
    E.icp_forward(lambda b: {'pose': net}, 0.05, 7, icp=oracle_icp, method='point_to_plane', normal_radius=0.07,
                  estimate_normals=oracle_normals)(batch)
    assert calls[0] == ('normals', 0.07, 30)


def test_normal_kernels_do_not_spill(tmp_path):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    kernels = ('k_normals_init', 'k_normalsE')
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'normals.cu'),
                                                    '-o', str(tmp_path / 'normals.o')],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert len(entries) == len(kernels), [e[0] for e in entries]
    for k in kernels:
        hit = [e for e in entries if k in e[0]]
        assert len(hit) == 1, k
    for name, _, st, ld in entries:
        assert (st, ld) == ('0', '0'), (name, st, ld)
    # the device functions the kernels call (sincos's slow path) too
    assert set(re.findall(r'bytes spill (?:stores|loads)', text)) and \
        set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
