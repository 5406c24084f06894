"""Multi-scale ICP without a GPU: the float64 oracle's voxel down-sampling (tests/multiscale_icp_oracle.py) against an
independent restatement, the real pair on which the pyramid widens ICP's basin of convergence, `eval.icp_refine`'s
call layout with fakes, the command lines' flags and usage errors, and the compiler's report on voxel.cu."""
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import icp_oracle as I
import multiscale_icp_oracle as M
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import register as R
from test_colored_icp_host import _eval_3dmatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def restated(xyz, voxel, attr=None):
    """The down-sampling contract in plain Python: a dict voxel -> member list, filled point by point."""
    xyz = [tuple(map(float, p)) for p in np.asarray(xyz, np.float64).reshape(-1, 3)]
    if not xyz:
        return np.zeros((0, 3)), None
    lo = [min(p[d] for p in xyz) for d in range(3)]
    cells = {}
    for i, p in enumerate(xyz):
        key = tuple(int(math.floor((p[d] - (lo[d] - 0.5 * voxel)) / voxel)) for d in range(3))
        cells.setdefault(key, []).append(i)

    def mean(rows, members):
        out = []
        for d in range(3):
            s = 0.0
            for i in members:
                s += float(rows[i][d])
            out.append(s / len(members))
        return out
    keys = sorted(cells)
    pts = np.array([mean(xyz, cells[k]) for k in keys])
    att = None if attr is None else np.array([mean(np.asarray(attr, np.float64), cells[k]) for k in keys])
    return pts, att


def check_against_restatement(xyz, voxel, attr=None):
    got, got_attr, members = M.voxel_down_sample(xyz, voxel, attr)
    want, want_attr = restated(xyz, voxel, attr)
    assert np.array_equal(got, want.reshape(-1, 3))
    if attr is not None:
        assert np.array_equal(got_attr, want_attr.reshape(-1, 3))
    assert sum(len(m) for m in members) == len(np.asarray(xyz).reshape(-1, 3))
    assert all((np.diff(m) > 0).all() for m in members)
    return got, members


def test_points_on_the_faces_of_the_anchored_grid():
    """lo = 0 and V = 0.25 put the faces at -0.125 + k V, all exactly representable: a point on a face belongs to the
    voxel above it."""
    faces = np.array([[0.0, 0.0, 0.0], [0.125, 0.0, 0.0], [0.375, 0.125, 0.0], [0.125, 0.375, 0.625],
                      [0.1, 0.0, 0.0], [0.124, 0.2, 0.3]])
    got, members = check_against_restatement(faces, 0.25)
    v = M.voxel_indices(faces, 0.25)
    assert v[:, 0].tolist() == [0, 1, 2, 1, 0, 0]
    assert [m.tolist() for m in members] == [[0, 4], [5], [1], [3], [2]]        # (0,0,0) (0,1,1) (1,0,0) ...


def test_duplicates_one_point_and_empty_clouds():
    rng = np.random.default_rng(1)
    base = rng.uniform(-1, 1, (50, 3))
    dup = np.concatenate([base, base[::3], base[:5]])
    rgb = rng.uniform(0, 1, dup.shape)
    got, members = check_against_restatement(dup, 0.3, rgb)
    assert sum(len(m) for m in members) == dup.shape[0]
    one, _, m1 = M.voxel_down_sample(np.array([[1.5, -2.0, 3.25]]), 0.05)
    assert np.array_equal(one, np.array([[1.5, -2.0, 3.25]])) and [m.tolist() for m in m1] == [[0]]
    empty, ea, m0 = M.voxel_down_sample(np.zeros((0, 3)), 0.05, np.zeros((0, 3)))
    assert empty.shape == (0, 3) and ea.shape == (0, 3) and m0 == []


def test_an_analytic_lattice():
    """A 6 x 5 x 4 lattice 0.5 + 0.1 g at voxel 0.25: the grid starts at 0.5 - 0.125, so lattice point g falls in voxel
    floor((0.1 g + 0.125) / 0.25) = (4 g + 5) // 10 per axis, at least 0.025 from any face."""
    g = np.stack(np.meshgrid(np.arange(6), np.arange(5), np.arange(4), indexing='ij'), -1).reshape(-1, 3)
    xyz = 0.5 + 0.1 * g
    got, members = check_against_restatement(xyz, 0.25)
    vox = (4 * g + 5) // 10
    want = sorted(set(map(tuple, vox.tolist())))
    assert len(want) == 3 * 3 * 2 and len(members) == len(want)
    for key, m in zip(want, members):
        assert m.tolist() == np.nonzero((vox == key).all(axis=1))[0].tolist(), key
    assert np.array_equal(M.voxel_indices(xyz, 0.25), vox)


def test_bounding_box_anchoring_is_not_origin_anchoring():
    """0.0 and 0.09 share the origin-anchored voxel [0, 0.1); with the grid at lo - V/2 = -0.05 they do not."""
    xyz = np.array([[0.0, 0.0, 0.0], [0.09, 0.0, 0.0]])
    assert np.floor(xyz[0, 0] / 0.1) == np.floor(xyz[1, 0] / 0.1)
    got, members = check_against_restatement(xyz, 0.1)
    assert len(members) == 2
    # and a cloud's rows depend on its own minimum only: shifting it by a multiple of V shifts them
    moved, _, _ = M.voxel_down_sample(xyz + 0.25, 0.1)
    assert np.allclose(moved, got + 0.25, rtol=0, atol=1e-15)


def test_index_range_and_non_finite_are_refused():
    with pytest.raises(ValueError):
        M.voxel_down_sample(np.array([[0.0, 0.0, 0.0], [70000.0 * 0.01, 0.0, 0.0]]), 0.01)
    with pytest.raises(ValueError):
        M.voxel_down_sample(np.array([[0.0, np.nan, 0.0]]), 0.01)
    M.voxel_down_sample(np.array([[0.0, 0.0, 0.0], [65535.0 * 0.25, 0.0, 0.0]]), 0.25)      # index 65535 is kept


# The perturbed real pair the GPU test also uses: single-level point-to-plane ICP at the finest radius misses the
# ground truth, the pyramid reaches it with the same iteration budget.
BASIN = dict(fixture=('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'), seed=703, deg=10.0, metres=0.15,
             voxels=[0.1, 0.05, 0.0], level_iters=[50, 30, 14], radius=0.0375, method='point_to_plane')


def basin_case():
    from test_gpu_icp import perturb
    from test_gpu_register import gt_log_pair
    s, t, gt = gt_log_pair(*BASIN['fixture'])
    return s, t, gt, perturb(gt, BASIN['seed'], BASIN['deg'], BASIN['metres'])


def pose_error(pose, gt):
    """-> (rotation error in degrees, translation error in metres)."""
    c = (np.trace(np.asarray(pose)[:, :3] @ gt[:, :3].T) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0)))), float(np.linalg.norm(np.asarray(pose)[:, 3] - gt[:, 3]))


def reached(pose, gt):
    rot, trans = pose_error(pose, gt)
    return rot < 5.0 and trans < 0.1


def test_the_pyramid_widens_the_basin_on_a_real_pair():
    s, t, gt, init = basin_case()
    assert not reached(init, gt)
    one = M.single_level(BASIN['method'], s, t, init, BASIN['radius'], sum(BASIN['level_iters']))
    pyr = M.multiscale_icp(s, t, init, BASIN['voxels'], None, BASIN['level_iters'], radius=BASIN['radius'],
                           method=BASIN['method'])
    assert not reached(one['pose'], gt), pose_error(one['pose'], gt)
    assert reached(pyr['pose'], gt), pose_error(pyr['pose'], gt)
    assert pyr['levels'].shape == (3, 4) and (pyr['levels'][:, 3] < BASIN['level_iters']).all()


def plane(rng, n):
    g = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing='ij'), -1).reshape(-1, 2) * 0.01
    g = g + rng.uniform(-0.002, 0.002, g.shape)
    return np.concatenate([g, 0.3 * g[:, :1] ** 2 + 1.0], axis=1)


@pytest.mark.parametrize('method', ['point_to_point', 'point_to_plane', 'generalized', 'colored'])
def test_icp_refine_pyramid_call_layout(method):
    """Per level: one down-sampling call over all 2B clouds (none at V = 0), normals and gradients at 2 R_l, then icp
    at R_l with I_l iterations from the previous level's pose."""
    rng = np.random.default_rng(2)
    B = 2
    src, tgt = [plane(rng, 12) for _ in range(B)], [plane(rng, 12) for _ in range(B)]
    cols = ([np.full((c.shape[0], 3), 0.5) for c in src], [np.full((c.shape[0], 3), 0.25) for c in tgt])
    calls = []

    def down(clouds, v, colors=None):
        calls.append(('down', len(clouds), v, colors is not None))
        outs = [M.voxel_down_sample(c, v, None if colors is None else k)
                for c, k in zip(clouds, colors or [None] * len(clouds))]
        return [o[0] for o in outs], None if colors is None else [o[1] for o in outs]

    def normals(clouds, r, max_nn):
        calls.append(('normals', len(clouds), r, max_nn))
        return [np.tile([0.0, 0.0, 1.0], (c.shape[0], 1)) for c in clouds]

    def gradients(clouds, nrm, k, r, max_nn):
        calls.append(('gradients', len(clouds), r, max_nn))
        return [np.zeros_like(c) for c in clouds]

    def icp(s, t, init, r, it, **kw):
        calls.append(('icp', r, it, [c.shape[0] for c in s], np.asarray(init).copy()))
        pose = np.asarray(init, np.float64).copy()
        pose[:, :, 3] += r                                  # a recognisable pose for the next level to start from
        return pose, np.tile([1.0, 0.0, 0.0, float(it)], (len(s), 1))

    init = np.tile(np.eye(3, 4), (B, 1, 1))
    kw = dict(icp=icp, estimate_normals=normals, color_gradients=gradients, voxel_down_sample=down,
              colors=cols if method == 'colored' else None)
    pose, res, levels = E.icp_refine(src, tgt, init, 0.015, 7, method, normal_max_nn=20, voxels=[0.04, 0.02, 0.0],
                                     level_iters=[5, 4, 3], return_levels=True, **kw)
    seq = []
    for v, r, it in ((0.04, 0.04, 5), (0.02, 0.02, 4), (0.0, 0.015, 3)):
        if v > 0:
            seq.append(('down', 2 * B, v, method == 'colored'))
        if method != 'point_to_point':
            seq.append(('normals', 2 * B if method == 'generalized' else B, 2.0 * r, 20))
        if method == 'colored':
            seq.append(('gradients', B, 2.0 * r, 30))
        seq.append(('icp', r, it))
    assert [c[:3] if c[0] == 'icp' else c for c in calls] == seq
    icps = [c for c in calls if c[0] == 'icp']
    assert icps[2][3] == [c.shape[0] for c in src]                     # the last level runs on the full clouds
    assert icps[0][3] == [M.voxel_down_sample(c, 0.04)[0].shape[0] for c in src]
    assert np.array_equal(icps[0][4], init)                             # pose chaining
    assert np.allclose(icps[1][4][:, :, 3], 0.04) and np.allclose(icps[2][4][:, :, 3], 0.06)
    assert np.allclose(pose[:, :, 3], 0.075) and levels.shape == (B, 3, 4)
    assert levels[:, :, 3].tolist() == [[5, 4, 3]] * B and np.array_equal(res, levels[:, 2])
    # radii given explicitly
    calls.clear()
    E.icp_refine(src, tgt, init, 0.015, 7, method, voxels=[0.04, 0.02], radii=[0.08, 0.03], **kw)
    assert [c[1:3] for c in calls if c[0] == 'icp'] == [(0.08, 7), (0.03, 7)]
    # without voxels: today's sequence, one level, no down-sampling; voxels=[0], radii=[R] makes the same calls
    calls.clear()
    p0, r0 = E.icp_refine(src, tgt, init, 0.015, 7, method, **kw)
    plain = [c[:3] if c[0] == 'icp' else c for c in calls]
    assert not any(c[0] == 'down' for c in calls) and plain[-1] == ('icp', 0.015, 7)
    calls.clear()
    p1, r1, lv = E.icp_refine(src, tgt, init, 0.015, 7, method, voxels=[0.0], radii=[0.015], return_levels=True, **kw)
    assert [c[:3] if c[0] == 'icp' else c for c in calls] == plain
    assert np.array_equal(p0, p1) and np.array_equal(r0, r1) and lv.shape == (B, 1, 4)


def test_icp_refine_refuses_bad_pyramids():
    src = [np.zeros((3, 3))]
    for kw in (dict(voxels=[0.02, 0.04]), dict(voxels=[0.02, 0.02]), dict(voxels=[0.0, 0.02]), dict(voxels=[]),
               dict(voxels=[0.04, -0.02]), dict(voxels=[0.04, 0.02], radii=[0.04]),
               dict(voxels=[0.04], level_iters=[5, 5]), dict(voxels=[0.04], radii=[float('inf')]),
               dict(voxels=[0.04], radii=[0.0]), dict(voxels=[0.04], level_iters=[-1]),
               dict(voxels=[0.04], normal_radius=0.1), dict(voxels=[0.04], normals=([None], [None]))):
        with pytest.raises(ValueError):
            E.icp_refine(src, src, np.eye(3, 4)[None], 0.02, icp=lambda *a, **k: None, **kw)


REG = ['a.ply', 'b.ply', '--ckpt', 'c/ckpt/m.pth']


def test_flags_parse_and_icp_kwargs():
    opt = R.parse_args(REG + ['--icp', '0.01', '--icp_voxels', '0.04,0.02,0.01', '--icp_radii', '0.04,0.02,0.01',
                              '--icp_level_iters', '50,30,14', '--icp_method', 'colored'])
    assert (opt.icp_voxels, opt.icp_radii, opt.icp_level_iters) == ([0.04, 0.02, 0.01], [0.04, 0.02, 0.01],
                                                                   [50, 30, 14])
    kw = E.icp_kwargs(opt)
    assert (kw['voxels'], kw['radii'], kw['level_iters']) == ([0.04, 0.02, 0.01], [0.04, 0.02, 0.01], [50, 30, 14])
    opt = R.parse_args(REG + ['--icp', '0.01', '--icp_voxels', '0.04,0'])
    assert E.icp_kwargs(opt)['radii'] is None and E.icp_kwargs(opt)['level_iters'] is None
    for argv in (REG, REG + ['--icp', '0.03'], REG + ['--icp', '0.03', '--icp_method', 'colored']):
        assert not {'voxels', 'radii', 'level_iters'} & set(E.icp_kwargs(R.parse_args(argv)))
    ap = MW.parser()
    opt = ap.parse_args(['a.ply', 'b.ply', 'c.ply', '--ckpt', 'x', '--out', 'o', '--icp', '0.02', '--icp_voxels',
                         '0.05,0.025', '--icp_level_iters', '10,5'])
    E.check_icp_arguments(ap, opt, colors=True)
    assert (opt.icp_voxels, opt.icp_level_iters) == ([0.05, 0.025], [10, 5])


BAD = [(['--icp_voxels', '0.04'], '--icp_voxels needs --icp'),
       (['--icp_level_iters', '5'], '--icp_level_iters needs --icp'),
       (['--icp', '0.01', '--icp_radii', '0.04'], '--icp_radii needs --icp_voxels'),
       (['--icp', '0.01', '--icp_level_iters', '5'], '--icp_level_iters needs --icp_voxels'),
       (['--icp', '0.01', '--icp_voxels', '0.04,0.02', '--icp_radii', '0.04'], '1 values for 2 voxels'),
       (['--icp', '0.01', '--icp_voxels', '0.04,0.02', '--icp_level_iters', '5,5,5'], '3 values for 2 voxels'),
       (['--icp', '0.01', '--icp_voxels', '0.02,0.04'], 'strictly decreasing'),
       (['--icp', '0.01', '--icp_voxels', '0,0.02'], 'strictly decreasing'),
       (['--icp', '0.01', '--icp_voxels', '0.04,nan'], 'strictly decreasing'),
       (['--icp', '0.01', '--icp_voxels', '0.04', '--icp_radii', 'inf'], 'finite and > 0'),
       (['--icp', '0.01', '--icp_voxels', '0.04', '--icp_radii', '-0.1'], 'finite and > 0'),
       (['--icp', '0.01', '--icp_voxels', '0.04', '--icp_level_iters', '-1'], '>= 0'),
       (['--icp', '0.01', '--icp_voxels', '0.04', '--normal_radius', '0.1'], '--normal_radius does not go'),
       (['--icp', '0.01', '--icp_voxels', '0.04,x'], 'comma-separated float')]


@pytest.mark.parametrize('extra,msg', BAD)
def test_usage_errors_before_the_checkpoint(extra, msg, capsys, tmp_path):
    """The checkpoint does not exist: the usage error comes first, on every command line."""
    ckpt = str(tmp_path / 'none' / 'ckpt' / 'm.pth')
    runs = [lambda: R.main(['a.ply', 'b.ply', '--ckpt', ckpt] + extra),
            lambda: MW.main(['a.ply', 'b.ply', 'c.ply', '--ckpt', ckpt, '--out', str(tmp_path / 'o')] + extra),
            lambda: _eval_3dmatch().main(['--root', 'r', '--info', 'i.pkl', '--gt', 'g', '--ckpt', ckpt] + extra)]
    for run in runs:
        with pytest.raises(SystemExit) as e:
            run()
        err = capsys.readouterr().err
        assert e.value.code == 2 and msg in err, err


def test_eval_3dmatch_passes_the_pyramid_to_icp_forward(monkeypatch):
    ev = _eval_3dmatch()
    args = ev.parser().parse_args(['--root', 'r', '--info', 'i.pkl', '--gt', 'g', '--ckpt', 'm.pth', '--icp', '0.02',
                                   '--icp_voxels', '0.05,0', '--icp_level_iters', '9,4'])
    seen = {}
    monkeypatch.setattr(ev.E, 'icp_forward', lambda fn, *a, **kw: seen.update(kw))
    monkeypatch.setattr(ev, 'get_config', lambda name: {}, raising=False)
    monkeypatch.setattr(ev, 'RegTR', lambda cfg: type('M', (), {'to': lambda s, d: s, 'eval': lambda s: s,
                                                               'load_state_dict': lambda s, *a, **k: None})(),
                        raising=False)
    monkeypatch.setattr(ev.torch, 'load', lambda *a, **k: {})
    monkeypatch.setattr(ev, 'GraphedRegTR', lambda m: m, raising=False)
    ev.network_forward(args)
    assert (seen['voxels'], seen['radii'], seen['level_iters']) == ([0.05, 0.0], None, [9, 4])


def test_voxel_kernels_do_not_spill():
    """voxel.cu's own kernels (the minima, the keys, the means) and the shared head-flag and offset kernels: no
    spills."""
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    from regtr_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        r = subprocess.run([nvcc] + build.NVCC_FLAGS + ['-Xptxas', '-v', '-c', os.path.join(build.CSRC, 'voxel.cu'),
                                                        '-o', os.path.join(tmp, 'voxel.o')],
                           capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    text = r.stdout + r.stderr
    entries = re.findall(r"Compiling entry function '(\w+)'[^\n]*\n[^\n]*Function properties for \w+\n\s*(\d+) "
                         r"bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n[^\n]*Used (\d+) "
                         r"registers", text)
    own = sorted(n for n in ('k_cloud_min', 'k_voxel_keys', 'k_voxel_mean64', 'k_head_flags', 'k_cloud_offsets')
                 if any(n in e[0] for e in entries))
    assert own == ['k_cloud_min', 'k_cloud_offsets', 'k_head_flags', 'k_voxel_keys', 'k_voxel_mean64'], entries
    for name, _, st, ld, regs in entries:
        assert (st, ld) == ('0', '0'), (name, st, ld)
    assert set(re.findall(r'(\d+) bytes spill (?:stores|loads)', text)) == {'0'}
