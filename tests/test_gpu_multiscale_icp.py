"""Voxel down-sampling (`ops.voxel_down_sample`, regtr_voxel_down_sample) and multi-scale ICP (`eval.icp_refine` with
voxels=) on the device against the float64 oracle (tests/multiscale_icp_oracle.py), on the real 3DMatch fixtures and
on synthetic 3DMatch-shaped pairs, coloured by `colored_icp_oracle.texture`.

Covered: down-sampling at 1 to 10 cm with and without colours (membership, counts and order exact, means within
1e-12), stacked against one call per cloud, reruns, an empty cloud, the launch count and the key-range status; every
level of the pyramid of all four ICP methods against the oracle's single-level ICP on the device's own normals and
gradients, with the same iteration count; the batch against one call per pair; voxels=[0] against voxels=None; the
perturbed real pair that only the pyramid recovers; `register --icp_voxels` end to end and `multiway`'s pair
registration with a colored pyramid."""
import os

import numpy as np
import pytest
import torch

import colored_icp_oracle as C
import gicp_oracle as G
import icp_oracle as I
import multiscale_icp_oracle as M
from regtr_b200 import lib, ops
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from test_gpu_colored_icp import REAL, _checkpoint, coloured_pairs
from test_gpu_icp import RADIUS, _run_register, perturb
from test_multiscale_icp_host import BASIN, basin_case, reached

pytestmark = pytest.mark.gpu
VOXELS = [0.05, 0.025, 0.0]
LEVEL_ITERS = [20, 15, 10]


def clouds_and_colours():
    pairs = coloured_pairs()
    return [c for p in pairs for c in p[:2]], [c for p in pairs for c in p[3:]]


def check_down(dev, dev_rgb, xyz, v, rgb):
    want, want_rgb, _ = M.voxel_down_sample(xyz, v, rgb)
    got = dev.cpu().numpy()
    assert got.shape == want.shape, (v, got.shape, want.shape)
    assert np.abs(got - want).max(initial=0.0) <= 1e-12
    if rgb is not None:
        assert np.abs(dev_rgb.cpu().numpy() - want_rgb).max(initial=0.0) <= 1e-12


@pytest.mark.parametrize('v', [0.01, 0.025, 0.05, 0.1])
def test_voxel_down_sample_against_the_oracle(v):
    clouds, rgbs = clouds_and_colours()
    out, out_rgb = ops.voxel_down_sample(clouds, v, colors=rgbs)
    plain, none = ops.voxel_down_sample(clouds, v)
    assert none is None and len(out) == len(clouds)
    again, again_rgb = ops.voxel_down_sample(clouds, v, colors=rgbs)
    for b, (c, k) in enumerate(zip(clouds, rgbs)):
        assert out[b].dtype == torch.float64 and out[b].shape[1] == 3
        check_down(out[b], out_rgb[b], c, v, k)
        assert torch.equal(plain[b], out[b]) and torch.equal(again[b], out[b]) and torch.equal(again_rgb[b], out_rgb[b])
        alone, alone_rgb = ops.voxel_down_sample([c], v, colors=[k])
        assert torch.equal(alone[0], out[b]) and torch.equal(alone_rgb[0], out_rgb[b]), b


def test_empty_cloud_launch_count_and_key_range():
    clouds, rgbs = clouds_and_colours()
    batch = [clouds[0], np.zeros((0, 3)), clouds[1][:1], clouds[2]]
    out, _ = ops.voxel_down_sample(batch, 0.03)
    assert out[1].shape == (0, 3) and torch.equal(out[2], torch.from_numpy(clouds[1][:1]).cuda())
    for b in (0, 3):
        assert torch.equal(out[b], ops.voxel_down_sample([batch[b]], 0.03)[0][0])
    counts = []
    for cl, v in (([clouds[0]], 0.01), (clouds, 0.1), ([np.zeros((0, 3))], 0.05), (clouds * 3, 0.02)):
        before = ops.LAUNCHES
        ops.voxel_down_sample(cl, v)
        counts.append(ops.LAUNCHES - before)
    assert counts == [ops.voxel_down_sample_launches()] * 4
    far = np.array([[0.0, 0.0, 0.0], [70000.0 * 0.01, 0.0, 0.0]])
    with pytest.raises(lib.RegtrLibError, match='voxel 0.01'):
        ops.voxel_down_sample([clouds[0], far], 0.01)
    with pytest.raises(lib.RegtrLibError):
        ops.voxel_down_sample([np.array([[0.0, np.inf, 0.0]])], 0.01)
    status = ops.new_status(torch.device('cuda'))
    ops.voxel_down_sample([far], 0.01, status=status)
    assert int(status.item()) & ops.STATUS_KEY_RANGE
    ok = ops.new_status(torch.device('cuda'))
    ops.voxel_down_sample([np.array([[0.0, 0.0, 0.0], [65535.0 * 0.25, 0.0, 0.0]])], 0.25, status=ok)
    assert int(ok.item()) == 0
    with pytest.raises(ValueError):
        ops.voxel_down_sample([clouds[0]], 0.0)
    with pytest.raises(ValueError):
        ops.voxel_down_sample([clouds[0]], 0.02, colors=[rgbs[0][1:]])


def method_kw(method):
    return dict(loss='huber', loss_k=0.02) if method in ('point_to_plane', 'generalized') else {}


def oracle_level(method, s, t, init, r, it, kw, icp_kw):
    """The oracle's single-level ICP on the device's level inputs (its normals and gradients)."""
    a = lambda x: x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)        # noqa: E731
    if method == 'point_to_point':
        return I.icp(s, t, init, r, it)
    nt = a(kw['tgt_normals'])
    if method == 'colored':
        return C.icp(s, t, nt, a(kw['src_colors']), a(kw['tgt_colors']), a(kw['tgt_color_gradients']), init, r, it,
                     **icp_kw)
    sn = a(kw['src_normals']) if method == 'generalized' else None
    return G.icp(s, t, nt, init, r, it, method=method, src_normals=sn, **icp_kw)


def run_pyramid(pairs, method, **kw):
    """icp_refine's pyramid over pairs (src, tgt, init, src_rgb, tgt_rgb), recording every level's icp call."""
    calls = []

    def icp(s, t, init, r, it, **k):
        out = ops.icp(s, t, init, r, it, **k)
        calls.append((s, t, init.clone() if torch.is_tensor(init) else init, r, it, k, out))
        return out
    init = torch.from_numpy(np.stack([p[2] for p in pairs])).cuda()
    colors = ([p[3] for p in pairs], [p[4] for p in pairs]) if method == 'colored' else None
    pose, res, levels = E.icp_refine([p[0] for p in pairs], [p[1] for p in pairs], init, RADIUS, 30, method, icp=icp,
                                     colors=colors, voxels=VOXELS, level_iters=LEVEL_ITERS, return_levels=True, **kw)
    return pose, res, levels, calls


@pytest.mark.parametrize('method', ['point_to_point', 'point_to_plane', 'generalized', 'colored'])
def test_every_level_against_the_oracle(method):
    pairs = coloured_pairs()
    kw = method_kw(method)
    pose, res, levels, calls = run_pyramid(pairs, method, **kw)
    assert levels.shape == (len(pairs), 3, 4) and torch.equal(levels[:, 2], res) and len(calls) == 3
    assert torch.equal(calls[0][2], torch.from_numpy(np.stack([p[2] for p in pairs])).cuda())
    for l, (s_l, t_l, init, r, it, k, (lp, lr)) in enumerate(calls):
        v = VOXELS[l]
        assert (r, it) == ((v if v > 0 else RADIUS), LEVEL_ITERS[l])
        if l > 0:
            assert torch.equal(init, calls[l - 1][6][0])                         # chained from the previous level
        assert torch.equal(levels[:, l], lr)
        lp, lr = lp.cpu().numpy(), lr.cpu().numpy()
        for b, p in enumerate(pairs):
            s, t = (p[0], p[1]) if v == 0 else (s_l[b].cpu().numpy(), t_l[b].cpu().numpy())
            if v > 0:
                assert np.abs(s - M.voxel_down_sample(p[0], v)[0]).max() <= 1e-12
                assert np.abs(t - M.voxel_down_sample(p[1], v)[0]).max() <= 1e-12
            kb = {name: x[b] for name, x in k.items() if isinstance(x, (list, tuple))}
            o = oracle_level(method, s, t, init[b].cpu().numpy(), r, it, kb,
                             {} if method == 'point_to_point' else {n: x for n, x in kw.items()})
            assert int(lr[b, 3]) == o['iterations'], (method, l, b, lr[b], o['iterations'])
            assert np.linalg.norm(lp[b] - o['pose']) <= 1e-9, (method, l, b)
            assert abs(int(lr[b, 2]) - o['k']) <= 2, (method, l, b, lr[b, 2], o['k'])
            assert abs(lr[b, 1] - o['rmse']) <= 1e-12 * o['rmse'], (method, l, b, lr[b, 1], o['rmse'])
    print(f'{method} per-level iterations: {levels[:, :, 3].cpu().numpy().astype(int).tolist()}')


@pytest.mark.parametrize('method', ['point_to_plane', 'colored'])
def test_batch_equals_one_call_per_pair_and_zero_level_is_single_level(method):
    pairs = coloured_pairs(seeds=(4011,))
    pose, res, levels, _ = run_pyramid(pairs, method)
    again = run_pyramid(pairs, method)
    assert torch.equal(pose, again[0]) and torch.equal(levels, again[2])
    for b, p in enumerate(pairs):
        p1, r1, l1, _ = run_pyramid([p], method)
        assert torch.equal(p1[0], pose[b]) and torch.equal(l1[0], levels[b]), b
    init = torch.from_numpy(np.stack([p[2] for p in pairs])).cuda()
    colors = ([p[3] for p in pairs], [p[4] for p in pairs]) if method == 'colored' else None
    src, tgt = [p[0] for p in pairs], [p[1] for p in pairs]
    a = E.icp_refine(src, tgt, init, RADIUS, 30, method, colors=colors)
    z = E.icp_refine(src, tgt, init, RADIUS, 30, method, colors=colors, voxels=[0], radii=[RADIUS])
    assert torch.equal(a[0], z[0]) and torch.equal(a[1], z[1])


def test_the_pyramid_recovers_the_perturbed_real_pair():
    s, t, gt, init = basin_case()
    x = torch.from_numpy(init[None]).cuda()
    one, _ = E.icp_refine([s], [t], x, BASIN['radius'], sum(BASIN['level_iters']), BASIN['method'])
    pyr, _, levels = E.icp_refine([s], [t], x, BASIN['radius'], 30, BASIN['method'], voxels=BASIN['voxels'],
                                  level_iters=BASIN['level_iters'], return_levels=True)
    want = M.multiscale_icp(s, t, init, BASIN['voxels'], None, BASIN['level_iters'], radius=BASIN['radius'],
                            method=BASIN['method'])
    assert not reached(one[0].cpu().numpy(), gt) and reached(pyr[0].cpu().numpy(), gt)
    assert np.abs(pyr[0].cpu().numpy() - want['pose']).max() <= 1e-6
    print(f'basin pair: per-level iterations {levels[0, :, 3].cpu().numpy().astype(int).tolist()}, oracle '
          f'{want["levels"][:, 3].astype(int).tolist()}')


def test_register_cli_with_a_pyramid(tmp_path):
    cfg, run = _checkpoint(tmp_path)
    src_file, tgt_file = os.path.join(REAL, 'modelnet_test_2_0.ply'), os.path.join(REAL, 'modelnet_test_2_1.ply')
    s, t = P.load_point_cloud(src_file), P.load_point_cloud(tgt_file)
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'pyr',
                         ['--icp', '0.03', '--icp_method', 'point_to_plane', '--icp_voxels', '0.08,0.04,0',
                          '--icp_level_iters', '20,10,5'])
    res = np.load(str(tmp_path / 'pyr' / 'result.npz'))
    sx, tx = R.crop(cfg, s), R.crop(cfg, t)
    pose, out, levels = E.icp_refine([sx], [tx], torch.from_numpy(res['pose_coarse'][None]).cuda(), 0.03, 30,
                                     'point_to_plane', voxels=[0.08, 0.04, 0.0], level_iters=[20, 10, 5],
                                     return_levels=True)
    assert np.array_equal(res['pose_icp'], pose[0].cpu().numpy()) and np.array_equal(res['icp'], out[0].cpu().numpy())
    assert np.array_equal(res['icp_levels'], levels[0].cpu().numpy())
    assert (line['icp_voxels'], line['icp_radii'], line['icp_level_iters']) == ([0.08, 0.04, 0.0], [0.08, 0.04, 0.03],
                                                                               [20, 10, 5])
    assert line['icp_levels'] == levels[0].cpu().numpy().tolist() and line['icp_iterations'] == int(out[0, 3])


def test_multiway_pairs_with_a_colored_pyramid(tmp_path):
    cfg, run = _checkpoint(tmp_path)
    model = R.load_model(cfg, str(run / 'ckpt' / 'model-best.pth'))
    s = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_0.ply'))
    t = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_1.ply'))
    u = perturb(np.eye(3, 4), 9, 5.0, 0.02)
    frags = [s, t, s @ u[:, :3].T + u[:, 3]]
    cols = [C.texture(f, 0.5) for f in frags]
    got = MW.register_pairs(model, frags, 2, 0.03, 30, 'colored', colors=cols, icp_lambda_geometric=0.95,
                            icp_voxels=[0.08, 0.04, 0.0], icp_level_iters=[10, 10, 5])
    coarse = MW.register_pairs(model, frags, 2)
    for p, (i, j) in enumerate(MW.all_pairs(3)):
        want, _ = E.icp_refine([frags[j]], [frags[i]], torch.from_numpy(coarse[p:p + 1]).cuda(), 0.03, 30, 'colored',
                               colors=([cols[j]], [cols[i]]), lambda_geometric=0.95, voxels=[0.08, 0.04, 0.0],
                               level_iters=[10, 10, 5])
        assert np.array_equal(got[p], want[0].cpu().numpy()), p
