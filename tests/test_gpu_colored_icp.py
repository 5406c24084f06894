"""Colour gradients (`ops.color_gradients`, regtr_color_gradients) and colored ICP (`ops.icp` with method='colored')
on the device against the float64 oracle (tests/colored_icp_oracle.py), on the real 3DMatch fixtures and on synthetic
3DMatch-shaped pairs.

No coloured scan exists among the fixtures, so every cloud is coloured procedurally (`colored_icp_oracle.texture`, a
smooth function of world position): the target as it lies and the source after its ground-truth pose, so that both
clouds of a pair agree where they overlap.  Only the real pairs with a benchmark ground-truth pose are used.

Covered: gradients at several max_nn, stacked and alone, reruns; the final pose, fitness, RMSE and iterations and the
state after 0..3 iterations with and without a robust kernel; batching and reruns; the launch count; lambda = 1 against
point-to-plane; the errors; `python -m regtr_b200.register --icp R --icp_method colored` end to end and `multiway`'s
pair registration with colored ICP on three fragments."""
import ctypes
import os

import numpy as np
import pytest
import torch

import colored_icp_oracle as C
from conftest import GOLDEN
from regtr_b200 import lib, ops
from regtr_b200 import eval as E
from regtr_b200 import multiway as MW
from regtr_b200 import pointio as P
from regtr_b200 import register as R
from test_gpu_icp import RADIUS, _run_register, perturb, synthetic_pairs
from test_gpu_register import gt_log_pair

pytestmark = pytest.mark.gpu
REAL = os.path.join(GOLDEN, 'real')
NR = 2.0 * RADIUS              # the normal radius and the gradient radius icp_refine uses
K_DIFF = []


def coloured_pairs(real=True, seeds=(4001, 4002)):
    """(src, tgt, init, src_rgb, tgt_rgb): the two real 3DMatch pairs with a gt.log pose and synthetic pairs, each
    starting from its ground truth perturbed."""
    out = []
    if real:
        for i, (fx, scene) in enumerate((('real_3dmatch_redkitchen_0_5', '7-scenes-redkitchen'),
                                         ('real_3dmatch_sun3d_hotel3_8_15', 'sun3d-hotel_umd-maryland_hotel3'))):
            s, t, p = gt_log_pair(fx, scene)
            out.append((s, t, perturb(p, 100 + i)) + C.colour_pair(s, t, p))
    from regtr_b200.synthetic import make_3dmatch_pair
    for seed, (s, t, init) in zip(seeds, synthetic_pairs(seeds)):
        gt = make_3dmatch_pair(seed)['pose']
        out.append((s, t, init) + C.colour_pair(s, t, gt))
    return out


def device_inputs(pairs):
    """Target normals and gradients on the device, as icp_refine makes them: -> (normals, gradients) lists."""
    tgts = [t for _, t, _, _, _ in pairs]
    normals = ops.estimate_normals(tgts, NR, 30)
    grads = ops.color_gradients(tgts, normals, [c for _, _, _, _, c in pairs], NR, 30)
    return normals, grads


def device_icp(pairs, normals, grads, max_iteration=30, **kw):
    return ops.icp([s for s, _, _, _, _ in pairs], [t for _, t, _, _, _ in pairs],
                   torch.from_numpy(np.stack([p for _, _, p, _, _ in pairs])).cuda(), RADIUS, max_iteration,
                   method='colored', tgt_normals=normals, src_colors=[c for _, _, _, c, _ in pairs],
                   tgt_colors=[c for _, _, _, _, c in pairs], tgt_color_gradients=grads, **kw)


def check_gradients(dev, xyz, normals, rgb, r, max_nn=30):
    want = C.color_gradients(xyz, normals, rgb, r, max_nn)
    err = np.abs(dev - want) / (1.0 + np.abs(want))
    assert err.max() <= 1e-9, err.max()
    return (want != 0).any(axis=1).mean()


def test_gradients_against_the_oracle():
    pairs = coloured_pairs()
    clouds = [t for _, t, _, _, _ in pairs] + [s for s, _, _, _, _ in pairs[:1]]
    rgbs = [c for _, _, _, _, c in pairs] + [c for _, _, _, c, _ in pairs[:1]]
    normals = ops.estimate_normals(clouds, NR, 30)
    grads = ops.color_gradients(clouds, normals, rgbs, NR, 30)
    for c, n, k, g in zip(clouds, normals, rgbs, grads):
        assert g.shape == c.shape and g.dtype == torch.float64
        share = check_gradients(g.cpu().numpy(), c, n.cpu().numpy(), k, NR)
        assert share > 0.9, share


def test_gradients_other_max_nn_and_stacking():
    pairs = coloured_pairs(seeds=(4003,))
    clouds = [pairs[0][1], pairs[2][0][:5001], pairs[1][1]]
    rgbs = [pairs[0][4], pairs[2][3][:5001], pairs[1][4]]
    normals = ops.estimate_normals(clouds, NR, 30)
    for max_nn in (1, 3, 4, 17, 64):
        out = ops.color_gradients(clouds, normals, rgbs, NR, max_nn)
        again = ops.color_gradients(clouds, normals, rgbs, NR, max_nn)
        for b, c in enumerate(clouds):
            assert torch.equal(again[b], out[b])
            alone = ops.color_gradients([c], [normals[b]], [rgbs[b]], NR, max_nn)
            assert torch.equal(alone[0], out[b]), (max_nn, b)
            if max_nn < 4:
                assert not out[b].any()
            elif max_nn in (4, 64) and b < 2:
                check_gradients(out[b].cpu().numpy(), c, normals[b].cpu().numpy(), rgbs[b], NR, max_nn)


def check_against_oracle(pose, res, pairs, normals, grads, max_iteration=30, **kw):
    pose, res = pose.cpu().numpy(), res.cpu().numpy()
    for b, (s, t, p, sc, tc) in enumerate(pairs):
        o = C.icp(s, t, normals[b].cpu().numpy(), sc, tc, grads[b].cpu().numpy(), p, RADIUS, max_iteration, **kw)
        rot_err = np.linalg.norm(pose[b, :, :3] - o['pose'][:, :3])
        trans_err = np.linalg.norm(pose[b, :, 3] - o['pose'][:, 3])
        assert rot_err <= 1e-9 and trans_err <= 1e-9, (b, rot_err, trans_err)
        assert int(res[b, 3]) == o['iterations'], (b, res[b], o['iterations'])
        K_DIFF.append(abs(int(res[b, 2]) - o['k']))
        assert abs(int(res[b, 2]) - o['k']) <= 2, (b, res[b, 2], o['k'])
        assert abs(res[b, 1] - o['rmse']) <= 1e-12 * o['rmse'], (b, res[b, 1], o['rmse'])
        assert res[b, 0] == res[b, 2] / len(s)
    return res


@pytest.mark.parametrize('kw', [{}, dict(loss='huber', loss_k=0.02), dict(loss='tukey', loss_k=0.05,
                                                                           lambda_geometric=0.5)])
def test_colored_icp_against_the_oracle(kw):
    pairs = coloured_pairs()
    normals, grads = device_inputs(pairs)
    pose, res = device_icp(pairs, normals, grads, **kw)
    assert pose.shape == (4, 3, 4) and pose.dtype == torch.float64 and res.shape == (4, 4)
    r = check_against_oracle(pose, res, pairs, normals, grads, **kw)
    assert (r[:2, 0] > 0.2).all()
    print(f'colored ICP {kw or "l2"} iterations: {r[:, 3].astype(int).tolist()}')


def test_state_after_each_of_the_first_iterations():
    pairs = coloured_pairs(seeds=(4003,))[:1] + coloured_pairs(False, (4003,))
    normals, grads = device_inputs(pairs)
    for it in range(4):
        for kw in ({}, dict(loss='cauchy', loss_k=0.03)):
            pose, res = device_icp(pairs, normals, grads, it, **kw)
            r = check_against_oracle(pose, res, pairs, normals, grads, it, **kw)
            assert (r[:, 3] == it).all()
            if it == 0:
                assert np.array_equal(pose.cpu().numpy(), np.stack([p for _, _, p, _, _ in pairs]))


def test_batch_equals_one_call_per_pair_and_reruns_are_identical():
    pairs = coloured_pairs(seeds=(4004,))
    syn = pairs[2]
    far = (syn[0][:3000], syn[1][:5000] + 40.0, syn[2], syn[3][:3000], syn[4][:5000])   # no correspondences
    cut = (pairs[1][0][:7001], pairs[1][1], pairs[1][2], pairs[1][3][:7001], pairs[1][4])
    batch = [pairs[0], far, cut, syn]
    normals, grads = device_inputs(batch)
    pose, res = device_icp(batch, normals, grads)
    again = device_icp(batch, normals, grads)
    assert torch.equal(pose, again[0]) and torch.equal(res, again[1])
    for b, pr in enumerate(batch):
        n1, g1 = device_inputs([pr])
        assert torch.equal(n1[0], normals[b]) and torch.equal(g1[0], grads[b])
        p1, r1 = device_icp([pr], n1, g1)
        assert torch.equal(p1[0], pose[b]) and torch.equal(r1[0], res[b]), b
    assert res[1].cpu().numpy().tolist() == [0.0, 0.0, 0.0, 1.0]


def test_launch_count():
    pairs = coloured_pairs(False, (4005,))
    normals, grads = device_inputs(pairs)
    before = ops.LAUNCHES
    ops.color_gradients([pairs[0][1]] * 3, normals * 3, [pairs[0][4]] * 3, NR)
    assert ops.LAUNCHES - before == ops.normals_launches()
    counts = []
    loose = dict(relative_fitness=1e-2, relative_rmse=1e-2)
    never = dict(relative_fitness=0.0, relative_rmse=0.0)
    for batch, kw, done_early in ((pairs, loose, True), (pairs * 8, loose, True), (pairs, never, False),
                                  (pairs * 8, never, False)):
        before = ops.LAUNCHES
        _, res = device_icp(batch, normals * (len(batch)), grads * len(batch), 30, **kw)
        torch.cuda.synchronize()
        counts.append(ops.LAUNCHES - before)
        iters = res[:, 3].cpu().numpy()
        assert (iters < 30).all() if done_early else (iters == 30).all(), iters
    assert counts == [ops.icp_launches(30)] * 4, counts


def test_lambda_one_reproduces_point_to_plane():
    """With lambda_geometric = 1 the geometric row is point-to-plane's own (sqrt(1) = 1 scales nothing) and the
    photometric row is zero, so the sums, the update and everything after are bit for bit point-to-plane's."""
    pairs = coloured_pairs(seeds=(4006,))
    normals, grads = device_inputs(pairs)
    init = torch.from_numpy(np.stack([p for _, _, p, _, _ in pairs])).cuda()
    plane = {}
    for kw in ({}, dict(loss='huber', loss_k=0.02)):
        a = device_icp(pairs, normals, grads, lambda_geometric=1.0, **kw)
        b = ops.icp([s for s, _, _, _, _ in pairs], [t for _, t, _, _, _ in pairs], init, RADIUS, 30,
                    method='point_to_plane', tgt_normals=normals, **kw)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), kw
        plane[kw.get('loss', 'l2')] = b[0]
    assert not torch.equal(device_icp(pairs, normals, grads)[0], plane['l2'])


def test_errors():
    pairs = coloured_pairs(False, (4007,))
    s, t, p, sc, tc = pairs[0]
    normals, grads = device_inputs(pairs)
    init = torch.from_numpy(p[None]).cuda()
    base = dict(method='colored', tgt_normals=normals, src_colors=[sc], tgt_colors=[tc], tgt_color_gradients=grads)
    for drop in ('tgt_normals', 'src_colors', 'tgt_colors', 'tgt_color_gradients'):
        kw = dict(base)
        del kw[drop]
        with pytest.raises(ValueError):
            ops.icp([s], [t], init, RADIUS, **kw)
    for name, bad in (('src_colors', [sc[:-1]]), ('tgt_colors', [tc[:, :2]]), ('tgt_color_gradients', [grads[0][1:]]),
                      ('tgt_normals', [normals[0][1:]]), ('src_colors', [sc, sc])):
        with pytest.raises(ValueError):
            ops.icp([s], [t], init, RADIUS, **dict(base, **{name: bad}))
    for lam in (-0.01, 1.01, float('nan')):
        with pytest.raises(ValueError, match='lambda_geometric'):
            ops.icp([s], [t], init, RADIUS, lambda_geometric=lam, **base)
    with pytest.raises(ValueError):
        ops.color_gradients([t], normals, [tc[1:]], NR)
    with pytest.raises(ValueError):
        ops.color_gradients([t], normals, [tc], NR, max_nn=65)
    bound = ops.overlap_coord_bound(NR)
    far = np.array([[0.0, 0.0, 0.0], [bound * 1.001, 0.0, 0.0]])
    with pytest.raises(lib.RegtrLibError, match='color_gradients: a coordinate'):
        ops.color_gradients([far], [np.zeros((2, 3))], [np.zeros((2, 3))], NR)
    # the C entry point refuses inconsistent colour options
    L = lib.load()
    opt = ops.IcpOptions(0, 1.0, 1e-3)
    opt.tgt_colors = grads[0].data_ptr()
    dev = torch.device('cuda')
    xyz, offs, lens = ops._stack_pairs([s], [t], 'icp', dev)
    n = sum(lens)
    ws = ops.workspace(L.regtr_icp_ws_bytes(n, 1), dev)
    state = ops.workspace(L.regtr_icp_state_bytes(n), dev, 'scan_state', zero=True)
    pose = torch.empty((1, 3, 4), dtype=torch.float64, device=dev)
    out = torch.empty((1, 4), dtype=torch.float64, device=dev)
    status = ops.new_status(dev)
    nrm = normals[0].contiguous()

    def call(o):
        return L.regtr_icp(xyz.data_ptr(), offs.data_ptr(), 1, n, init.data_ptr(), RADIUS, ops.overlap_cell(RADIUS),
                           3, 1e-6, 1e-6, nrm.data_ptr(), None, ctypes.addressof(o), pose.data_ptr(), out.data_ptr(),
                           status.data_ptr(), ws.data_ptr(), ws.numel(), state.data_ptr(), state.numel(), None)
    assert call(opt) != 0                                           # target colours without source colours
    opt = ops.IcpOptions(0, 1.0, 1e-3)
    col = torch.from_numpy(np.concatenate([sc, tc])).cuda()
    opt.src_colors, opt.tgt_colors, opt.tgt_color_gradients = col.data_ptr(), col.data_ptr(), grads[0].data_ptr()
    opt.lambda_geometric = 1.5
    assert call(opt) != 0
    opt.lambda_geometric = 0.5
    assert call(opt) == 0
    torch.cuda.synchronize()


def test_report_largest_k_difference():
    print(f'largest |k_device - k_oracle|: {max(K_DIFF) if K_DIFF else "n/a"}')
    assert not K_DIFF or max(K_DIFF) <= 2


def _checkpoint(tmp_path):
    from regtr_b200.config import get_config
    from regtr_b200.train import write_config
    from regtr_b200.weights import random_state_dict
    cfg = get_config('modelnet')
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    torch.save({'state_dict': random_state_dict(cfg, 43), 'step': 1}, str(run / 'ckpt' / 'model-best.pth'))
    write_config(cfg, 'modelnet', str(run / 'config.yaml'))
    return cfg, run


def test_register_cli_with_colored_icp(tmp_path):
    cfg, run = _checkpoint(tmp_path)
    s = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_0.ply'))
    t = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_1.ply'))
    src_file, tgt_file = str(tmp_path / 'src.ply'), str(tmp_path / 'tgt.ply')
    P.write_ply(src_file, s, colors=C.texture(s, 0.5))
    P.write_ply(tgt_file, t, colors=C.texture(t, 0.5))
    radius = 0.05
    line = _run_register(tmp_path, run, src_file, tgt_file, tmp_path / 'col',
                         ['--icp', str(radius), '--icp_method', 'colored', '--icp_lambda_geometric', '0.9'])
    res = np.load(str(tmp_path / 'col' / 'result.npz'))
    coarse = res['pose'][-1]
    _, sc = P.load_point_cloud_colors(src_file)
    _, tc = P.load_point_cloud_colors(tgt_file)
    sx, tx = R.crop(cfg, s), R.crop(cfg, t)
    sc, tc = R.crop_colors(cfg, s, sc), R.crop_colors(cfg, t, tc)
    normals = ops.estimate_normals([tx], 2.0 * radius, 30)
    grads = ops.color_gradients([tx], normals, [tc], 2.0 * radius, 30)
    pose, out = ops.icp([sx], [tx], torch.from_numpy(coarse[None]).cuda(), radius, 30, method='colored',
                        tgt_normals=normals, src_colors=[sc], tgt_colors=[tc], tgt_color_gradients=grads,
                        lambda_geometric=0.9)
    pose, out = pose[0].cpu().numpy(), out[0].cpu().numpy()
    assert np.array_equal(res['pose_icp'], pose) and np.array_equal(res['icp'], out)
    assert (line['icp_method'], line['icp_lambda_geometric'], line['icp_iterations']) == ('colored', 0.9, int(out[3]))
    assert open(tmp_path / 'col' / 'pose.txt').read() == R.pose_text(pose)


def test_multiway_pairs_with_colored_icp(tmp_path):
    """Three fragments: every pair's colored ICP equals icp_refine on the network's pose with the fragments'
    colours."""
    cfg, run = _checkpoint(tmp_path)
    model = R.load_model(cfg, str(run / 'ckpt' / 'model-best.pth'))
    s = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_0.ply'))
    t = P.load_point_cloud(os.path.join(REAL, 'modelnet_test_2_1.ply'))
    u = perturb(np.eye(3, 4), 9, 5.0, 0.02)
    frags = [s, t, s @ u[:, :3].T + u[:, 3]]
    cols = [C.texture(f, 0.5) for f in frags]
    radius = 0.05
    got = MW.register_pairs(model, frags, 2, radius, 30, 'colored', colors=cols, icp_lambda_geometric=0.95)
    coarse = MW.register_pairs(model, frags, 2)
    for p, (i, j) in enumerate(MW.all_pairs(3)):
        want, _ = E.icp_refine([frags[j]], [frags[i]], torch.from_numpy(coarse[p:p + 1]).cuda(), radius, 30,
                               'colored', colors=([cols[j]], [cols[i]]), lambda_geometric=0.95)
        assert np.array_equal(got[p], want[0].cpu().numpy()), p
