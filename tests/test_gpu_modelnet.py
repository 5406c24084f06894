"""ModelNet40 training pairs on the device (regtr_modelnet_augment / modelnet.ModelNetPrep) against a float64 oracle
in the kernel's operation order and against the host restatement; the trainer's ModelNet branch; the benchmark
script's loop."""
import importlib.util
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import stats

from regtr_b200 import modelnet as MN
from regtr_b200 import ops
from regtr_b200 import trainer as T
from regtr_b200.config import get_config
from regtr_b200.regtr import RegTR
from regtr_b200.synthetic import make_modelnet_shapes
from regtr_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def shapes_on_device(n, seed, n_dup=0):
    return MN.ModelNetShapes.from_arrays(make_modelnet_shapes(n, seed=seed, n_dup=n_dup)).to(DEV)


# ------------------------------------------------------------------------------------------------ the oracle

def oracle_masks(raw, directions, k, gamma):
    """Crop masks in the kernel's order: float64 centroid (4 strided partial sums per thread over 512 threads, then a
    halving tree), fp32 centroid and differences, float64 distances ((x u0 + y u1) + z u2), the threshold between
    order statistics k and k + 1 with numpy's interpolation.  -> (masks (2, n) bool, distances, thresholds)."""
    n = len(raw)
    pad = np.zeros((2048, 3))
    pad[:n] = raw
    acc = ((pad[0:512] + pad[512:1024]) + pad[1024:1536]) + pad[1536:2048]
    h = 256
    while h:
        acc = acc[:h] + acc[h:2 * h]
        h //= 2
    c = (acc[0] / n).astype(np.float32)
    cen = (raw - c).astype(np.float64)
    masks, dists, thrs = [], [], []
    for u in directions:
        d = (cen[:, 0] * u[0] + cen[:, 1] * u[1]) + cen[:, 2] * u[2]
        if k < 0:
            thr = 0.0
        else:
            s = np.sort(d)
            diff = s[k + 1] - s[k]
            thr = s[k + 1] - diff * (1.0 - gamma) if gamma >= 0.5 else s[k] + diff * gamma
        masks.append(d > thr); dists.append(d); thrs.append(thr)
    return np.stack(masks), dists, thrs


def recover(out_pts, ref_pts):
    """Row index into ref_pts of every output row (nearest), and the distance."""
    d2 = ((out_pts[:, None, :].astype(np.float64) - ref_pts[None, :, :].astype(np.float64)) ** 2).sum(-1)
    i = d2.argmin(1)
    return i, np.sqrt(d2[np.arange(len(i)), i])


def transform64(m, x):
    """fp32 of the float64 rigid transform (((m0 x + m1 y) + m2 z) + m3)."""
    m = m.astype(np.float64); x = x.astype(np.float64)
    return np.stack([((m[a, 0] * x[:, 0] + m[a, 1] * x[:, 1]) + m[a, 2] * x[:, 2]) + m[a, 3] for a in range(3)],
                    1).astype(np.float32)


@pytest.mark.parametrize('partial', [[0.7, 0.7], [0.5, 0.5]])
def test_noise_free_pairs_against_the_float64_oracle(partial):
    sh = shapes_on_device(6, seed=3)
    cfg = get_config('modelnet', partial=partial)
    prep = MN.ModelNetPrep(cfg, sh, seed=9, noise=0.0)
    items = [0, 3, 5, 3, 1]
    out = prep(items, step=7)
    aug = out['aug']
    corr = out['correspondences']
    prep.check()
    assert torch.equal(out['pose'].cpu(), torch.from_numpy(aug['pose']))          # the host's pose, bit for bit
    host_pose = [MN.euler_transform(aug['euler'][b], aug['trans'][b], cfg.rot_mag)[1] for b in range(len(items))]
    assert np.array_equal(np.stack(host_pose), aug['pose'])
    margins = []
    for b, it in enumerate(items):
        raw = sh.points[it]
        masks, dists, thrs = oracle_masks(raw, aug['directions'][b], aug['k'], aug['gamma'])
        # the product host restatement (numpy's own mean / dot / percentile) on the same draws
        host = np.stack([MN.crop_mask(raw, np.float32(aug['p_keep']), aug['directions'][b][s]) for s in (0, 1)])
        if not np.array_equal(host, masks):
            for s in (0, 1):
                bad = np.nonzero(host[s] != masks[s])[0]
                margins += list(np.abs(dists[s][bad] - thrs[s]))
        src_clean = transform64(aug['transform'][b], raw)
        si, sd = recover(out['src_xyz'][b].cpu().numpy(), src_clean)
        ti, td = recover(out['tgt_xyz'][b].cpu().numpy(), raw)
        scale = np.abs(raw).max() + np.abs(src_clean).max()
        assert sd.max() <= 1e-6 * scale and td.max() <= 1e-6 * scale
        for idx, side in ((si, 0), (ti, 1)):
            assert len(np.unique(idx)) == MN.RESAMPLE_POINTS and masks[side][idx].all()
        assert np.array_equal(out['src_overlap'][b].cpu().numpy(), masks[1][si])
        assert np.array_equal(out['tgt_overlap'][b].cpu().numpy(), masks[0][ti])
        assert np.array_equal(corr[b].cpu().numpy(), MN.correspondences(si, ti, len(raw)))
        assert corr[b].dtype == torch.int64 and out['tgt_raw'][b].data_ptr() == sh.device_points[it].data_ptr()
    if margins:
        print('host / oracle mask differences at distance margins', margins)
    assert len(margins) <= 2


# ------------------------------------------------------------------------------------------------ distributions

def _launch(sh, params, step, noise):
    status = ops.new_status(DEV)
    items = torch.zeros(1, dtype=torch.int32, device=DEV)
    k, g = MN.percentile_position(sh.device_points.shape[1], np.float32(0.7))
    r = ops.modelnet_augment(sh.device_points, params, items, 21, step, k, g, noise, MN.JITTER_CLIP,
                             MN.RESAMPLE_POINTS, status)
    assert int(status.item()) == 0
    return r


def test_subset_is_uniform_and_jitter_is_the_clipped_normal():
    sh = shapes_on_device(1, seed=4)
    raw = sh.points[0]
    rng = np.random.default_rng(0)
    m, _ = MN.euler_transform(rng.random(3), rng.uniform(-0.5, 0.5, 3), 45.0)
    dirs = MN.sphere_direction(2 * np.pi * rng.random(2), 2 * rng.random(2) - 1)
    params = torch.from_numpy(np.concatenate([dirs.reshape(-1), m.reshape(-1).astype(np.float64)])[None]).to(DEV)
    masks = oracle_masks(raw, dirs, *MN.percentile_position(len(raw), np.float32(0.7)))[0]
    kept = np.nonzero(masks[1])[0]
    rank = np.full(len(raw), -1); rank[kept] = np.arange(len(kept))
    n_steps, nb = 300, 8
    table = np.zeros((nb, nb))
    noise = []
    for step in range(n_steps):
        xyz, _, _, _ = _launch(sh, params, step, 0.0)
        ti, _ = recover(xyz[1].cpu().numpy(), raw)
        np.add.at(table, (np.arange(len(ti)) * nb // len(ti), rank[ti] * nb // len(kept)), 1)
        if step < 20:
            jit, _, _, _ = _launch(sh, params, step, MN.JITTER_SCALE)
            noise.append((jit[1].cpu().double() - xyz[1].cpu().double()).numpy().ravel())
    # position bin x kept-rank bin: independent and uniform; every step fills each position bin equally
    assert table.sum() == n_steps * MN.RESAMPLE_POINTS and (rank[kept] >= 0).all()
    expected = np.outer(table.sum(1), table.sum(0)) / table.sum()
    chi2, p = stats.chisquare(table.ravel(), expected.ravel(), ddof=2 * (nb - 1))
    print('subset chi-square', chi2, 'p', p)
    assert p > 1e-3
    widths = np.bincount(np.arange(len(kept)) * nb // len(kept))      # every kept point equally likely
    assert stats.chisquare(table.sum(0), table.sum() * widths / len(kept)).pvalue > 1e-3
    noise = np.concatenate(noise)
    assert np.abs(noise).max() <= MN.JITTER_CLIP + 1e-6
    assert abs(noise.mean()) < 4 * 0.01 / np.sqrt(len(noise))
    assert abs(noise.std() / 0.01 - 1) < 0.02
    ks = stats.kstest(noise, stats.norm(0, 0.01).cdf)
    print('jitter KS', ks)
    assert ks.pvalue > 1e-3


# -------------------------------------------------------------------------------------------- determinism, cost

def _bytes(out, B):
    return [out[k][b].cpu().numpy().tobytes() for k in ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap')
            for b in range(B)] + [c.cpu().numpy().tobytes() for c in out['correspondences']] + \
        [out['pose'].cpu().numpy().tobytes()]


def test_batches_are_deterministic_and_pairs_independent():
    sh = shapes_on_device(5, seed=6, n_dup=8)
    cfg = get_config('modelnet')
    a = MN.ModelNetPrep(cfg, sh, seed=2)([4, 1, 2], step=11)
    b = MN.ModelNetPrep(cfg, sh, seed=2)([4, 1, 2], step=11)
    assert _bytes(a, 3) == _bytes(b, 3)
    alone = MN.ModelNetPrep(cfg, sh, seed=2)([4], step=11)
    others = MN.ModelNetPrep(cfg, sh, seed=2)([4, 3], step=11)
    pair0 = lambda o: [o[k][0].cpu().numpy().tobytes() for k in ('src_xyz', 'tgt_xyz', 'src_overlap')] + \
        [o['correspondences'][0].cpu().numpy().tobytes(), o['pose'][0].cpu().numpy().tobytes()]
    assert pair0(a) == pair0(alone) == pair0(others)
    c = MN.ModelNetPrep(cfg, sh, seed=2)([4, 1, 2], step=12)
    assert _bytes(a, 3) != _bytes(c, 3)


def test_one_launch_per_batch_and_bad_input_is_reported():
    sh = shapes_on_device(3, seed=7)
    prep = MN.ModelNetPrep(get_config('modelnet'), sh, seed=1)
    for B in (1, 4, 16):
        n0 = ops.LAUNCHES
        prep(list(np.arange(B) % 3))
        assert ops.LAUNCHES - n0 == 1
    prep.check()
    with pytest.raises(ValueError):
        prep([3])
    bad = make_modelnet_shapes(2, seed=8)
    bad[1, 5, 0] = np.nan
    prep = MN.ModelNetPrep(get_config('modelnet'), MN.ModelNetShapes.from_arrays(bad).to(DEV), seed=1)
    prep([0, 1])
    with pytest.raises(ValueError, match='not finite'):
        prep.check()


# ------------------------------------------------------------------------------------------------------ trainer

def make_opt(log_path, **kw):
    opt = SimpleNamespace(log_path=str(log_path), resume=None, debug=False, summary_every=1000,
                          validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=2)
    opt.__dict__.update(kw)
    return opt


def _run(tmp_path, name, niter, resume=None, validate_every=3, base_lr=1e-4):
    cfg = get_config('modelnet', train_batch_size=2, val_batch_size=2, base_lr=base_lr)
    train_set = MN.ModelNetShapes.from_arrays(make_modelnet_shapes(5, seed=30))
    val_set = MN.ModelNetPairs(MN.ModelNetShapes.from_arrays(make_modelnet_shapes(2, seed=31)), cfg)
    trainer = T.Trainer(make_opt(tmp_path / name, validate_every=validate_every, resume=resume), niter=niter,
                        grad_clip=cfg.grad_clip, seed=5)
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, 12), strict=True)
    trainer.fit(model, train_set, val_set)
    return model, trainer, str(tmp_path / name / 'ckpt')


def _state_equal(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a.cpu().reshape(-1).view(torch.uint8), b.cpu().reshape(-1).view(torch.uint8))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_state_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_state_equal(x, y) for x, y in zip(a, b))
    return a == b


def test_modelnet_trainer_resumes_exactly_and_validates_on_the_deterministic_pairs(tmp_path, monkeypatch):
    scores = []
    real = T.Trainer._run_validation

    def spy(self, model, val_set, step, **kw):
        assert isinstance(val_set, MN.ModelNetPairs)
        s = real(self, model, val_set, step, **kw)
        scores.append(s)
        return s
    monkeypatch.setattr(T.Trainer, '_run_validation', spy)
    _, _, ck_a = _run(tmp_path, 'a', niter=6)                  # 3 steps per epoch
    _, _, ck_b = _run(tmp_path, 'b', niter=3)
    _, _, ck_c = _run(tmp_path, 'c', niter=3, resume=os.path.join(ck_b, 'model-3.pth'))
    a = torch.load(os.path.join(ck_a, 'model-6.pth'))
    c = torch.load(os.path.join(ck_c, 'model-6.pth'))
    assert a['step'] == c['step'] == 6
    for k in ('state_dict', 'optimizer', 'scheduler', 'trainer'):
        assert _state_equal(a[k], c[k]), k
    assert a['trainer'] == dict(seed=5, steps_per_epoch=3, batch_size=2, dataset_len=5)
    # validations at steps 3 and 6 of run a, 3 of run b, 6 of run c: equal weights give equal scores
    assert len(scores) == 4 and all(0.0 <= s <= 1.0 for s in scores)
    assert scores[0] == scores[2] and scores[1] == scores[3]


def test_modelnet_training_loss_falls(tmp_path):
    cfg = get_config('modelnet', train_batch_size=4, base_lr=5e-4)
    train_set = MN.ModelNetShapes.from_arrays(make_modelnet_shapes(4, seed=40))
    trainer = T.Trainer(make_opt(tmp_path / 'log'), niter=24, grad_clip=cfg.grad_clip, seed=4)
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, 11), strict=True)
    totals = []
    real = model.compute_loss

    def record(pred, b):
        losses = real(pred, b)
        totals.append(losses['total'].detach())
        return losses
    model.compute_loss = record
    trainer.fit(model, train_set)
    totals = torch.stack(totals).cpu().numpy()
    print('training totals:', np.array2string(totals, precision=4))
    assert len(totals) == 24 and np.all(np.isfinite(totals))
    assert totals[-6:].mean() < totals[:6].mean()


# ----------------------------------------------------------------------------------------------------- evaluation

def test_eval_script_loop_end_to_end(tmp_path):
    spec = importlib.util.spec_from_file_location('eval_modelnet', os.path.join(ROOT, 'scripts', 'eval_modelnet.py'))
    ev = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ev)
    from regtr_b200 import eval as E
    from regtr_b200.regtr import GraphedRegTR
    cfg = get_config('modelnet')
    pairs = MN.ModelNetPairs(MN.ModelNetShapes.from_arrays(make_modelnet_shapes(3, seed=50)), cfg,
                             partial=ev.PARTIAL['ModelLoNet'])
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, 13), strict=True)
    model = model.to(DEV).eval()
    with torch.no_grad():
        summary, metrics, poses = ev.run_benchmark(GraphedRegTR(model), pairs, 1, str(tmp_path), DEV)
    saved = np.load(tmp_path / 'pred_transforms.npy')
    assert saved.shape == (3, 1, 3, 4) and np.array_equal(saved, poses)
    for i in range(3):
        batch = pairs.collate([i], DEV)
        data = {'points_src': torch.stack(batch['src_xyz']), 'points_ref': torch.stack(batch['tgt_xyz']),
                'points_raw': torch.stack(batch['tgt_raw']), 'transform_gt': batch['pose']}
        m = E.compute_modelnet_metrics(data, torch.from_numpy(saved[i]).to(DEV))
        for k in m:
            np.testing.assert_array_equal(metrics[k][i:i + 1], m[k])
    assert set(summary) == set(E.summarize_modelnet_metrics(metrics))
