"""The training loop on the device (regtr_b200.trainer): the meter and pose-error kernels against the float64 oracle,
the whole loop against the hand-written training sequence, exact resume, checkpoints that the evaluation loads, faults
inside a step, the cost of a loop step over a bare step, and a falling training loss.  Data: synthetic 3DMatch-format
pairs written to tmp_path and the two real pairs of tests/golden/real."""
import logging
import math
import os
import pickle
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

import train_data_oracle as DO
import trainer_oracle as O
from regtr_b200 import augment as A
from regtr_b200 import data as D
from regtr_b200 import ops
from regtr_b200 import trainer as T
from regtr_b200.config import get_config
from regtr_b200.regtr import RegTR
from regtr_b200.synthetic import make_3dmatch_pair
from regtr_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
DEV = torch.device('cuda', 0)


# --------------------------------------------------------------------------------------------------- helpers

def write_synthetic(root, n_train, n_val, n_pts=4000, seed=0):
    """A 3DMatch-format dataset: <root>/<phase>/scene/cloud_bin_<i>.pth (float64 ndarrays) and <phase>_info.pkl."""
    for phase, n in (('train', n_train), ('val', n_val)):
        infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
        os.makedirs(os.path.join(root, phase, 'scene'), exist_ok=True)
        for i in range(n):
            p = make_3dmatch_pair(seed + 1000 * (phase == 'val') + i, n_target=n_pts)
            rels = [f'{phase}/scene/cloud_bin_{2 * i}.pth', f'{phase}/scene/cloud_bin_{2 * i + 1}.pth']
            for rel, x in zip(rels, (p['src_xyz'], p['tgt_xyz'])):
                torch.save(np.asarray(x, np.float64), os.path.join(root, rel))
            pose = np.asarray(p['pose'], np.float64)
            infos['rot'].append(pose[:, :3]); infos['trans'].append(pose[:, 3:])
            infos['src'].append(rels[0]); infos['tgt'].append(rels[1]); infos['overlap'].append(0.5)
        with open(os.path.join(root, f'{phase}_info.pkl'), 'wb') as f:
            pickle.dump(infos, f)
    return str(root)


def datasets(root):
    return (D.ThreeDMatchPairs(root, os.path.join(root, 'train_info.pkl'), pin=True, float64=True),
            D.ThreeDMatchPairs(root, os.path.join(root, 'val_info.pkl'), pin=True, float64=True))


def write_real(root):
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    for s, t, p, row in DO.real_pairs(GOLDEN):
        for rel, x in ((row['src'], s), (row['tgt'], t)):
            os.makedirs(os.path.join(root, os.path.dirname(rel)), exist_ok=True)
            torch.save(x, os.path.join(root, rel))
        infos['rot'].append(p[:, :3]); infos['trans'].append(p[:, 3:])
        infos['src'].append(row['src']); infos['tgt'].append(row['tgt']); infos['overlap'].append(row['overlap'])
    with open(os.path.join(root, 'info.pkl'), 'wb') as f:
        pickle.dump(infos, f)
    return D.ThreeDMatchPairs(str(root), os.path.join(root, 'info.pkl'), pin=True, float64=True)


def make_opt(log_path, **kw):
    opt = SimpleNamespace(log_path=str(log_path), resume=None, debug=False, summary_every=1000,
                          validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=2)
    opt.__dict__.update(kw)
    return opt


def make_model(cfg, seed=11):
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, seed), strict=True)
    return model


def state_equal(a, b):
    """Nested states equal, tensors bit for bit (NaN included)."""
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and \
            torch.equal(a.cpu().reshape(-1).view(torch.uint8), b.cpu().reshape(-1).view(torch.uint8))
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(state_equal(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(state_equal(x, y) for x, y in zip(a, b))
    return a == b


def same_bits(dev_vals, ref_vals):
    """Equal bit for bit, NaN payloads aside (the GPU's default NaN is not the x86 one)."""
    a = np.asarray(dev_vals, np.float64).ravel()
    b = np.asarray(ref_vals, np.float64).ravel()
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64))


@pytest.fixture
def no_sync():
    torch.cuda.set_sync_debug_mode('error')
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---------------------------------------------------------------------------------------------- meter kernel

SEQS = [
    [1.5, 2.25, float('nan'), 0.1, 3.0, 1e30, -7.0],
    [float('nan'), 1.0, 2.0, float('inf'), 4.0],
    [float('inf'), 1.0, float('-inf'), 3.0, float('nan')],
    list(np.random.default_rng(1).standard_normal(200).astype(np.float32) * 13.0),
]


@pytest.mark.parametrize('seq', range(len(SEQS)))
def test_meter_update_is_bit_identical_to_the_oracle(seq):
    totals = [float(np.float32(v)) for v in SEQS[seq]]
    other = [float(np.float32(v * 0.37 + 1.0)) for v in totals]
    banks = [torch.zeros((2, 4), dtype=torch.float64, device=DEV) for _ in range(2)]
    smooth = torch.zeros(2, dtype=torch.float64, device=DEV)
    log = torch.zeros(1 + 3, dtype=torch.int64, device=DEV)
    ref = [[O.Meter(), O.Meter()] for _ in range(2)]
    ema = O.Smooth()
    clear_at = len(totals) // 2
    for step, (t, o) in enumerate(zip(totals, other), 1):
        if step == clear_at:                         # the second bank is cleared mid-way (a summary)
            banks[1].zero_()
            ref[1] = [O.Meter(), O.Meter()]
        vals = [torch.tensor(o, dtype=torch.float32, device=DEV), torch.tensor(t, dtype=torch.float32, device=DEV)]
        ops.meter_update(vals, banks, step, total_key=1, smooth=smooth, log=log)
        for r in ref:
            r[0].update(o); r[1].update(t)
        ema.update(t, step)
    for bank, r in zip(banks, ref):
        assert same_bits(bank.cpu().numpy(), [m.row() for m in r])
    v, is_set = smooth.cpu().tolist()
    assert is_set == 1.0 and same_bits([v], [ema.value])
    lg = log.cpu().tolist()
    assert lg[0] == len(ema.skipped) and lg[1:1 + min(3, lg[0])] == ema.skipped[:3]


def test_meter_update_is_one_launch_without_sync(no_sync):
    banks = [torch.zeros((3, 4), dtype=torch.float64, device=DEV) for _ in range(2)]
    smooth = torch.zeros(2, dtype=torch.float64, device=DEV)
    log = torch.zeros(5, dtype=torch.int64, device=DEV)
    vals = [torch.full((), float(i), device=DEV) for i in range(3)]
    n0 = ops.LAUNCHES
    ops.meter_update(vals, banks, 7, total_key=2, smooth=smooth, log=log)
    assert ops.LAUNCHES - n0 == 1
    ops.meter_update(vals, banks[:1], 8)
    assert ops.LAUNCHES - n0 == 2


# ----------------------------------------------------------------------------------------- pose-error kernel

def _poses(rng, L, B, angles_deg, trans_scale):
    gt = np.zeros((B, 3, 4), np.float32)
    pred = np.zeros((L, B, 3, 4), np.float32)
    for b in range(B):
        R = Rotation.random(random_state=int(rng.integers(1 << 30))).as_matrix()
        t = rng.normal(size=3) * 2.0
        gt[b] = np.concatenate([R, t[:, None]], 1)
        for l in range(L):
            ang = angles_deg[(l * B + b) % len(angles_deg)]
            d = Rotation.from_rotvec(np.deg2rad(ang) * Rotation.random(random_state=int(rng.integers(1 << 30)))
                                     .apply([1.0, 0.0, 0.0])).as_matrix()
            pred[l, b, :, :3] = d @ R
            pred[l, b, :, 3] = t + rng.normal(size=3) * trans_scale[(l + b) % len(trans_scale)]
    return pred, gt


def _run_pose_errors(pred, gt, chunks, thr=(10.0, 0.1)):
    L, B = pred.shape[:2]
    hist = torch.zeros((2, L, B), dtype=torch.float64, device=DEV)
    acc = torch.zeros((L, 4), dtype=torch.float64, device=DEV)
    off = 0
    for c in chunks:
        p = torch.from_numpy(np.ascontiguousarray(pred[:, off:off + c])).to(DEV)
        g = torch.from_numpy(np.ascontiguousarray(gt[off:off + c])).to(DEV)
        ops.pose_errors(p, g, hist[0], hist[1], acc, off, *thr)
        off += c
    return hist.cpu().numpy(), acc.cpu().numpy()


def test_pose_errors_against_float64_and_fp32_se3_compare(no_sync):
    from regtr_b200.eval import se3_compare
    rng = np.random.default_rng(3)
    pred, gt = _poses(rng, 6, 11, [0.0, 1e-3, 0.5, 3.0, 45.0, 120.0, 179.0, 179.99], [0.0, 1e-3, 0.05, 0.5])
    torch.cuda.set_sync_debug_mode(0)
    hist, acc = _run_pose_errors(pred, gt, [4, 5, 2])
    rot, trans = O.pose_errors(pred, gt)
    assert np.max(np.abs(hist[0] - rot)) <= 1e-9 and np.max(np.abs(hist[1] - trans)) <= 1e-9
    # fp32 se3_compare: its cosine carries up to DELTA of fp32 rounding (unit-norm rows: three 3-term dot products,
    # a sum and a scaling), and acos turns an error d of the cosine x into at most d / sqrt(1 - (|x| + d)^2), and
    # never more than 2 sqrt(d) (its slope blows up at +-1)
    DELTA = 2e-6
    ref = se3_compare(torch.from_numpy(pred).to(DEV), torch.from_numpy(gt).to(DEV)[None])
    r32, t32 = ref['rot_deg'].cpu().numpy().astype(np.float64), ref['trans'].cpu().numpy().astype(np.float64)
    x = np.abs(np.cos(np.deg2rad(rot)))
    room = 1.0 - np.minimum(x + DELTA, 1.0) ** 2
    slope_bound = np.where(room > 0, DELTA / np.sqrt(np.maximum(room, 1e-300)), np.inf)
    bound = np.degrees(np.minimum(slope_bound, 2.0 * np.sqrt(DELTA)))
    assert np.all(np.abs(r32 - rot) <= bound)
    assert np.all(np.abs(t32 - trans) <= 1e-5 * (1.0 + np.abs(trans) + np.abs(gt[None, :, :, 3]).sum(-1)))


def test_pose_errors_identity_180_success_and_reruns():
    gt = np.tile(np.eye(3, 4, dtype=np.float32), (2, 1, 1))
    gt[1, :, 3] = [0.5, -1.0, 2.0]
    pred = np.tile(gt[None], (2, 1, 1, 1))
    pred[1, :, :, :3] = np.diag([1.0, -1.0, -1.0]).astype(np.float32)     # 180 degrees about x
    pred[1, 1, :, 3] = np.diag([1.0, -1.0, -1.0]) @ gt[1, :, 3]            # translation error 0 for that pair
    hist, acc = _run_pose_errors(pred, gt, [2])
    assert np.all(hist[:, 0] == 0.0)                                        # identity: exactly 0 and 0
    assert np.all(np.abs(hist[0, 1] - 180.0) <= 1e-12) and hist[1, 1, 1] == 0.0
    # n_success away from the thresholds (rot 10 deg, trans 0.1): exact, and every run is bit-identical
    rng = np.random.default_rng(5)
    pred, gt = _poses(rng, 6, 40, [0.5, 3.0, 8.0, 12.0, 30.0], [0.0, 0.03, 0.2])
    rot, trans = O.pose_errors(pred, gt)
    assert np.min(np.abs(rot - 10.0)) > 1e-6 and np.min(np.abs(trans - 0.1)) > 1e-6     # far beyond the 1e-9 error
    runs = [_run_pose_errors(pred, gt, [7, 13, 20]) for _ in range(3)]
    ok = (rot < 10.0) & (trans < 0.1)
    assert np.array_equal(runs[0][1][:, 2], ok.sum(1).astype(np.float64)) and np.all(runs[0][1][:, 3] == 40)
    assert 0 < ok.sum() < ok.size
    for h, a in runs[1:]:
        assert np.array_equal(h.view(np.int64), runs[0][0].view(np.int64))
        assert np.array_equal(a.view(np.int64), runs[0][1].view(np.int64))
    assert np.max(np.abs(runs[0][1][:, 0] - rot.sum(1))) <= 1e-9 * 40


# ------------------------------------------------------------------------------------------------ whole loop

def _hand_written(cfg, ds, order, seed, n_steps):
    """test_end_to_end_training_step_on_real_pairs' sequence, plus StepLR.step(): (model, optimizer, scheduler,
    per-step loss values)."""
    from regtr_b200 import optim
    model = make_model(cfg).cuda()
    opt, sched = model.configure_optimizers()
    prep = A.TrainingPrep(cfg, seed=seed)
    vals = []
    for batch in D.PairStream(ds, order[:n_steps], workers=2):
        b = prep(batch)
        loss = model.compute_loss(model.forward_train(b, train_encoder=True), b)
        opt.zero_grad(set_to_none=True)
        loss['total'].backward()
        optim.clip_grad_norm_(model.parameters(), cfg.grad_clip)
        opt.step()
        sched.step()
        vals.append({k: v.item() for k, v in loss.items()})
    prep.check()
    return model, opt, sched, vals


def test_trainer_equals_the_hand_written_sequence_on_real_pairs(tmp_path):
    ds = write_real(tmp_path / 'data')
    cfg = get_config('3dmatch', scheduler_param=[2, 0.5])
    n_steps, seed = 3, 21
    trainer = T.Trainer(make_opt(tmp_path / 'log'), niter=n_steps, grad_clip=cfg.grad_clip, seed=seed)
    model = make_model(cfg)
    trainer.fit(model, ds)
    order = [b for e in range(n_steps) for b in T.epoch_batches(seed, e, len(ds), cfg.train_batch_size)]
    ref_model, ref_opt, ref_sched, vals = _hand_written(cfg, ds, order, seed, n_steps)
    assert state_equal(model.state_dict(), ref_model.state_dict())
    assert state_equal(model.optimizer.state_dict(), ref_opt.state_dict())
    assert state_equal(model.scheduler.state_dict(), ref_sched.state_dict())
    assert model.scheduler.get_last_lr()[0] == cfg.base_lr * 0.5
    # the meters: the summary meter holds steps 2.. (cleared by the summary of step 1), the EMA all steps
    ema, meters = O.Smooth(), {k: O.Meter() for k in vals[0]}
    for step, v in enumerate(vals, 1):
        ema.update(v['total'], step)
        if step > 1:
            for k in v:
                meters[k].update(v[k])
    got = trainer.summary_meter.stats.cpu().numpy()
    assert same_bits(got, [meters[k].row() for k in trainer.summary_meter.keys])
    assert same_bits([trainer.loss_smooth()], [ema.value])


def _run(tmp_path, name, data, niter, resume=None, validate_every=3):
    cfg = get_config('3dmatch', train_batch_size=2, val_batch_size=2)
    train_set, val_set = datasets(data)
    log = tmp_path / name
    trainer = T.Trainer(make_opt(log, validate_every=validate_every, resume=resume), niter=niter,
                        grad_clip=cfg.grad_clip, seed=5)
    model = make_model(cfg, seed=12)
    trainer.fit(model, train_set, val_set)
    return model, str(log / 'ckpt')


def test_exact_resume_and_checkpoints(tmp_path):
    data = write_synthetic(tmp_path / 'data', n_train=7, n_val=2)        # 4 steps per epoch, the last one partial
    model_a, ck_a = _run(tmp_path, 'a', data, niter=6)
    _, ck_b = _run(tmp_path, 'b', data, niter=3)
    _, ck_c = _run(tmp_path, 'c', data, niter=3, resume=os.path.join(ck_b, 'model-3.pth'))
    a = torch.load(os.path.join(ck_a, 'model-6.pth'))
    c = torch.load(os.path.join(ck_c, 'model-6.pth'))
    assert a['step'] == c['step'] == 6
    for k in ('state_dict', 'optimizer', 'scheduler', 'trainer'):
        assert state_equal(a[k], c[k]), k
    assert a['trainer'] == dict(seed=5, steps_per_epoch=4, batch_size=2, dataset_len=7)
    assert state_equal(torch.load(os.path.join(ck_a, 'model-3.pth'))['state_dict'],
                       torch.load(os.path.join(ck_b, 'model-3.pth'))['state_dict'])
    # the manager's files: both checkpoints kept, the best named first
    assert sorted(os.listdir(ck_a)) == ['checkpoints.txt', 'model-3.pth', 'model-6.pth']
    lines = open(os.path.join(ck_a, 'checkpoints.txt')).read().split('\n')
    assert lines[0] in ('Best step: 3', 'Best step: 6') and lines[1:] == ['model-3.pth', 'model-6.pth']
    assert sorted(os.listdir(ck_c)) == ['checkpoints.txt', 'model-6.pth']
    # the best checkpoint loads strictly into a fresh RegTR, as scripts/eval_3dmatch.py loads it; the checkpoint of
    # the last step reproduces the trained model's forward bit for bit
    cfg = model_a.cfg
    best = int(lines[0].split(':')[1])
    fresh = RegTR(cfg)
    fresh.load_state_dict(torch.load(os.path.join(ck_a, f'model-{best}.pth'), map_location='cpu')['state_dict'],
                          strict=True)
    fresh = RegTR(cfg).to(DEV)
    fresh.load_state_dict(a['state_dict'], strict=True)
    fresh.eval(); model_a.eval()
    _, val_set = datasets(data)
    batch = A.TrainingPrep(cfg)(D.collate_pair([val_set[0], val_set[1]]), augment=False)
    o1 = fresh({'src_xyz': batch['src_xyz'], 'tgt_xyz': batch['tgt_xyz']})
    o2 = model_a({'src_xyz': batch['src_xyz'], 'tgt_xyz': batch['tgt_xyz']})
    assert torch.equal(o1['pose'], o2['pose'])
    assert all(torch.equal(x, y) for x, y in zip(o1['src_feat'], o2['src_feat']))


# ---------------------------------------------------------------------------------------------------- faults

def test_detached_nan_total_is_skipped_and_named(tmp_path, caplog):
    data = write_synthetic(tmp_path / 'data', n_train=3, n_val=0)
    train_set, _ = datasets(data)
    cfg = get_config('3dmatch', train_batch_size=1)
    trainer = T.Trainer(make_opt(tmp_path / 'log'), niter=3, grad_clip=cfg.grad_clip, seed=1)
    model = make_model(cfg)
    trainer.setup(model, train_set)
    real = model.compute_loss
    totals = []

    def nan_at_step_2(pred, b):
        losses = real(pred, b)
        if b['aug']['step'] == 1:
            losses = {k: v.detach() for k, v in losses.items()}
            losses['total'] = torch.full((), float('nan'), device=DEV)
        totals.append(losses['total'].item())
        return losses
    model.compute_loss = nan_at_step_2
    batches = [D.collate_pair([train_set[i]]) for i in range(3)]
    snap = None
    for step, batch in enumerate(batches, 1):
        if step == 2:
            snap = {k: v.clone() for k, v in model.state_dict().items()}
            opt_steps = [float(s['step']) for s in model.optimizer.state.values()]
            last_epoch = model.scheduler.last_epoch
        trainer.training_step(model, batch, step)
        if step == 2:
            assert state_equal(snap, model.state_dict())
            assert [float(s['step']) for s in model.optimizer.state.values()] == opt_steps
            assert model.scheduler.last_epoch == last_epoch
            assert all(p.grad is None for p in model.parameters())      # zero_grad ran, no backward
    ema = O.Smooth()
    for step, v in enumerate(totals, 1):
        ema.update(v, step)
    assert ema.skipped == [2] and same_bits([trainer.loss_smooth()], [ema.value])
    with caplog.at_level(logging.WARNING, logger='regtr_b200.trainer'):
        trainer.report_nonfinite()
    msgs = [r.getMessage() for r in caplog.records if 'not finite' in r.getMessage()]
    assert len(msgs) == 1 and 'Instance [1]' in msgs[0] and 'cloud_bin_2.pth' in msgs[0] and '(step 2)' in msgs[0]
    trainer.close()


def test_a_raising_step_is_logged_and_the_loop_goes_on(tmp_path, caplog):
    data = write_synthetic(tmp_path / 'data', n_train=3, n_val=1)
    train_set, val_set = datasets(data)
    cfg = get_config('3dmatch', train_batch_size=1, val_batch_size=1)
    trainer = T.Trainer(make_opt(tmp_path / 'log', validate_every=3), niter=3, grad_clip=cfg.grad_clip, seed=2)
    model = make_model(cfg)
    real, calls = model.forward_train, []

    def raise_second(batch, train_encoder=False):
        calls.append(1)
        if len(calls) == 2:
            raise RuntimeError('injected fault')
        return real(batch, train_encoder=train_encoder)
    model.forward_train = raise_second
    with caplog.at_level(logging.ERROR, logger='regtr_b200.trainer'):
        trainer.fit(model, train_set, val_set)
    errs = [r.getMessage() for r in caplog.records if 'injected fault' in r.getMessage()]
    assert len(errs) == 1 and 'Instance [' in errs[0]
    ck = torch.load(tmp_path / 'log' / 'ckpt' / 'model-3.pth')
    assert ck['step'] == 3 and len(calls) == 3
    assert {float(s['step']) for s in ck['optimizer']['state'].values()} == {2.0}


# ------------------------------------------------------------------------------------------------------ cost

def test_a_loop_step_costs_one_launch_and_no_sync_over_the_bare_step(tmp_path):
    from regtr_b200 import optim
    data = write_synthetic(tmp_path / 'data', n_train=2, n_val=0)
    train_set, _ = datasets(data)
    cfg = get_config('3dmatch', train_batch_size=2)
    trainer = T.Trainer(make_opt(tmp_path / 'log'), niter=10, grad_clip=cfg.grad_clip, seed=3)
    model = make_model(cfg)
    trainer.setup(model, train_set)
    batch = D.collate_pair([train_set[0], train_set[1]])

    def bare(step):
        trainer.prep.step = step - 1
        b = trainer.prep(batch)
        losses = model.compute_loss(model.forward_train(b, train_encoder=True), b)
        model.optimizer.zero_grad()
        losses['total'].backward()
        optim.clip_grad_norm_(model.parameters(), max_norm=cfg.grad_clip)
        model.optimizer.step()
        model.scheduler.step()

    def measure(fn):
        torch.cuda.synchronize()
        n0 = ops.LAUNCHES
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter('always')
            torch.cuda.set_sync_debug_mode('warn')
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        return ops.LAUNCHES - n0, sum('synchroniz' in str(x.message) for x in w)

    trainer.training_step(model, batch, 1)                 # creates the meters and the optimizer state
    bare(2)
    l_bare, s_bare = measure(lambda: bare(3))
    l_loop, s_loop = measure(lambda: trainer.training_step(model, batch, 3))
    assert l_loop == l_bare + 1, (l_loop, l_bare)
    assert s_loop == s_bare, (s_loop, s_bare)
    trainer.close()


# ------------------------------------------------------------------------------------------------- learning

def test_training_loss_falls(tmp_path):
    """Deterministic: 4 synthetic pairs of ~4000 points, batches of 2, AdamW at lr 5e-4 (10x the reference's
    0.0001, so that a few steps show the trend), 24 steps; the mean total of the last 6 steps is below that of the
    first 6."""
    data = write_synthetic(tmp_path / 'data', n_train=4, n_val=0, seed=40)
    train_set, _ = datasets(data)
    cfg = get_config('3dmatch', train_batch_size=2, base_lr=5e-4)
    trainer = T.Trainer(make_opt(tmp_path / 'log'), niter=24, grad_clip=cfg.grad_clip, seed=4)
    model = make_model(cfg)
    totals = []
    real = model.compute_loss

    def record(pred, b):
        losses = real(pred, b)
        totals.append(losses['total'].detach())
        return losses
    model.compute_loss = record
    trainer.fit(model, train_set)
    totals = torch.stack(totals).cpu().numpy()
    assert len(totals) == 24 and np.all(np.isfinite(totals))
    print('training totals:', np.array2string(totals, precision=4))
    assert totals[-6:].mean() < totals[:6].mean()
