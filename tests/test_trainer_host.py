"""CPU tests of the training loop (regtr_b200.trainer, regtr_b200.train): the float64 meter / EMA oracle against the
reference's AverageMeter and loss_smooth rule, CheckpointManager against the reference's CheckPointManager (files,
checkpoints.txt bytes, loading both ways), the epoch sampler and the step conversions, the log strings, the builtin
3dmatch config's dataset keys, the CLI's config recovery, and the C struct layouts of the bookkeeping kernels."""
import math
import os
import re
import shutil
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import trainer_oracle as O
from oracle import ref_bridge
from regtr_b200 import trainer as T

needs_ref = pytest.mark.skipif(not ref_bridge.available(), reason='the reference tree is not on this machine')

SEQS = [
    [1.5, 2.25, float('nan'), 0.1, 3.0],
    [float('nan'), 1.0, 2.0],
    [float('inf'), 1.0, 2.0, float('-inf'), 3.0],
    [1.0, float('inf'), float('nan'), 2.0, float('-inf'), 0.5],
    [float('-inf'), float('nan')],
    list(np.random.default_rng(0).standard_normal(300).astype(np.float32).astype(np.float64) * 7.3),
]


def _ref():
    """The reference's utils.misc, cvhelpers.misc and cvhelpers.torch_helpers, unmodified (through the bridge)."""
    ref_bridge.modules()
    import cvhelpers.misc as cm
    import cvhelpers.torch_helpers as th
    import utils.misc as um
    return SimpleNamespace(um=um, cm=cm, th=th)


@needs_ref
@pytest.mark.parametrize('seq', range(len(SEQS)))
def test_oracle_meter_equals_reference_average_meter(seq):
    um = _ref().um
    ref, ours = um.AverageMeter('k'), O.Meter()
    for v in SEQS[seq]:
        ref.update(torch.tensor(v, dtype=torch.float32))
        ours.update(float(np.float32(v)))
        assert repr((ref.sum, ref.sq_sum, ref.count, ref.val)) == repr((ours.sum, ours.sq_sum, ours.count, ours.val))


@needs_ref
def test_oracle_ema_is_the_reference_rule():
    """The rule of trainer.py:127-134, read from the reference source, applied to sequences with NaN, +-inf and a
    non-finite first value."""
    src = open(os.path.join(ref_bridge.REF_SRC, 'trainer.py')).read()
    assert "if loss_smooth is None:\n                        loss_smooth = losses['total'].item()" in src
    assert "elif not all_isfinite(losses['total']):" in src
    assert "loss_smooth = 0.99 * loss_smooth + 0.01 * losses['total'].item()" in src
    all_isfinite = _ref().th.all_isfinite
    for seq in SEQS:
        ref, warned = None, []
        ours = O.Smooth()
        for step, v in enumerate(seq, 1):
            t = torch.tensor(v, dtype=torch.float32)
            if ref is None:
                ref = t.item()
            elif not all_isfinite(t):
                warned.append(step)
            else:
                ref = 0.99 * ref + 0.01 * t.item()
            ours.update(float(np.float32(v)), step)
        assert repr(ref) == repr(ours.value) and warned == ours.skipped


def _tiny(seed):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(3, 4), torch.nn.Linear(4, 2))


@needs_ref
def test_checkpoint_manager_matches_the_reference(tmp_path, monkeypatch):
    th = _ref().th
    clock = [1_000_000.0]
    monkeypatch.setattr(time, 'time', lambda: clock[0])
    a = T.CheckpointManager(str(tmp_path / 'ours' / 'ckpt' / 'model'), max_to_keep=6, keep_checkpoint_every_n_hours=3.0)
    b = th.CheckPointManager(str(tmp_path / 'ref' / 'ckpt' / 'model'), max_to_keep=6, keep_checkpoint_every_n_hours=3.0)
    model = _tiny(0)
    scores = [0.1, 0.3, 0.2, 0.3, 0.0, 0.5, 0.4, 0.4, 0.1, 0.2, 0.6, 0.0, 0.0, 0.1, 0.55, 0.7, 0.2, 0.0, 0.0, 0.3]
    for i, s in enumerate(scores):
        clock[0] += 1800.0 if i % 3 else 5400.0          # crosses the 3-hour rule several times
        step = 100 * (i + 1)
        a.save(model, step, s)
        b.save(model, step, s)
        fa = sorted(os.listdir(tmp_path / 'ours' / 'ckpt'))
        fb = sorted(os.listdir(tmp_path / 'ref' / 'ckpt'))
        assert fa == fb, (step, fa, fb)
        assert (tmp_path / 'ours' / 'ckpt' / 'checkpoints.txt').read_bytes() == \
            (tmp_path / 'ref' / 'ckpt' / 'checkpoints.txt').read_bytes()
    assert len(fa) > 8       # permanent checkpoints were kept beyond the buffer
    # a fresh manager forgets the earlier checkpoints, as the reference's does
    T.CheckpointManager(str(tmp_path / 'ours' / 'ckpt' / 'model'))
    th.CheckPointManager(str(tmp_path / 'ref' / 'ckpt' / 'model'))
    assert (tmp_path / 'ours' / 'ckpt' / 'checkpoints.txt').read_bytes() == b'Best step: None\n'
    assert (tmp_path / 'ref' / 'ckpt' / 'checkpoints.txt').read_bytes() == b'Best step: None\n'


def _trained_regtr(seed):
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    torch.manual_seed(seed)
    cfg = get_config('3dmatch')
    m = RegTR(cfg)
    opt = torch.optim.AdamW(m.parameters(), lr=cfg.base_lr, weight_decay=cfg.weight_decay)
    sched = torch.optim.lr_scheduler.StepLR(opt, 2, 0.5)
    for _ in range(3):
        for p in m.parameters():
            p.grad = torch.randn_like(p) if p.requires_grad else None
        opt.step()
        sched.step()
    return m, opt, sched


def _fresh():
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    m = RegTR(get_config('3dmatch'))
    opt = torch.optim.AdamW(m.parameters(), lr=1.0)
    return m, opt, torch.optim.lr_scheduler.StepLR(opt, 7, 0.9)


def _assert_same_state(src, dst):
    (m0, o0, s0), (m1, o1, s1) = src, dst
    sd0, sd1 = m0.state_dict(), m1.state_dict()
    assert sd0.keys() == sd1.keys() and all(torch.equal(sd0[k], sd1[k]) for k in sd0)
    a, b = o0.state_dict(), o1.state_dict()
    assert a['param_groups'] == b['param_groups'] and a['state'].keys() == b['state'].keys()
    for k in a['state']:
        for n in a['state'][k]:
            assert torch.equal(a['state'][k][n], b['state'][k][n]), (k, n)
    assert s0.state_dict() == s1.state_dict()


@needs_ref
@pytest.mark.parametrize('writer', ['ours', 'reference'])
def test_checkpoints_load_across_managers(tmp_path, writer, caplog):
    th = _ref().th
    src = _trained_regtr(3)
    ours = T.CheckpointManager(str(tmp_path / 'a' / 'model'))
    ref = th.CheckPointManager(str(tmp_path / 'b' / 'model'))
    w, r = (ours, ref) if writer == 'ours' else (ref, ours)
    extra = dict(trainer=dict(seed=1, steps_per_epoch=5, batch_size=2, dataset_len=9)) if writer == 'ours' else {}
    w.save(src[0], 42, 0.5, optimizer=src[1], scheduler=src[2], **extra)
    path = str(tmp_path / ('a' if writer == 'ours' else 'b'))
    for target in (path, os.path.join(path, 'model-42.pth')):      # best of a directory, and a file
        dst = _fresh()
        with caplog.at_level('WARNING'):
            caplog.clear()
            step = r.load(target, dst[0], optimizer=dst[1], scheduler=dst[2])
        assert step == 42
        assert not [rec for rec in caplog.records if 'keys in checkpoint' in rec.getMessage()]
        _assert_same_state(src, dst)
    if writer == 'ours':
        assert ours.loaded_extra == {} and torch.load(os.path.join(path, 'model-42.pth'))['trainer'] == extra['trainer']
    else:
        assert ours.loaded_extra == {}


def test_load_warns_about_missing_and_unexpected_keys(tmp_path, caplog):
    m = _tiny(1)
    mgr = T.CheckpointManager(str(tmp_path / 'model'))
    mgr.save(m, 5, 1.0, trainer={'seed': 3})
    sd = torch.load(tmp_path / 'model-5.pth')
    sd['state_dict']['extra.weight'] = torch.zeros(1)
    del sd['state_dict']['0.bias']
    torch.save(sd, tmp_path / 'model-5.pth')
    with caplog.at_level('WARNING'):
        assert T.CheckpointManager().load(str(tmp_path), _tiny(2), optimizer=object()) == 5
    msgs = [r.getMessage() for r in caplog.records]
    assert "Unexpected keys in checkpoint: ['extra.weight']" in msgs
    assert "Missing keys in checkpoint: ['0.bias']" in msgs
    assert '"optimizer" ignored from checkpoint loading' in msgs


def test_epoch_sampler_covers_every_index_and_resumes():
    for n, bs in ((10, 3), (9, 3), (1, 2), (7, 1)):
        spe = T.steps_per_epoch(n, bs)
        assert spe == math.ceil(n / bs)
        for epoch in range(3):
            batches = T.epoch_batches(5, epoch, n, bs)
            assert len(batches) == spe and all(len(b) == bs for b in batches[:-1])
            assert sorted(i for b in batches for i in b) == list(range(n))
            assert batches == T.epoch_batches(5, epoch, n, bs)
        # the stream of a run equals the stream of a run resumed at any step
        full = [b for e in range(3) for b in T.epoch_batches(5, e, n, bs)]
        for k in range(len(full)):
            e, skip = divmod(k, spe)
            resumed = T.epoch_batches(5, e, n, bs)[skip:] + [b for e2 in range(e + 1, 3) for b in
                                                             T.epoch_batches(5, e2, n, bs)]
            assert resumed == full[k:]
    assert T.epoch_batches(5, 0, 50, 5) != T.epoch_batches(5, 1, 50, 5)
    assert T.epoch_batches(5, 0, 50, 5) != T.epoch_batches(6, 0, 50, 5)


def test_niter_and_validation_conversions():
    assert T.total_iterations(100, 7) == 100 and T.total_iterations(-70, 7) == 490
    assert T.validation_interval(-1, 7) == 7 and T.validation_interval(-3, 7) == 21
    assert T.validation_interval(0, 7) == 0 and T.validation_interval(50, 7) == 50


@needs_ref
def test_log_strings_match_the_reference():
    r = _ref()
    cases = [{'total': 0.123456, 'a': 12345.678, 'b': float('nan')},
             {'x': torch.tensor(1.5), 'hist': torch.arange(3.0), 'y': torch.tensor(2e-5, dtype=torch.float64)}]
    for d in cases:
        assert T.metrics_to_string(d) == r.um.metrics_to_string(d)
        assert T.metrics_to_string(d, '[Losses]') == r.um.metrics_to_string(d, '[Losses]')
    for s in (0, 0.7, 59.9, 61, 3599, 3600, 3661.5, 86399, 86400, 90061, 1e6, -5, -3725.2):
        assert T.pretty_time_delta(s) == r.cm.pretty_time_delta(s), s


@needs_ref
def test_builtin_3dmatch_config_has_the_reference_dataset_keys():
    from regtr_b200.config import get_config, load_config
    ref = load_config(os.path.join(ref_bridge.REF_SRC, 'conf', '3dmatch.yaml'))
    cfg = get_config('3dmatch')
    for k in ('root', 'train_batch_size', 'val_batch_size', 'test_batch_size', 'niter', 'augment_noise',
              'perturb_pose', 'overlap_radius', 'reg_success_thresh_rot', 'reg_success_thresh_trans'):
        assert cfg[k] == ref[k], k


def test_cli_config_recovery_on_resume(tmp_path):
    from regtr_b200 import train
    from regtr_b200.config import get_config
    run = tmp_path / 'run'
    (run / 'ckpt').mkdir(parents=True)
    (run / 'ckpt' / 'model-3.pth').write_bytes(b'')
    cfg = get_config('3dmatch')
    train.write_config(cfg, '3dmatch', str(run / 'config.yaml'))
    for resume in (run / 'ckpt' / 'model-3.pth', run / 'ckpt'):
        opt = train.parser().parse_args(['--resume', str(resume)])
        path = train.resolve_config(opt)
        assert os.path.samefile(path, run / 'config.yaml')
        assert dict(train.load_cfg(path)) == dict(cfg)
    with pytest.raises(SystemExit):
        train.resolve_config(train.parser().parse_args([]))
    opt = train.parser().parse_args(['--config', '3dmatch', '--info-dir', 'x', '--seed', '4'])
    assert (opt.info_dir, opt.seed, opt.summary_every, opt.validate_every, opt.nb_sanity_val_steps) == ('x', 4, 500, -1, 2)
    with pytest.raises(NotImplementedError, match='h5'):
        train.main(['--config', 'modelnet', '--logdir', str(tmp_path / 'logs')])


def test_bookkeeping_struct_layouts_match_the_header(tmp_path):
    """offsetof / sizeof of regtr_meter_args and regtr_pose_err_args, compiled from the header, against the numpy
    dtypes ops.meter_update / ops.pose_errors fill."""
    from regtr_b200 import lib, ops
    cc = shutil.which('cc') or shutil.which('gcc')
    if cc is None:
        pytest.skip('no C compiler')
    text = open(lib.HEADER).read()
    assert int(re.search(r'#define REGTR_METER_MAX_KEYS (\d+)', text).group(1)) == ops.METER_MAX_KEYS
    assert int(re.search(r'#define REGTR_METER_MAX_BANKS (\d+)', text).group(1)) == ops.METER_MAX_BANKS
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{lib.HEADER}"', 'int main(void) {']
    for name, dt in (('regtr_meter_args', ops.METER_ARGS), ('regtr_pose_err_args', ops.POSE_ERR_ARGS)):
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f in dt.names:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    lines += ['return 0;', '}']
    (tmp_path / 'l.c').write_text('\n'.join(lines))
    subprocess.run([cc, str(tmp_path / 'l.c'), '-o', str(tmp_path / 'l')], check=True)
    got = dict(l.split() for l in subprocess.run([str(tmp_path / 'l')], capture_output=True, text=True,
                                                  check=True).stdout.splitlines())
    for name, dt in (('regtr_meter_args', ops.METER_ARGS), ('regtr_pose_err_args', ops.POSE_ERR_ARGS)):
        assert int(got[name]) == dt.itemsize
        for f in dt.names:
            assert int(got[f'{name}.{f}']) == dt.fields[f][1], (name, f)


def test_bookkeeping_ops_reject_cpu_tensors():
    from regtr_b200 import ops
    from regtr_b200.lib import RegtrLibError
    with pytest.raises(RegtrLibError):
        ops.meter_update([torch.tensor(1.0)], [torch.zeros(1, 4, dtype=torch.float64)], 1)
    with pytest.raises(RegtrLibError):
        ops.pose_errors(torch.zeros(6, 1, 3, 4), torch.zeros(1, 3, 4), torch.zeros(6, 1, dtype=torch.float64),
                        torch.zeros(6, 1, dtype=torch.float64), torch.zeros(6, 4, dtype=torch.float64), 0, 10, 0.1)
