"""Training loop for RegTR on 3DMatch (SURVEY.md 8f N3): the reference's `Trainer.fit` / `_run_validation`
(src/trainer.py:38-175, 213-269), its `CheckPointManager` (cvhelpers/torch_helpers.py:98-242) and the bookkeeping of
`GenericRegModel` (training_step, train_summary_fn, validation_step, validation_epoch_end), on the library path:

    data.PairStream (read-ahead, pinned float64 clouds) -> augment.TrainingPrep -> RegTR.forward_train(train_encoder=True)
    -> compute_loss -> backward -> optim.clip_grad_norm_ -> optim.AdamW.step -> StepLR.step -> ops.meter_update

The reference reads every loss to the host on every step (AverageMeter.update calls .item(), and so does the
loss_smooth EMA).  Here the meters, the EMA and the log of non-finite totals live on the device and are updated by one
launch per step (`ops.meter_update`); they are read back only at summaries, validations and epoch ends, so a step adds
no host synchronisation to what the bare training step does.  Validation accumulates the pose errors on the device too
(`ops.pose_errors`).

Differences from the reference, on purpose:
  * resume continues exactly: the epoch and the position in it follow from the restored step, the epoch order is a
    function of (seed, epoch) and TrainingPrep.step follows the global step, so N steps in one run equal k steps, a
    save, a resume and N - k more steps bit for bit (the reference restarts epoch 0 with a fresh shuffle);
  * the warning for a non-finite total is logged when the meters are read back, not during the step;
  * the progress bar's loss is updated at summaries, not every step;
  * validation losses are the meters' means (fp64 sums), not the fp32 torch.mean of the stacked values.
"""
from __future__ import annotations

import logging
import math
import os
import sys
import time
import traceback
from typing import Dict, List, Optional

import numpy as np
import torch

from . import ops

LOG_CAPACITY = 1024           # non-finite totals remembered between two read-backs


# ------------------------------------------------------------------------------------------------ formatting helpers

def metrics_to_string(metrics, prefix=None) -> str:
    """utils/misc.py metrics_to_string: 'k: v' with 4 significant digits for every scalar, keys sorted."""
    s = ', '.join(f'{k}: {metrics[k]:.4g}' for k in sorted(list(metrics))
                  if isinstance(metrics[k], float) or np.ndim(metrics[k]) == 0)
    if prefix is not None:
        s = prefix + ' ' + s
    return s


def pretty_time_delta(seconds) -> str:
    """cvhelpers/misc.py pretty_time_delta: '1d2h3m4s', '2h3m4s', '3m4s' or '4s' (whole seconds, signed)."""
    sign = '-' if seconds < 0 else ''
    seconds = abs(int(seconds))
    days, seconds = divmod(seconds, 86400)
    hours, seconds = divmod(seconds, 3600)
    minutes, seconds = divmod(seconds, 60)
    if days > 0:
        return '%s%dd%dh%dm%ds' % (sign, days, hours, minutes, seconds)
    if hours > 0:
        return '%s%dh%dm%ds' % (sign, hours, minutes, seconds)
    if minutes > 0:
        return '%s%dm%ds' % (sign, minutes, seconds)
    return '%s%ds' % (sign, seconds)


# ------------------------------------------------------------------------------------------------------ checkpoints

class CheckpointManager:
    """Checkpoints in the reference's format and with its retention rules.

    `save(model, step, score, **kwargs)` writes `<save_path>-<step>.pth` = {'state_dict', 'step', then one entry per
    keyword: its state_dict() if it has one, else the value}.  The last `max_to_keep` checkpoints are kept; one that
    leaves that buffer is kept for good if it was saved after the next permanent time (one every
    `keep_checkpoint_every_n_hours`), else deleted unless it is the best.  The best is the latest checkpoint whose
    score is >= the best score in every component; the previous best is deleted when nothing else keeps it.
    `checkpoints.txt` lists 'Best step: <step>' and the kept files.  A new manager starts with an empty list.

    `load(path, model, **kwargs)` loads a file, or the best checkpoint of a directory, into the model (strict=False,
    warning about unexpected / missing keys) and into every keyword object with load_state_dict; returns the step.
    The checkpoint's entries that were not loaded are available as `loaded_extra`."""

    def __init__(self, save_path: Optional[str] = None, max_to_keep: int = 3, keep_checkpoint_every_n_hours: float = 6.0):
        if max_to_keep <= 0:
            raise ValueError('max_to_keep must be at least 1')
        self._max_to_keep = max_to_keep
        self._keep_every_s = keep_checkpoint_every_n_hours * 3600
        self._logger = logging.getLogger(self.__class__.__name__)
        self._permanent: List = []          # (file, time, step): never deleted
        self._buffer: List = []             # (file, time, step): the last max_to_keep
        self._next_save_time = time.time()
        self._best_score = None
        self._best_step = None
        self.loaded_extra: Dict = {}
        if save_path is not None:
            self._ckpt_dir = os.path.dirname(save_path)
            self._save_path = save_path + '-{}.pth'
            self._list_file = os.path.join(self._ckpt_dir, 'checkpoints.txt')
            os.makedirs(self._ckpt_dir, exist_ok=True)
            self._write_list()
        else:
            self._ckpt_dir = self._save_path = self._list_file = None

    def _write_list(self):
        names = [os.path.basename(c[0]) for c in self._permanent + self._buffer]
        with open(self._list_file, 'w') as fid:
            fid.write(f'Best step: {self._best_step}\n')
            fid.write('\n'.join(names))

    def save(self, model: torch.nn.Module, step: int, score=0.0, **kwargs):
        if self._save_path is None:
            raise AssertionError('Checkpoint manager must be initialized with save path for save().')
        fname = self._save_path.format(step)
        state = {'state_dict': {k: v for k, v in model.state_dict().items() if not v.is_sparse}, 'step': step}
        for k, v in kwargs.items():
            state[k] = v.state_dict() if getattr(v, 'state_dict', None) is not None else v
        torch.save(state, fname)
        self._logger.info(f'Saved checkpoint: {fname}')
        self._buffer.append((fname, time.time(), step))

        if self._best_score is None or np.all(np.array(score) >= np.array(self._best_score)):
            kept = [c[2] for c in self._buffer] + [c[2] for c in self._permanent]
            if self._best_score is not None and self._best_step not in kept:
                os.remove(self._save_path.format(self._best_step))
            self._best_score, self._best_step = score, step
            self._logger.info('Checkpoint is current best, score={}'.format(
                np.array_str(np.array(self._best_score), precision=3)))

        while len(self._buffer) > self._max_to_keep:
            old = self._buffer.pop(0)
            if old[1] > self._next_save_time:
                self._permanent.append(old)
                self._next_save_time = old[1] + self._keep_every_s
            elif self._best_step != old[2]:
                os.remove(old[0])
        self._write_list()

    def load(self, save_path: str, model: Optional[torch.nn.Module] = None, **kwargs) -> int:
        if os.path.isdir(save_path):
            with open(os.path.join(save_path, 'checkpoints.txt')) as fid:
                line = fid.readline()
            assert line.startswith('Best'), 'checkpoints.txt not in expected format.'
            save_path = os.path.join(save_path, 'model-{}.pth'.format(int(line.split(':')[1])))
        state = torch.load(save_path, map_location=None if torch.cuda.is_available() else torch.device('cpu'))
        step = state.get('step', 0)
        if 'state_dict' in state and model is not None:
            res = model.load_state_dict(state['state_dict'], strict=False)
            if len(res.unexpected_keys) > 0:
                self._logger.warning(f'Unexpected keys in checkpoint: {res.unexpected_keys}')
            if len(res.missing_keys) > 0:
                self._logger.warning(f'Missing keys in checkpoint: {res.missing_keys}')
        for k, obj in kwargs.items():
            try:
                if k in state and getattr(obj, 'load_state_dict', None) is not None:
                    obj.load_state_dict(state[k])
                else:
                    self._logger.warning(f'"{k}" ignored from checkpoint loading')
            except ValueError as e:
                self._logger.error(f'Loading {k} from checkpoint failed due to error "{e}", but ignoring and proceeding...')
        self.loaded_extra = {k: v for k, v in state.items() if k not in ('state_dict', 'step') and k not in kwargs}
        self._logger.info(f'Loaded models from {save_path}')
        return step


# -------------------------------------------------------------------------------------------------------- sampling

def steps_per_epoch(n: int, batch_size: int) -> int:
    """Batches per epoch: the last partial batch is kept (the DataLoader's drop_last=False)."""
    return -(-n // batch_size)


def epoch_batches(seed: int, epoch: int, n: int, batch_size: int) -> List[List[int]]:
    """The shuffled batches of one epoch: a permutation of range(n) that depends on (seed, epoch) only."""
    perm = np.random.default_rng([int(seed), int(epoch)]).permutation(n).tolist()
    return [perm[a:a + batch_size] for a in range(0, n, batch_size)]


def total_iterations(niter: int, spe: int) -> int:
    """niter > 0: steps; niter < 0: -niter epochs (trainer.py:64)."""
    return niter if niter > 0 else spe * -niter


def validation_interval(validate_every: int, spe: int) -> int:
    """validate_every < 0: every -validate_every epochs (trainer.py:67-70); 0 means validation only."""
    return -validate_every * spe if validate_every < 0 else validate_every


# ----------------------------------------------------------------------------------------------------------- meters

class DeviceMeters:
    """A StatsMeter (utils/misc.py) whose AverageMeters live on the device: row k of `stats` holds (val, sum, sq_sum,
    count) of key k in fp64, updated by `ops.meter_update`.  `read()` computes avg and var on the host with the
    reference's expressions."""

    def __init__(self, keys, device):
        self.keys = list(keys)
        self.stats = torch.zeros((len(self.keys), 4), dtype=torch.float64, device=device)
        self.fed = False                    # a key exists once a value was offered, even a skipped one

    def clear(self):
        self.stats.zero_()
        self.fed = False

    def read(self) -> Dict[str, Dict[str, float]]:
        if not self.fed:
            return {}
        out = {}
        for k, (val, s, sq, count) in zip(self.keys, self.stats.cpu().tolist()):
            count = int(count)
            m = dict(val=val if count else 0, sum=s, sq_sum=sq, count=count, avg=0, var=None)
            if count:
                m['avg'] = s / count
                m['var'] = sq / count - m['avg'] ** 2
            out[k] = m
        return out

    def averages(self) -> Dict[str, float]:
        return {k: m['avg'] for k, m in self.read().items()}


# ---------------------------------------------------------------------------------------------------------- trainer

def _summary_writers(log_path: str):
    try:
        from torch.utils.tensorboard import SummaryWriter
    except ImportError as exc:
        logging.getLogger(__name__).warning(f'tensorboard is not importable ({exc}): no summaries are written')
        return None, None
    return (SummaryWriter(os.path.join(log_path, 'train'), flush_secs=10),
            SummaryWriter(os.path.join(log_path, 'val'), flush_secs=10))


class Trainer:
    """`Trainer(opt, niter, grad_clip, seed).fit(model, train_set, val_set)`: the reference's training loop for a
    `RegTR` on `ThreeDMatchPairs(float64=True, pin=True)` datasets.  `opt` carries the reference's command-line
    options: log_path, resume, debug, summary_every, validate_every, nb_sanity_val_steps, num_workers.  The batch
    sizes, augmentation and validation thresholds come from `model.cfg`.  Needs a CUDA device."""

    def __init__(self, opt, niter: int, grad_clip: float = 0.0, seed: int = 0):
        self.logger = logging.getLogger(__name__)
        self.opt = opt
        self.niter = int(niter)
        self.grad_clip = float(grad_clip)
        self.seed = int(seed)
        self.log_path = opt.log_path
        self.train_writer, self.val_writer = _summary_writers(self.log_path)
        self.saver = CheckpointManager(os.path.join(self.log_path, 'ckpt', 'model'), max_to_keep=6,
                                       keep_checkpoint_every_n_hours=3.0)
        self.prep = None
        self.epoch_meter = self.summary_meter = None
        self._smooth = self._log = None
        self._batch_info: Dict[int, tuple] = {}
        self._trainer_info: Dict = {}

    # ------------------------------------------------------------------------------------------------ one step
    def setup(self, model, train_set=None):
        """Everything a training step needs: the device, the optimizer and scheduler (configure_optimizers), the
        batch preparation, and the device meters.  Called by fit()."""
        from .augment import TrainingPrep
        if not torch.cuda.is_available():
            raise RuntimeError('Trainer needs a CUDA device: the training step runs on the library\'s sm_90a kernels')
        dev = torch.device('cuda', torch.cuda.current_device())
        model.to(dev)
        model.configure_optimizers()
        self.device = dev
        self.prep = TrainingPrep(model.cfg, seed=self.seed)
        self.epoch_meter = self.summary_meter = None
        self._smooth = torch.zeros(2, dtype=torch.float64, device=dev)
        self._log = torch.zeros(1 + LOG_CAPACITY, dtype=torch.int64, device=dev)
        self._batch_info = {}
        if train_set is not None:
            bs = int(model.cfg.train_batch_size)
            self._trainer_info = dict(seed=self.seed, steps_per_epoch=steps_per_epoch(len(train_set), bs),
                                      batch_size=bs, dataset_len=len(train_set))

    def training_step(self, model, batch, global_step: int):
        """Step `global_step` (counted from 1) on a collated batch: TrainingPrep at step global_step - 1,
        forward_train, compute_loss, zero_grad; then, if the total is differentiable, backward, clipping, optimizer
        and scheduler steps; then one meter launch.  An exception is logged with the batch and swallowed, as in the
        reference.  Returns the losses (or None)."""
        self.prep.step = global_step - 1
        losses = None
        try:
            b = self.prep(batch)
            pred = model.forward_train(b, train_encoder=True)
            losses = model.compute_loss(pred, b)
            model.optimizer.zero_grad()
            if 'total' in losses and losses['total'].requires_grad:
                losses['total'].backward()
                if self.grad_clip > 0:
                    from .optim import clip_grad_norm_
                    clip_grad_norm_(model.parameters(), max_norm=self.grad_clip)
                model.optimizer.step()
                model.scheduler.step()
            self._batch_info[global_step] = (b['idx'] if 'idx' in b else None, b.get('src_path'), b.get('tgt_path'))
            self._update_meters(losses, global_step)
        except Exception as inst:
            _, _, tb = sys.exc_info()
            while tb.tb_next is not None:
                tb = tb.tb_next
            fname = os.path.split(tb.tb_frame.f_code.co_filename)[1]
            self.logger.error(f'{type(inst)} at {fname}:{tb.tb_lineno} - {inst}\n'
                              f'Instance {batch.get("idx")}, src_path: {batch.get("src_path")}, '
                              f'tgt_path: {batch.get("tgt_path")}')
            self.logger.debug(traceback.format_exc())
        return losses

    def _update_meters(self, losses, global_step: int):
        if self.epoch_meter is None:
            self.epoch_meter = DeviceMeters(losses.keys(), self.device)
            self.summary_meter = DeviceMeters(losses.keys(), self.device)
        keys = self.epoch_meter.keys
        ops.meter_update([losses[k] for k in keys], [self.epoch_meter.stats, self.summary_meter.stats], global_step,
                         total_key=keys.index('total') if 'total' in keys else -1, smooth=self._smooth, log=self._log)
        self.epoch_meter.fed = self.summary_meter.fed = True

    def loss_smooth(self) -> Optional[float]:
        """The reference's loss_smooth (None before the first step).  Synchronises."""
        v, is_set = self._smooth.cpu().tolist()
        return v if is_set else None

    def report_nonfinite(self):
        """Log the reference's warning for every step whose total was not finite since the last report (read-back
        point: synchronises), then forget those steps."""
        log = self._log.cpu().tolist()
        n = int(log[0])
        for s in log[1:1 + min(n, LOG_CAPACITY)]:
            idx, sp, tp = self._batch_info.get(int(s), (None, None, None))
            self.logger.warning('Total loss is not finite, Ignoring...\n'
                                f'Instance {idx}, src_path: {sp}, tgt_path: {tp} (step {int(s)})')
        if n > LOG_CAPACITY:
            self.logger.warning(f'{n - LOG_CAPACITY} more steps had a non-finite total loss')
        if n:
            self._log.zero_()
        self._batch_info.clear()

    def _train_summary(self, model, step: int, tbar=None):
        """train_summary_fn: the summary meter's averages as losses/<k>, the learning rate; then clear the meter."""
        self.report_nonfinite()
        if self.summary_meter is not None:
            avg = self.summary_meter.averages()
            self._write_scalars(self.train_writer, model, step, losses=avg)
            self.summary_meter.clear()
        else:
            self._write_scalars(self.train_writer, model, step)
        s = self.loss_smooth()
        if tbar is not None and s is not None:
            tbar.set_description('Loss:{:.3g}'.format(s))

    @staticmethod
    def _write_scalars(writer, model, step, losses=None, metrics=None):
        """_generic_summary_function: scalar losses and metrics, and the scheduler's learning rate."""
        if writer is None:
            return
        for tag, d in (('losses', losses), ('metrics', metrics)):
            for k, v in (d or {}).items():
                if np.ndim(v) == 0:
                    writer.add_scalar(f'{tag}/{k}', v, step)
        if getattr(model, 'scheduler', None) is not None:
            writer.add_scalar('lr', model.scheduler.get_last_lr()[0], step)

    # ------------------------------------------------------------------------------------------------- the loop
    def fit(self, model, train_set, val_set=None):
        from tqdm import tqdm

        from .data import PairStream
        opt = self.opt
        self.setup(model, train_set)
        bs = self._trainer_info['batch_size']
        spe = self._trainer_info['steps_per_epoch']
        n = len(train_set)
        if opt.resume is not None:
            first_step = global_step = self.saver.load(opt.resume, model, optimizer=model.optimizer,
                                                       scheduler=model.scheduler)
        else:
            first_step = global_step = 0
        torch.autograd.set_detect_anomaly(bool(opt.debug))
        epoch, skip = divmod(global_step, spe)
        info = self.saver.loaded_extra.get('trainer') if opt.resume is not None else None
        if info is not None and (info.get('dataset_len') != n or info.get('batch_size') != bs):
            epoch, skip = -(-global_step // spe), 0
            self.logger.warning(f'Resuming with {n} training pairs in batches of {bs}; the checkpoint was written with '
                                f'{info.get("dataset_len")} in batches of {info.get("batch_size")}: starting epoch '
                                f'{epoch} from its first batch')
        elif info is not None and info.get('seed') != self.seed:
            self.logger.warning(f'Resuming with seed {self.seed}; the checkpoint was written with seed {info.get("seed")}')
        total_iter = total_iterations(self.niter, spe)

        if opt.validate_every < 0:
            opt.validate_every = validation_interval(opt.validate_every, spe)
            self.logger.info('Validation interval set to {} steps'.format(opt.validate_every))
        try:
            if opt.validate_every == 0:
                self._run_validation(model, val_set, step=global_step, save_ckpt=False)
                return
            if opt.nb_sanity_val_steps > 0:
                self._run_validation(model, val_set, step=global_step, limit_steps=opt.nb_sanity_val_steps)

            done = False
            while not done:
                batches = epoch_batches(self.seed, epoch, n, bs)
                self.logger.info('Starting epoch {} (steps {} - {})'.format(epoch, global_step,
                                                                            global_step + len(batches) - skip))
                tbar = tqdm(total=len(batches), initial=skip, ncols=80, smoothing=0)
                model.train()
                torch.set_grad_enabled(True)
                t_epoch = time.perf_counter()
                stream = iter(PairStream(train_set, batches[skip:], workers=opt.num_workers))
                try:
                    for batch_idx, batch in enumerate(stream, start=skip):
                        global_step += 1
                        self.training_step(model, batch, global_step)
                        tbar.update(1)
                        if global_step == first_step + 1 or global_step % opt.summary_every == 0:
                            self._train_summary(model, global_step, tbar)
                        if global_step % opt.validate_every == 0:
                            desc = tbar.desc
                            tbar.close()
                            self._run_validation(model, val_set, step=global_step)
                            tbar = tqdm(total=len(batches), ncols=80, initial=batch_idx + 1, desc=desc[:-2])
                        if global_step - first_step >= total_iter:
                            done = True
                            break
                finally:
                    stream.close()
                tbar.close()
                self.report_nonfinite()
                avg = self.epoch_meter.averages() if self.epoch_meter is not None else {}
                self.logger.info('Epoch {} complete in {}. Average train losses: '.format(
                    epoch, pretty_time_delta(time.perf_counter() - t_epoch)) + metrics_to_string(avg) + '\n')
                if self.epoch_meter is not None:
                    self.epoch_meter.clear()
                epoch += 1
                skip = 0
            self.logger.info('Ending training. Number of training steps = {}'.format(global_step))
        finally:
            self.close()

    def close(self):
        """Flush and close the summary writers."""
        for w in (self.train_writer, self.val_writer):
            if w is not None:
                w.close()

    # ------------------------------------------------------------------------------------------------ validation
    def _run_validation(self, model, val_set, step: int, limit_steps: int = -1, save_ckpt: bool = True):
        """_run_validation + validation_step / validation_epoch_end: loss meters and pose errors of every validation
        batch on the device, read back once; the score is reg_success_final.  Saves a checkpoint when save_ckpt."""
        from .augment import TrainingPrep
        from .data import PairStream
        if val_set is None:
            return 0.0
        cfg = model.cfg
        vbs = int(cfg.val_batch_size)
        batches = [list(range(a, min(a + vbs, len(val_set)))) for a in range(0, len(val_set), vbs)]
        if limit_steps > 0:
            batches = batches[:limit_steps]
            self.logger.info(f'Performing validation dry run with {len(batches)} steps')
        else:
            self.logger.info(f'Running validation (step {step})...')
        n_pairs = sum(len(b) for b in batches)
        model.eval()
        prep = TrainingPrep(cfg, seed=self.seed)
        meter, hist, acc, offset = None, None, None, 0
        with torch.no_grad():
            for batch in PairStream(val_set, batches, workers=self.opt.num_workers):
                b = prep(batch, augment=False)
                pred = model(b)
                losses = model.compute_loss(pred, b)
                if meter is None:
                    meter = DeviceMeters(losses.keys(), self.device)
                    nl = pred['pose'].shape[0]
                    hist = torch.zeros((2, nl, max(n_pairs, 1)), dtype=torch.float64, device=self.device)
                    acc = torch.zeros((nl, 4), dtype=torch.float64, device=self.device)
                ops.meter_update([losses[k] for k in meter.keys], [meter.stats], step)
                meter.fed = True
                ops.pose_errors(pred['pose'].contiguous(), b['pose'].contiguous(), hist[0], hist[1], acc, offset,
                                cfg.reg_success_thresh_rot, cfg.reg_success_thresh_trans)
                offset += len(batch['src_xyz'])
            prep.check()
        val_losses = meter.averages() if meter is not None else {}
        metrics = pose_metrics(acc, hist[:, :, :offset]) if acc is not None else {}
        if metrics:
            self.logger.info(f'Aggregating metrics, total number of instances: {offset}')
        score = metrics.get('reg_success_final', 0.0)
        self._write_scalars(self.val_writer, model, step, losses=val_losses, metrics=metrics)
        if self.val_writer is not None:
            for k, v in metrics.items():
                if k.endswith('hist'):
                    self.val_writer.add_histogram(f'metrics/{k}', v, step)
        log_str = ['Validation ended:', metrics_to_string(val_losses, '[Losses]'), metrics_to_string(metrics, '[Metrics]')]
        self.logger.info('\n'.join(log_str))
        if save_ckpt:
            self.saver.save(model, step, score, optimizer=model.optimizer, scheduler=model.scheduler,
                            trainer=dict(self._trainer_info))
        model.train()
        return score


def pose_metrics(acc: torch.Tensor, hist: torch.Tensor) -> Dict:
    """eval.aggregate_metrics from the device accumulators of ops.pose_errors: acc (L, 4) = (sum rot, sum trans,
    n_success, n), hist (2, L, n) = the rot / trans histories.  Names and order of _aggregate_metrics."""
    acc = acc.cpu().tolist()
    hist = hist.cpu()
    nl = len(acc)
    out = {}
    for p in range(nl):
        suffix = f'{p}' if p < nl - 1 else 'final'
        s_rot, s_trans, n_ok, n = acc[p]
        out[f'rot_err_deg_{suffix}'] = s_rot / n if n else math.nan
        out[f'rot_err_{suffix}_hist'] = hist[0, p]
        out[f'trans_err_{suffix}'] = s_trans / n if n else math.nan
        out[f'trans_err_{suffix}_hist'] = hist[1, p]
        out[f'reg_success_{suffix}'] = n_ok / n if n else math.nan
    return out
