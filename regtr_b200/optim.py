"""Optimizer step on the library's kernels: gradient-norm clipping and Adam / AdamW.

The reference's training iteration ends with (trainer.py, generic_reg_model.py):

    clip_grad_norm_(model.parameters(), cfg.grad_clip); optimizer.step(); scheduler.step()

`clip_grad_norm_`, `AdamW` and `Adam` below are drop-in replacements for torch's that run on regtr_grad_norm /
regtr_grad_scale (3 launches) and regtr_adam_step + regtr_split_refresh (2 launches), whatever the number of
parameters, without a host synchronisation.  `AdamW` / `Adam` subclass torch's optimizers: param groups,
state_dict / load_state_dict (torch's state layout: a CPU float32 `step`, `exp_avg`, `exp_avg_sq`) and LR schedulers
are torch's own machinery, and only `step()` differs.

After the update, the TF32 (hi, lo) splits that `ops.split_weight` caches on every updated weight are rewritten in
place (bit-identical to a fresh split) and re-keyed to the parameter's new version: the next forward finds them in
the cache, and a CUDA graph captured before the step (GraphedRegTR) still reads valid weights.
"""
from __future__ import annotations

import numpy as np
import torch

from . import lib as _lib
from . import ops

CHUNK = 8192            # REGTR_OPTIM_CHUNK: elements per chunk of the multi-tensor launches
TILE = 32               # tile edge of regtr_split_refresh

_GRAD_REF = np.dtype([('g', '<u8'), ('n', '<i8'), ('first', '<i8')])
_ADAM = np.dtype([('p', '<u8'), ('g', '<u8'), ('m', '<u8'), ('v', '<u8'), ('n', '<i8'), ('first', '<i8'),
                  ('decay', '<f4'), ('wd', '<f4'), ('b1w', '<f4'), ('b2', '<f4'), ('one_m_b2', '<f4'),
                  ('rcp_bc2_sqrt', '<f4'), ('neg_step_size', '<f4'), ('eps', '<f4'), ('flags', '<u4'), ('pad', '<u4')])
_VIEW = np.dtype([('src', '<u8'), ('hi', '<u8'), ('lo', '<u8'), ('s0', '<i8'), ('s1', '<i8'), ('first', '<i8'),
                  ('rows', '<i4'), ('cols', '<i4')])
assert (_GRAD_REF.itemsize, _ADAM.itemsize, _VIEW.itemsize) == (24, 88, 56)     # the C structs' sizes

_FRESH, _COUPLED, _DECOUPLED = 1, 2, 4


def _check(t, what):
    if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.layout == torch.strided):
        raise _lib.RegtrLibError(f'{what}: expected a contiguous CUDA float32 tensor, got {t.dtype} {t.layout} on '
                                 f'{t.device} (contiguous: {t.is_contiguous()}); the library optimizer has no fallback')


def _upload(rows: np.ndarray, device):
    """Copy a descriptor table to the device without a host sync: a fresh pinned buffer per call (the caching host
    allocator does not hand it out again before the copy has finished), copied on the current stream."""
    host = torch.empty(rows.nbytes, dtype=torch.uint8, pin_memory=True)
    host.numpy()[:] = rows.view(np.uint8)
    return host.to(device, non_blocking=True)


def _chunks(n: int) -> int:
    return (n + CHUNK - 1) // CHUNK


def clip_grad_norm_(parameters, max_norm, norm_type=2.0, error_if_nonfinite=False, foreach=None):
    """torch.nn.utils.clip_grad_norm_ on the library's kernels: scales every gradient in place by
    min(1, max_norm / (total_norm + 1e-6)) and returns the total 2-norm as a 0-d CUDA tensor (tensor(0.) when no
    parameter has a gradient).  The coefficient stays on the device.  Only the 2-norm is implemented, and
    error_if_nonfinite=True (which needs the norm on the host) is not."""
    if float(norm_type) != 2.0:
        raise NotImplementedError(f'clip_grad_norm_: norm_type={norm_type!r}; the library implements the 2-norm only')
    if error_if_nonfinite:
        raise NotImplementedError('clip_grad_norm_: error_if_nonfinite=True needs a host synchronisation')
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    grads = [p.grad for p in parameters if p.grad is not None]
    if not grads:
        return torch.tensor(0.0)
    dev = grads[0].device
    for g in grads:
        _check(g, 'clip_grad_norm_: grad')
        if g.device != dev:
            raise _lib.RegtrLibError('clip_grad_norm_: every gradient must be on one device')
    L = _lib.load()
    rows = np.zeros(len(grads), dtype=_GRAD_REF)
    first = 0
    for i, g in enumerate(grads):
        rows[i] = (g.data_ptr(), g.numel(), first)
        first += _chunks(g.numel())
    with torch.cuda.device(dev):
        table = _upload(rows, dev)
        out = torch.empty(2, dtype=torch.float32, device=dev)
        ws = ops.workspace(L.regtr_grad_norm_ws_bytes(first), dev, 'grad_norm')
        _lib.check(L.regtr_grad_norm(table.data_ptr(), len(grads), first, float(max_norm), out.data_ptr(),
                                     ws.data_ptr(), ws.numel(), ops._stream()), 'regtr_grad_norm')
        _lib.check(L.regtr_grad_scale(table.data_ptr(), len(grads), first, out[1:].data_ptr(), ops._stream()),
                   'regtr_grad_scale')
    ops._count(3 if first else 1)
    return out[0]


def _split_views(p, version):
    """(views of p's split cache keyed at `version`, keys of its stale entries)."""
    cache = p.__dict__.get('_regtr_split')
    if not cache:
        return [], []
    live, stale = [], []
    base = p.data_ptr() - p.storage_offset() * p.element_size()
    for key, (hi, lo) in cache.items():
        if key[-1] != version:
            stale.append(key)
            continue
        off, shape, stride, transpose = key[0], key[1], key[2], key[3]
        rows, cols = (shape[1], shape[0]) if transpose else shape
        s0, s1 = (stride[1], stride[0]) if transpose else stride
        if tuple(hi.shape) != (rows, cols) or not (hi.is_contiguous() and lo.is_contiguous()):
            raise _lib.RegtrLibError('split cache entry does not match its view')
        live.append((base + off * 4, hi.data_ptr(), lo.data_ptr(), s0, s1, rows, cols))
    return live, stale


class _LibraryAdam:
    """step() of Adam / AdamW on regtr_adam_step + regtr_split_refresh (mixed into torch's classes)."""

    _DECOUPLED = False

    def _check_options(self):
        for group in self.param_groups:
            for opt in ('amsgrad', 'maximize', 'capturable', 'differentiable'):
                if group.get(opt, False):
                    raise NotImplementedError(f'{type(self).__name__}: {opt}=True is not supported by the library step')
            if group.get('fused'):
                raise NotImplementedError(f'{type(self).__name__}: fused=True selects torch\'s fused kernel; the '
                                          'library step is its own multi-tensor launch')
            if isinstance(group['lr'], torch.Tensor) or any(isinstance(b, torch.Tensor) for b in group['betas']):
                raise NotImplementedError(f'{type(self).__name__}: tensor lr / betas are not supported (host scalars only)')

    @torch.no_grad()
    def step(self, closure=None):
        """One Adam / AdamW update of every parameter that has a gradient (the others, their state and their version
        counter stay untouched), then the refresh of their cached weight splits.  Two launches, no host sync."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self._check_options()
        L = _lib.load()
        name = type(self).__name__
        todo, dev = [], None
        for group in self.param_groups:            # validate everything before any state changes
            for p in group['params']:
                if p.grad is None:
                    continue
                _check(p, f'{name}: parameter')
                _check(p.grad, f'{name}: grad')
                dev = p.device if dev is None else dev
                if p.device != dev:
                    raise _lib.RegtrLibError(f'{name}: every parameter must be on one device')
                state = self.state[p]
                if state:
                    if state['step'].is_cuda:
                        raise _lib.RegtrLibError(f'{name}: a device `step` (capturable state) would need a host '
                                                 'sync; load the state with a CPU step')
                    _check(state['exp_avg'], f'{name}: exp_avg')
                    _check(state['exp_avg_sq'], f'{name}: exp_avg_sq')
                todo.append((group, p))
        rows, params, first = [], [], 0
        for group, p in todo:
            lr, (b1, b2), eps, wd = group['lr'], group['betas'], group['eps'], group['weight_decay']
            state = self.state[p]
            flags = 0
            if len(state) == 0:                    # torch's layout; the kernel reads the new moments as zeros
                state['step'] = torch.tensor(0.0, dtype=torch.float32)
                state['exp_avg'] = torch.empty_like(p, memory_format=torch.preserve_format)
                state['exp_avg_sq'] = torch.empty_like(p, memory_format=torch.preserve_format)
                flags |= _FRESH
            state['step'] += 1
            t = state['step'].item()               # a CPU tensor: no device sync
            bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
            if wd != 0:
                flags |= _DECOUPLED if group.get('decoupled_weight_decay', self._DECOUPLED) else _COUPLED
            rcp = np.float32(1.0) / np.float32(bc2 ** 0.5)
            rows.append((p.data_ptr(), p.grad.data_ptr(), state['exp_avg'].data_ptr(), state['exp_avg_sq'].data_ptr(),
                         p.numel(), first, 1 - lr * wd, wd, 1 - b1, b2, 1 - b2, rcp, -(lr / bc1), eps, flags, 0))
            first += _chunks(p.numel())
            params.append(p)
        if not params:
            return loss
        with torch.cuda.device(dev):
            table = _upload(np.array(rows, dtype=_ADAM), dev)
            _lib.check(L.regtr_adam_step(table.data_ptr(), len(rows), first, ops._stream()), 'regtr_adam_step')
            ops._count(1 if first else 0)
            vrows, tiles, stale = [], 0, []
            for p in params:
                live, old = _split_views(p, p._version)
                stale.append(old)
                for v in live:
                    vrows.append(v[:5] + (tiles,) + v[5:])
                    tiles += ((v[5] + TILE - 1) // TILE) * ((v[6] + TILE - 1) // TILE)
            if tiles:
                vt = _upload(np.array(vrows, dtype=_VIEW), dev)
                _lib.check(L.regtr_split_refresh(vt.data_ptr(), len(vrows), tiles, ops._stream()), 'regtr_split_refresh')
                ops._count(1)
        # the parameters changed in place behind autograd's back: bump their versions (saved tensors of an older
        # forward now fail autograd's check, as after torch's step), then re-key the refreshed splits to them
        old = [p._version for p in params]
        torch.autograd.graph.increment_version(params)
        for p, v0, gone in zip(params, old, stale):
            cache = p.__dict__.get('_regtr_split')
            if not cache:
                continue
            for k in gone:
                del cache[k]
            for k in [k for k in cache if k[-1] == v0]:
                cache[k[:-1] + (p._version,)] = cache.pop(k)
        return loss


class AdamW(_LibraryAdam, torch.optim.AdamW):
    """torch.optim.AdamW whose step() runs on the library's kernels (see the module docstring).  amsgrad, maximize,
    capturable, differentiable, fused=True and a tensor lr are rejected."""

    _DECOUPLED = True

    def __init__(self, params, *args, **kwargs):
        super().__init__(params, *args, **kwargs)
        self._check_options()


class Adam(_LibraryAdam, torch.optim.Adam):
    """torch.optim.Adam (coupled weight decay) whose step() runs on the library's kernels."""

    def __init__(self, params, *args, **kwargs):
        super().__init__(params, *args, **kwargs)
        self._check_options()
