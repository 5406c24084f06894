"""Pair-level data parallelism (SURVEY.md 8e): every pair is independent end to end, so ranks take contiguous slices
of the batch.  Inference needs one all_gather of the poses (6*B_local*12 floats).  Training (`Trainer(...,
process_group=...)`) needs, per step, one all-reduce of the four loss normalisers (`losses.compute_loss_device`) and
one of the gradient bucket (`GradBucket`).  Works with the nccl (GPU) and gloo backends; training uses only
all_reduce and broadcast on CUDA tensors."""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist

DEFAULT_TIMEOUT_S = 600         # process-group timeout of `python -m regtr_b200.train` under torchrun


def shard_range(n_pairs: int, rank: int, world: int):
    """Contiguous, balanced slice [lo, hi) of `n_pairs` for `rank` (first ranks take the remainder)."""
    base, rem = divmod(n_pairs, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_poses(pose_local: torch.Tensor, n_pairs: int):
    """pose_local (L, B_local, 3, 4) -> (L, n_pairs, 3, 4) on every rank, in global pair order."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return pose_local
    world, rank = dist.get_world_size(), dist.get_rank()
    L = pose_local.shape[0]
    b_max = -(-n_pairs // world)
    buf = pose_local.new_zeros((L, b_max, 3, 4))
    buf[:, :pose_local.shape[1]] = pose_local
    out = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(out, buf)
    parts = []
    for r in range(world):
        lo, hi = shard_range(n_pairs, r, world)
        parts.append(out[r][:, :hi - lo])
    return torch.cat(parts, dim=1)


# ------------------------------------------------------------------------------------------------------ training

def torchrun_env(environ=None):
    """(rank, world_size, local_rank) from torchrun's RANK, WORLD_SIZE and LOCAL_RANK, or None when WORLD_SIZE is
    unset.  Raises ValueError on values that do not describe a rank of the world."""
    env = os.environ if environ is None else environ
    if 'WORLD_SIZE' not in env:
        return None
    try:
        world = int(env['WORLD_SIZE'])
        rank = int(env.get('RANK', '0'))
        local = int(env.get('LOCAL_RANK', str(rank)))
    except ValueError as exc:
        raise ValueError(f'torchrun environment: {exc}') from exc
    if world < 1 or not 0 <= rank < world or local < 0:
        raise ValueError(f'torchrun environment: RANK={rank}, WORLD_SIZE={world}, LOCAL_RANK={local}')
    return rank, world, local


def group_rank_world(group) -> tuple:
    """(rank, world size) in `group`; (0, 1) for None."""
    if group is None:
        return 0, 1
    return group.rank(), group.size()


def check_batch_size(batch_size: int, world: int):
    """Data-parallel training shards the global batch over the ranks: every rank needs at least one pair of a full
    batch."""
    if batch_size < world:
        raise ValueError(f'train_batch_size {batch_size} is smaller than the world size {world}: every rank must hold '
                         'at least one pair of a batch')


def broadcast_tensors(tensors: Sequence[torch.Tensor], group, src: int = 0):
    """Overwrite every tensor with rank `src`'s (initial weights and buffers).  The copy back is an in-place torch op,
    so version counters move and cached weight splits of the old values are not reused."""
    for t in tensors:
        buf = t.detach().clone()
        dist.broadcast(buf, group_src(group, src), group=group)
        with torch.no_grad():
            t.copy_(buf)


def group_src(group, rank_in_group: int) -> int:
    """The global rank of `rank_in_group` (broadcast takes global ranks)."""
    try:
        return dist.get_global_rank(group, rank_in_group)
    except (AttributeError, ValueError, RuntimeError):
        return rank_in_group


def broadcast_string(s: Optional[str], group, src: int = 0, capacity: int = 4096) -> str:
    """Rank `src`'s string on every rank, through one CUDA byte tensor (all ranks pass the same capacity)."""
    dev = torch.device('cuda', torch.cuda.current_device())
    buf = torch.zeros(capacity + 4, dtype=torch.uint8)
    if s is not None:
        raw = s.encode('utf-8')
        if len(raw) > capacity:
            raise ValueError(f'broadcast_string: {len(raw)} bytes, at most {capacity}')
        buf[:4] = torch.from_numpy(np.array([len(raw)], '<u4').view(np.uint8))
        buf[4:4 + len(raw)] = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
    d = buf.to(dev)
    dist.broadcast(d, group_src(group, src), group=group)
    h = d.cpu().numpy()
    n = int(h[:4].view('<u4')[0])
    return bytes(h[4:4 + n]).decode('utf-8')


class GradBucket:
    """The gradient exchange of a data-parallel step: one flat fp32 CUDA bucket holding, in order, the gradient of
    every trainable parameter, `n_vals` loss values, a failure flag and one has-gradient flag per parameter.  A step
    packs it (one launch of regtr_bucket_copy), sums it over the ranks (one all-reduce), reads the flags back (one
    D2H of the tail) and unpacks the gradients (one launch).  A rank that failed, or holds no pair, packs zeros and its
    flags, so no rank ever waits for a collective that another rank skipped."""

    def __init__(self, params: List[torch.nn.Parameter], n_vals: int):
        from .optim import CHUNK
        self.params = [p for p in params if p.requires_grad]
        self.n_vals = int(n_vals)
        self.offs, off = [], 0
        for p in self.params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous()):
                raise ValueError('GradBucket: every trainable parameter must be a contiguous CUDA float32 tensor')
            self.offs.append(off)
            off += p.numel()
        self.n_grad = off
        self.n_total = off + self.n_vals + 1 + len(self.params)
        self.chunk = CHUNK

    def _copy(self, rows, bucket, unpack: bool):
        from . import lib as _lib
        from . import ops
        from .optim import _upload
        table = np.zeros(len(rows), dtype=_BUCKET_REF)
        first = 0
        for i, (ptr, n, off) in enumerate(rows):
            table[i] = (ptr, n, first, off)
            first += -(-n // self.chunk)
        if not len(rows):
            return
        t = _upload(table, bucket.device)
        L = _lib.load()
        _lib.check(L.regtr_bucket_copy(t.data_ptr(), len(rows), first, bucket.data_ptr(), int(unpack), ops._stream()),
                   'regtr_bucket_copy')
        ops._count(1)

    def exchange(self, vals: Optional[List[torch.Tensor]], failed: bool, group):
        """Sum every rank's gradients and `vals` (0-d fp32 CUDA tensors; None: zeros) over `group`.  Returns None on
        every rank when any rank failed (the gradients are then left as they are), else the (n_vals,) device vector
        of summed values; the parameters that have a gradient on some rank get the summed gradient."""
        dev = self.params[0].device
        bucket = torch.empty(self.n_total, dtype=torch.float32, device=dev)
        flags = np.zeros(1 + len(self.params), np.float32)
        flags[0] = 1.0 if failed else 0.0
        rows = []
        for i, (p, off) in enumerate(zip(self.params, self.offs)):
            g = None if failed else p.grad
            if g is not None:
                if not (g.is_cuda and g.dtype == torch.float32 and g.is_contiguous()):
                    raise ValueError('GradBucket: gradients must be contiguous CUDA float32 tensors')
                flags[1 + i] = 1.0
            rows.append((0 if g is None else g.data_ptr(), p.numel(), off))
        if vals is not None and not failed:
            if len(vals) != self.n_vals:
                raise ValueError(f'GradBucket: {len(vals)} values, expected {self.n_vals}')
            rows += [(v.data_ptr(), 1, self.n_grad + k) for k, v in enumerate(vals)]
        else:
            rows.append((0, self.n_vals, self.n_grad))
        from .optim import _upload
        flag_dev = _upload(flags.view(np.uint8), dev).view(torch.float32)
        rows.append((flag_dev.data_ptr(), flags.size, self.n_grad + self.n_vals))
        self._copy(rows, bucket, unpack=False)
        dist.all_reduce(bucket, op=dist.ReduceOp.SUM, group=group)
        tail = bucket[self.n_grad + self.n_vals:].cpu().numpy()
        if tail[0] != 0:
            return None
        back = []
        for p, off, has in zip(self.params, self.offs, tail[1:]):
            if has == 0:
                continue
            if p.grad is None:
                p.grad = torch.empty_like(p)
            back.append((p.grad.data_ptr(), p.numel(), off))
        self._copy(back, bucket, unpack=True)
        return bucket[self.n_grad:self.n_grad + self.n_vals]


_BUCKET_REF = np.dtype([('t', '<u8'), ('n', '<i8'), ('first', '<i8'), ('off', '<i8')])
assert _BUCKET_REF.itemsize == 32                  # the C struct's size
