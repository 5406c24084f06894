"""Training batches for 3DMatch on the library's kernels (SURVEY.md 8f N3): overlap ground truth and the reference's
augmentations, from a collated batch to what `RegTR.forward_train` and `compute_loss` read.

Replaces, for the train phase of the reference's loader (/root/reference/src/data_loaders/__init__.py:16-23,
threedmatch.py:79-106):
  * `compute_overlap` (utils/pointcloud.py:8-65) on the aligned float64 clouds: `ops.overlap_nn` (float64 distances,
    strict radius test, nearest first, lowest index on ties);
  * RigidPerturb(cfg.perturb_pose) -> Jitter(cfg.augment_noise) -> ShufflePoints(30000) -> RandomSwap()
    (data_loaders/transforms.py:15-149): `ops.train_augment`.

Randomness: the few per-pair scalars (rotation axis and angle, translation, Euler angles, which side is perturbed,
whether to swap) are drawn on the host from `numpy.random.default_rng([seed, step, pair])`, the same block of
7 uniforms and 4 normals in every mode; the per-point noise (Philox4x32-10) and the permutations (a keyed Feistel
bijection) are drawn on the device from (seed, step, pair, side, point index).  So every draw depends only on
(seed, step, pair position, side, point index), not on the mode or the noise scale.  The reference's global numpy /
torch random streams are not reproduced.

Nothing here synchronises with the host: the correspondences are a lazy entry (reading it costs one D2H of the
counts), and the status word of every call is copied back asynchronously and checked at the next call, when the
correspondences are read, or by `check()`.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from . import ops
from .lazy import LazyDict

MAX_PTS = 30000                      # ShufflePoints(max_pts=30000), transforms.py:98
N_UNIFORM, N_NORMAL = 7, 4           # host draws per pair, in every mode
_INT_MAX = 2 ** 31 - 1


def pair_draws(seed: int, step: int, pair: int):
    """The host block of pair `pair` at (seed, step): (7 uniforms in [0, 1), 4 standard normals)."""
    rng = np.random.default_rng([int(seed), int(step), int(pair)])
    return rng.random(N_UNIFORM), rng.standard_normal(N_NORMAL)


def sample_draws(seed: int, step: int, B: int) -> Dict[str, np.ndarray]:
    """Per-pair scalars of RigidPerturb and RandomSwap:
      axis (B,3): uniform on the sphere (so3_common.uniform_2_sphere: phi ~ U[0, 2 pi), cos theta ~ U[-1, 1));
      angle (B,): N(0,1) * 0.1 pi / sqrt(3) (SO3.sample_small, std 0.1); trans (B,3): N(0,1) * 0.1 / sqrt(3);
      euler (B,3): U[0, 2 pi) (z, y, x angles of _sample_pose_large);
      perturb_source (B,): `random.random() > 0.5`; swap (B,): `random.random() > 0.5`."""
    u = np.empty((B, N_UNIFORM)); g = np.empty((B, N_NORMAL))
    for b in range(B):
        u[b], g[b] = pair_draws(seed, step, b)
    phi, cos_t = 2 * np.pi * u[:, 0], 2.0 * u[:, 1] - 1.0
    sin_t = np.sin(np.arccos(cos_t))
    return dict(axis=np.stack([sin_t * np.cos(phi), sin_t * np.sin(phi), cos_t], axis=1),
                angle=g[:, 0] * (0.1 * np.pi / np.sqrt(3)), trans=g[:, 1:4] * (0.1 / np.sqrt(3)),
                euler=2 * np.pi * u[:, 2:5], perturb_source=u[:, 5] > 0.5, swap=u[:, 6] > 0.5)


def rotation_axis_angle(axis: np.ndarray, angle: float) -> np.ndarray:
    """Rodrigues' formula (SO3.exp of axis * angle)."""
    k = np.array([[0.0, -axis[2], axis[1]], [axis[2], 0.0, -axis[0]], [-axis[1], axis[0], 0.0]])
    return np.eye(3) + np.sin(angle) * k + (1.0 - np.cos(angle)) * (k @ k)


def rotation_zyx(euler: np.ndarray) -> np.ndarray:
    """scipy Rotation.from_euler('zyx', euler).as_matrix(): extrinsic z, then y, then x: Rx(e2) Ry(e1) Rz(e0)."""
    (cz, cy, cx), (sz, sy, sx) = np.cos(euler), np.sin(euler)
    rz = np.array([[cz, -sz, 0.0], [sz, cz, 0.0], [0.0, 0.0, 1.0]])
    ry = np.array([[cy, 0.0, sy], [0.0, 1.0, 0.0], [-sy, 0.0, cy]])
    rx = np.array([[1.0, 0.0, 0.0], [0.0, cx, -sx], [0.0, sx, cx]])
    return rx @ ry @ rz


def perturbations(draws: Dict[str, np.ndarray], mode: str) -> np.ndarray:
    """(B,3,4) float64 perturbation P of each pair before centring: 'small' = (axis-angle rotation | translation),
    'large' = (ZYX Euler rotation | 0), 'none' = identity."""
    B = draws['angle'].shape[0]
    P = np.zeros((B, 3, 4))
    for b in range(B):
        if mode == 'small':
            P[b, :, :3] = rotation_axis_angle(draws['axis'][b], draws['angle'][b])
            P[b, :, 3] = draws['trans'][b]
        elif mode == 'large':
            P[b, :, :3] = rotation_zyx(draws['euler'][b])
        elif mode == 'none':
            P[b, :, :3] = np.eye(3)
        else:
            raise ValueError(f'perturb mode {mode!r}: expected none, small or large')
    return P


class TrainingPrep:
    """`prep(batch, augment=True)` -> the training batch on the device.

    `batch`: a `collate_pair` dict (`ThreeDMatchPairs(..., float64=True)` keeps the clouds and the pose in float64
    as stored; host tensors should be pinned, device tensors are used where they are).  Returned keys:
      src_xyz / tgt_xyz: lists of fp32 views into one packed buffer; src_overlap / tgt_overlap: lists of bool views;
      pose (B,3,4) fp32; correspondences: list of (2, M_b) int64 (lazy: one D2H of the counts when read);
      src_path / tgt_path (swapped where the pair was swapped), idx, overlap_p; aug: the host draws, the flags,
      seed and step.
    augment=False is the reference's val phase: overlap ground truth only, the clouds and the pose as given.
    `step` counts the calls; the draws of a call depend on (seed, step) only."""

    def __init__(self, cfg, seed: int = 0, max_pts: int = MAX_PTS, perturb_mode=None, noise=None):
        self.radius = float(cfg.overlap_radius)
        # conf/3dmatch.yaml: perturb_pose 'small', augment_noise 0.005
        self.mode = str(getattr(cfg, 'perturb_pose', 'small') if perturb_mode is None else perturb_mode)
        if self.mode not in ('none', 'small', 'large'):
            raise ValueError(f'perturb mode {self.mode!r}: expected none, small or large')
        self.noise = float(getattr(cfg, 'augment_noise', 0.005) if noise is None else noise)
        self.seed, self.max_pts, self.step = int(seed), int(max_pts), 0
        self.bound = None
        self._pending: List = []

    # -------------------------------------------------------------------------------- status (asynchronous check)
    def _raise_for(self, word: int, step: int):
        if word & (ops.STATUS_RANGE | 1):         # REGTR_STATUS_RANGE | REGTR_STATUS_KEY_RANGE
            raise ValueError(f'training data of step {step}: an aligned point has a coordinate beyond '
                             f'+-{self.bound:.3f} m, the range in which the overlap search at radius {self.radius} m '
                             f'is exact (or a coordinate is not finite)')

    def _check_pending(self, block: bool):
        keep = []
        for ev, word, step in self._pending:
            if block:
                ev.synchronize()
            elif not ev.query():
                keep.append((ev, word, step))
                continue
            self._raise_for(int(word[0]), step)
        self._pending = keep

    def check(self):
        """Wait for every earlier call and raise ValueError if one met a coordinate outside the exact range."""
        self._check_pending(block=True)

    # ------------------------------------------------------------------------------------------------------ call
    def __call__(self, batch: Dict, augment: bool = True) -> LazyDict:
        self._check_pending(block=False)
        src, tgt = list(batch['src_xyz']), list(batch['tgt_xyz'])
        B = len(src)
        if B == 0 or len(tgt) != B:
            raise ValueError('expected as many source as target clouds, at least one pair')
        step = self.step
        self.step += 1
        clouds = src + tgt
        pose_in = batch['pose']
        dev = next((t.device for t in clouds + [pose_in] if t.is_cuda), None)
        dev = torch.device('cuda', torch.cuda.current_device()) if dev is None else dev
        if self.bound is None:
            self.bound = ops.overlap_coord_bound(self.radius)
        lens = [int(t.shape[0]) for t in clouds]
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        n, n_src = int(offs[-1]), int(offs[B])
        if n >= 2 ** 30:
            raise ValueError(f'{n} points in one batch: at most 2^30 are supported')

        if augment:
            draws = sample_draws(self.seed, step, B)
            P = perturbations(draws, self.mode)
            flags = (ops.PREP_PERTURB_SRC * draws['perturb_source'] + ops.PREP_SWAP * draws['swap'] +
                     ops.PREP_CENTRE * (self.mode == 'small') + ops.PREP_SHUFFLE).astype(np.int32)
            noise, max_pts = self.noise, self.max_pts
        else:
            draws = None
            P = np.tile(np.eye(3, 4), (B, 1, 1))
            flags = np.zeros(B, np.int32)
            noise, max_pts = 0.0, _INT_MAX
        swap = (flags & ops.PREP_SWAP) != 0
        cin = [b + B * int(swap[b]) for b in range(B)] + [b + B * int(not swap[b]) for b in range(B)]
        out_lens = [min(lens[c], max_pts) for c in cin]
        out_offs = np.concatenate([[0], np.cumsum(out_lens)]).astype(np.int64)
        n_out = int(out_offs[-1])

        # every host-known small array in one pinned buffer, one asynchronous copy
        host_pose = not pose_in.is_cuda
        dbl = np.concatenate(([np.asarray(pose_in, dtype=np.float64).reshape(-1)] if host_pose else []) + [P.reshape(-1)])
        ints = np.concatenate([offs, out_offs, flags]).astype(np.int32)
        raw = np.empty(dbl.nbytes + ints.nbytes, np.uint8)
        raw[:dbl.nbytes] = dbl.view(np.uint8)
        raw[dbl.nbytes:] = ints.view(np.uint8)
        params = torch.from_numpy(raw).pin_memory().to(dev, non_blocking=True)
        dvals = params[:dbl.nbytes].view(torch.float64)
        ivals = params[dbl.nbytes:].view(torch.int32)
        if host_pose:
            pose64, pert = dvals[:12 * B].view(B, 3, 4), dvals[12 * B:].view(B, 3, 4)
        else:
            pose64, pert = pose_in.to(torch.float64).contiguous(), dvals.view(B, 3, 4)
        offs_d, out_offs_d, flags_d = ivals[:2 * B + 1], ivals[2 * B + 1:4 * B + 2], ivals[4 * B + 2:]

        xyz = torch.empty((n, 3), dtype=torch.float64, device=dev)
        for t, a, ln in zip(clouds, offs[:-1], lens):
            if ln:
                t = t.reshape(ln, 3)
                xyz[int(a):int(a) + ln].copy_(t if t.dtype == torch.float64 else t.to(dev, non_blocking=True),
                                              non_blocking=True)
        status = ops.new_status(dev)
        nn = ops.overlap_nn(xyz, offs_d, B, pose64, self.radius, status)
        out_xyz, out_mask, out_pose, corr, corr_offs = ops.train_augment(
            xyz, offs_d, B, n_src, pose64, nn, pert, flags_d, self.seed, step, noise, max_pts, out_offs_d, n_out)
        word = torch.empty(1, dtype=torch.int32, pin_memory=True)
        word.copy_(status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pending.append((ev, word, step))

        o = [int(v) for v in out_offs]
        xs = [out_xyz[o[s]:o[s + 1]] for s in range(2 * B)]
        ms = [out_mask[o[s]:o[s + 1]] for s in range(2 * B)]

        def correspondences():
            co = corr_offs.cpu().tolist()                 # the one D2H of this batch
            self._check_pending(block=True)
            return [corr[:, co[b]:co[b + 1]].long() for b in range(B)]

        out = LazyDict(lazy={'correspondences': correspondences},
                       src_xyz=xs[:B], tgt_xyz=xs[B:], src_overlap=ms[:B], tgt_overlap=ms[B:], pose=out_pose,
                       status=status)
        for k in ('src_path', 'tgt_path'):
            if k in batch:
                out[k] = list(batch[k])
        if 'src_path' in out and 'tgt_path' in out:
            for b in np.nonzero(swap)[0]:
                out['src_path'][b], out['tgt_path'][b] = out['tgt_path'][b], out['src_path'][b]
        for k in ('idx', 'overlap_p'):
            if k in batch:
                out[k] = batch[k]
        aug = dict(seed=self.seed, step=step, augment=bool(augment), mode=self.mode if augment else 'none',
                   noise=noise, max_pts=self.max_pts if augment else None, perturb=P, flags=flags,
                   perturb_source=(flags & ops.PREP_PERTURB_SRC) != 0, swap=swap)
        if draws is not None:
            aug.update({k: v for k, v in draws.items() if k not in aug})
        out['aug'] = aug
        return out
