"""ModelNet40 for RegTR: the reference's dataset (data_loaders/modelnet.py, ModelNetHdf) and its `crop` transform chain
(data_loaders/modelnet_transforms.py), with the training batches built on the device.

Dataset (`ModelNetShapes`):
  * `<root>/shape_names.txt` holds the class names; `<root>/{train,test}_files.txt` lists the h5 files, each entry
    stripped of its `data/modelnet40_ply_hdf5_2048/` prefix and joined to root.  The h5 datasets `data` and `label`
    are read (`normal` is not: normals never reach the model), and the shapes are filtered by the category list of
    `*_categoryfile` (`read_categories`: lines without their newline, sorted).  Train reads subset `train` with
    `train_categoryfile`, validation subset `test` with `val_categoryfile`, the benchmark subset `test` with
    `test_categoryfile`.  `idx` is the index of a shape after filtering.
  * The h5 read is `read_h5_files`, the only code that needs h5py (imported lazily through `h5_reader`); everything
    downstream starts from arrays: `ModelNetShapes.from_arrays(points, labels)`.

The crop chain (`crop_chain`, a host restatement in numpy):
    SplitSourceRef -> RandomCrop(partial) -> RandomTransformSE3_euler(rot_mag, trans_mag) -> Resampler(num_points)
    -> RandomJitter() -> ShufflePoints()
  * RandomCrop: per cloud, a direction from `uniform_2_sphere` (phi ~ U[0, 2 pi), then cos theta ~ U[-1, 1)); the
    distance is the dot product of the points minus their fp32 `np.mean` centroid with the float64 direction; the
    mask is d > np.percentile(d, (1 - p_keep) * 100) (linear interpolation), or d > 0 when p_keep == 0.5.  BOTH
    clouds are cropped with p_keep[0], as the reference does.  src_overlap[i]: raw point i survives the other
    cloud's crop (and likewise for the target).
  * RandomTransformSE3_euler: angles U[0,1) * pi * rot_mag / 180 for x, y, z; R = Rx Ry Rz; t ~ U[-trans_mag,
    trans_mag]^3; the 3x4 matrix is cast to float32 and applied to the source only; pose = se3_inv of it in float32.
  * Resampler: with two crop proportions both sizes are 717, the reference's "bug kept for Predator consistency":
    choice(n_kept, 717, replace=False) per cloud.  A crop that keeps fewer points is rejected (`ValueError`); the
    reference's repeat-sampling branch is not reached by any shipped config.
  * RandomJitter: clip(N(0, 0.01^2), +-0.05) added to the float32 points with its defaults, NOT cfg.augment_noise.
  * ShufflePoints: permutes the target first, then the source.
  * correspondences (2, M) int64: (source position, target position) of every raw point present in both outputs, in
    ascending raw index.  Item fields: src_xyz, tgt_xyz, tgt_raw (the uncropped shape), src_overlap, tgt_overlap,
    correspondences, pose, idx.
  * Only noise_type 'crop' yields a sample: for 'clean' and 'jitter' the reference's Resampler / ShufflePoints index
    a src_overlap that only RandomCrop creates, so those raise NotImplementedError.

Validation and test pairs (`ModelNetPairs`) are deterministic: `np.random.seed(idx)` runs again in RandomCrop, in
RandomTransformSE3_euler and in Resampler, and the jitter and the shuffle continue the stream Resampler left, so every
pair is a fixed function of (shape, idx, partial).  They are replayed here with `np.random.RandomState(idx)` reseeded
at the same three points, once at construction, and match the reference's pairs exactly (tests/golden).

Training batches (`ModelNetPrep`) are built on the device by one launch of `ops.modelnet_augment` from the
device-resident shapes: the same chain, in distribution, with counter-based draws (DESIGN.md section 8).
"""
from __future__ import annotations

import os
import types
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import ops
from .lazy import LazyDict

RESAMPLE_POINTS = 717                 # Resampler with two crop proportions (modelnet_transforms.py:92-93)
JITTER_SCALE, JITTER_CLIP = 0.01, 0.05   # RandomJitter() defaults
N_UNIFORM = 10                        # host draws per training pair: 2 x (phi, cos theta), 3 angles, 3 translations
H5_PREFIX = 'data/modelnet40_ply_hdf5_2048/'


# ------------------------------------------------------------------------------------------------------ dataset

def h5_reader():
    """The h5py module.  ModelNet40 is stored as h5 files, and reading them needs h5py."""
    try:
        import h5py
    except ImportError as exc:
        raise NotImplementedError('the ModelNet40 h5 files need h5py, which is not installed') from exc
    if not isinstance(h5py, types.ModuleType):        # a stand-in object registered in sys.modules reads nothing
        raise NotImplementedError('the ModelNet40 h5 files need h5py; sys.modules holds a stand-in for it')
    return h5py


def read_h5_files(fnames: Sequence[str], categories_idx: Optional[Sequence[int]]):
    """ModelNetHdf._read_h5_files without the normals: -> points (S, N, 3) float32, labels (S,) int64, in file order,
    keeping the shapes whose label is in categories_idx (all when None)."""
    h5py = h5_reader()
    points, labels = [], []
    for fname in fnames:
        f = h5py.File(fname, mode='r')
        data = np.asarray(f['data'][:], dtype=np.float32)[..., :3]
        lab = np.asarray(f['label'][:]).flatten().astype(np.int64)
        if categories_idx is not None:
            mask = np.isin(lab, categories_idx).flatten()
            data, lab = data[mask, ...], lab[mask, ...]
        points.append(data)
        labels.append(lab)
    return np.concatenate(points, axis=0), np.concatenate(labels, axis=0)


def read_categories(path: Optional[str]) -> Optional[List[str]]:
    """A `*_categoryfile`: its lines without the newline, sorted; None (every category) for an empty setting."""
    if not path:
        return None
    with open(path) as fid:
        cats = [line.rstrip('\n') for line in fid]
    cats.sort()
    return cats


class ModelNetShapes:
    """The shapes of one ModelNet40 subset: `points` (S, N, 3) float32 (host, or the device after `.to(device)`),
    `labels` (S,) int64, `classes` (the category names kept).  Item i is shape i after category filtering."""

    def __init__(self, root: str, subset: str = 'train', categories: Optional[Sequence[str]] = None):
        with open(os.path.join(root, 'shape_names.txt')) as fid:
            classes = [line.strip() for line in fid]
        category2idx = {c: i for i, c in enumerate(classes)}
        with open(os.path.join(root, f'{subset}_files.txt')) as fid:
            files = [os.path.join(root, line.strip().replace(H5_PREFIX, '')) for line in fid]
        if categories is not None:
            categories_idx = [category2idx[c] for c in categories]
            classes = list(categories)
        else:
            categories_idx = None
        points, labels = read_h5_files(files, categories_idx)
        self._set(points, labels, classes)

    @classmethod
    def from_arrays(cls, points, labels=None, classes: Optional[Sequence[str]] = None) -> 'ModelNetShapes':
        """Shapes from arrays: points (S, N, 3) (only xyz is kept), labels (S,) (zeros when None)."""
        obj = cls.__new__(cls)
        points = np.asarray(points)
        obj._set(np.ascontiguousarray(points[..., :3], dtype=np.float32),
                 np.zeros(len(points), np.int64) if labels is None else np.asarray(labels, np.int64).reshape(-1),
                 classes)
        return obj

    def _set(self, points, labels, classes):
        if points.ndim != 3 or points.shape[2] != 3 or len(labels) != len(points):
            raise ValueError(f'expected points (S, N, 3) and S labels, got {points.shape} and {len(labels)}')
        self.points, self.labels, self.classes = points, labels, classes
        self.device_points: Optional[torch.Tensor] = None

    def to(self, device) -> 'ModelNetShapes':
        """Upload the shapes once (12 N bytes per shape); `device_points` holds them."""
        if self.device_points is None or self.device_points.device != torch.device(device):
            self.device_points = torch.from_numpy(self.points).to(device)
        return self

    def __len__(self):
        return len(self.points)


# ------------------------------------------------------------------------------- the crop chain, restated on the host

def sphere_direction(phi: float, cos_theta: float) -> np.ndarray:
    """uniform_2_sphere from its two draws: (sin theta cos phi, sin theta sin phi, cos theta), theta = arccos."""
    theta = np.arccos(cos_theta)
    return np.stack((np.sin(theta) * np.cos(phi), np.sin(theta) * np.sin(phi), np.cos(theta)), axis=-1)


def crop_mask(xyz: np.ndarray, p_keep: np.float32, direction: np.ndarray) -> np.ndarray:
    """RandomCrop.crop's mask on float32 points (N, 3)."""
    centroid = np.mean(xyz, axis=0)
    d = np.dot(xyz - centroid, direction)
    if p_keep == 0.5:
        return d > 0
    return d > np.percentile(d, (1.0 - p_keep) * 100)


def percentile_position(n: int, p_keep: np.float32):
    """(k, gamma) of the crop threshold np.percentile(d, (1 - p_keep) * 100) over n distances: the threshold lies
    between the order statistics k and k + 1 with numpy's interpolation weight gamma.  (-1, 0.0) for p_keep == 0.5,
    where the crop keeps d > 0.  Read off numpy itself, so its dtype rules for q hold."""
    if p_keep == 0.5:
        return -1, 0.0
    q = (1.0 - p_keep) * 100
    k = int(np.floor(np.percentile(np.arange(n, dtype=np.float64), q)))
    k = min(max(k, 0), n - 2)
    step = np.zeros(n)
    step[k + 1:] = 1.0
    return k, float(np.percentile(step, q))


def check_partial(partial, n_pts: int, num_out: int = RESAMPLE_POINTS) -> np.float32:
    """p_keep[0] as the reference's float32, after checking that its crop keeps at least num_out of n_pts points."""
    if len(partial) != 2:
        raise ValueError(f'partial {list(partial)}: two crop proportions expected (conf/modelnet.yaml)')
    p = np.array(partial, dtype=np.float32)[0]
    if not 0.0 < p < 1.0:
        raise ValueError(f'partial {list(partial)}: the crop proportion must lie in (0, 1)')
    k, _ = percentile_position(n_pts, p)
    kept = n_pts // 2 if k < 0 else n_pts - 1 - k
    if kept < num_out:
        raise ValueError(f'partial {list(partial)} keeps about {kept} of {n_pts} points, fewer than the '
                         f'{num_out} the resampler draws')
    return p


def euler_transform(angle_draws, trans: np.ndarray, rot_mag: float):
    """RandomTransformSE3_euler.generate_transform from its draws (three U[0,1) values, the translation) and the
    float32 pose se3_inv of it: -> (transform (3,4) float32, pose (3,4) float32)."""
    ax, ay, az = (u * np.pi * rot_mag / 180.0 for u in angle_draws)
    cx, cy, cz, sx, sy, sz = np.cos(ax), np.cos(ay), np.cos(az), np.sin(ax), np.sin(ay), np.sin(az)
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    m = np.concatenate((rx @ ry @ rz, np.asarray(trans)[:, None]), axis=1).astype(np.float32)
    irot = m[:, :3].T
    return m, np.concatenate([irot, -irot @ m[:, 3:4]], axis=-1)


def crop_chain(raw: np.ndarray, partial, rot_mag: float, trans_mag: float, rng, idx: int = 0,
               deterministic: bool = False, num_out: int = RESAMPLE_POINTS) -> Dict:
    """The reference's crop chain on one raw shape (N, 3) float32 with the draws of `rng`, an object with numpy's
    legacy `uniform`, `choice`, `normal` and `permutation` (a RandomState, or a replay of recorded draws).
    deterministic: `rng.seed(idx)` before the crop, the transform and the resampler (SetDeterministic).
    -> the item fields (numpy arrays)."""
    raw = np.ascontiguousarray(raw, dtype=np.float32)
    p = check_partial(partial, len(raw), num_out)
    if deterministic:
        rng.seed(idx)
    masks = []
    for _ in range(2):
        phi = rng.uniform(0.0, 2 * np.pi)
        cos_theta = rng.uniform(-1.0, 1.0)
        masks.append(crop_mask(raw, p, sphere_direction(phi, cos_theta)))
    if deterministic:
        rng.seed(idx)
    angles = (rng.uniform(), rng.uniform(), rng.uniform())
    m, pose = euler_transform(angles, rng.uniform(-trans_mag, trans_mag, 3), rot_mag)
    if deterministic:
        rng.seed(idx)
    sel = []
    for mask in masks:
        kept = np.nonzero(mask)[0]
        if len(kept) < num_out:
            raise ValueError(f'a crop kept {len(kept)} points, fewer than the {num_out} the resampler draws')
        sel.append(kept[rng.choice(len(kept), num_out, replace=False)])
    src_pts = np.einsum('ij,bj->bi', m[:, :3], raw[sel[0]]) + m[:, 3:4].T      # se3_transform's float32 einsum
    tgt_pts = raw[sel[1]].copy()
    for pts in (src_pts, tgt_pts):
        pts += np.clip(rng.normal(0.0, scale=JITTER_SCALE, size=(num_out, 3)), a_min=-JITTER_CLIP, a_max=JITTER_CLIP)
    tgt_perm = rng.permutation(num_out)
    src_perm = rng.permutation(num_out)
    src_raw, tgt_raw_idx = sel[0][src_perm], sel[1][tgt_perm]
    return dict(src_xyz=src_pts[src_perm], tgt_xyz=tgt_pts[tgt_perm], tgt_raw=raw,
                src_overlap=masks[1][src_raw], tgt_overlap=masks[0][tgt_raw_idx],
                correspondences=correspondences(src_raw, tgt_raw_idx, len(raw)), pose=pose, idx=idx,
                src_raw_idx=src_raw, tgt_raw_idx=tgt_raw_idx, crop_masks=np.stack(masks))


def correspondences(src_raw: np.ndarray, tgt_raw: np.ndarray, n: int) -> np.ndarray:
    """(2, M) int64 positions of the raw points present in both outputs, in ascending raw index."""
    pos = np.full((2, n), -1, np.int64)
    pos[0, src_raw] = np.arange(len(src_raw))
    pos[1, tgt_raw] = np.arange(len(tgt_raw))
    both = np.nonzero((pos >= 0).all(axis=0))[0]
    return pos[:, both]


def _noise_type(cfg) -> None:
    nt = cfg.get('noise_type', 'crop')
    if nt != 'crop':
        raise NotImplementedError(f'noise_type {nt!r}: only crop yields a sample (the reference\'s Resampler and '
                                  'ShufflePoints index a src_overlap that only RandomCrop creates)')


class ModelNetPairs(torch.utils.data.Dataset):
    """The deterministic validation / test pairs of `shapes` (SetDeterministic in front of the crop chain), computed
    once here.  partial defaults to cfg.partial (the benchmark sets [0.7, 0.7] for ModelNet, [0.5, 0.5] for
    ModelLoNet).  Item i: the fields of `crop_chain` as tensors; `collate(indices, device)` builds a batch."""

    FIELDS = ('src_xyz', 'tgt_xyz', 'tgt_raw', 'src_overlap', 'tgt_overlap', 'correspondences', 'pose', 'idx')

    def __init__(self, shapes: ModelNetShapes, cfg, partial=None):
        _noise_type(cfg)
        self.partial = list(cfg.partial if partial is None else partial)
        self.rot_mag, self.trans_mag = float(cfg.rot_mag), float(cfg.trans_mag)
        self.items = []
        for i in range(len(shapes)):
            it = crop_chain(shapes.points[i], self.partial, self.rot_mag, self.trans_mag, np.random.RandomState(i),
                            idx=i, deterministic=True)
            self.items.append({k: torch.as_tensor(np.asarray(it[k])) for k in self.FIELDS})

    def __len__(self):
        return len(self.items)

    def __getitem__(self, i):
        return self.items[i]

    def collate(self, indices: Sequence[int], device) -> Dict:
        """collate_pair of the items on `device`: lists of clouds, masks and correspondences, pose (B,3,4) fp32."""
        its = [self.items[i] for i in indices]
        out = {k: [it[k].to(device, non_blocking=True) for it in its]
               for k in ('src_xyz', 'tgt_xyz', 'tgt_raw', 'src_overlap', 'tgt_overlap', 'correspondences')}
        out['pose'] = torch.stack([it['pose'] for it in its]).to(device)
        out['idx'] = [int(it['idx']) for it in its]
        return out


# ------------------------------------------------------------------------------------- training batches on the device

def pair_draws(seed: int, step: int, pair: int) -> np.ndarray:
    """The host block of pair `pair` at (seed, step): 10 uniforms in [0, 1)."""
    return np.random.default_rng([int(seed), int(step), int(pair)]).random(N_UNIFORM)


class ModelNetPrep:
    """`prep(items)` -> the training batch of the shapes `items` (a sequence of shape indices, or a dict with 'idx'),
    built on the device by one launch.

    Returned keys (those of augment.TrainingPrep): src_xyz / tgt_xyz: lists of (717, 3) fp32 views into one packed
    buffer; src_overlap / tgt_overlap: lists of bool views; pose (B,3,4) fp32; correspondences: list of (2, M_b)
    int64 (lazy: one D2H of the counts when read); idx; tgt_raw (views of the device shapes); aug: the draws.

    Per pair, the host draws 10 uniforms from `numpy.random.default_rng([seed, step, pair])`: (phi, cos theta) of the
    source's and of the target's crop direction, the three Euler draws and the translation (U[-trans_mag,
    trans_mag] = -trans_mag + 2 trans_mag u); the float32 transform and pose come from `euler_transform`, the
    restatement's own expressions.  The subset, its order and the jitter are drawn on the device from (seed, step,
    pair, side, raw index).  `step` counts the calls unless given.  pair_base: the position of the first pair in the
    global batch when `items` is a slice of it (data parallelism): pair b draws what pair pair_base + b of the whole
    batch draws.  The status word of every call is checked
    asynchronously at the next call, when the correspondences are read, or by `check()`."""

    def __init__(self, cfg, shapes: ModelNetShapes, seed: int = 0, noise: float = JITTER_SCALE,
                 clip: float = JITTER_CLIP):
        _noise_type(cfg)
        if shapes.device_points is None:
            raise ValueError('ModelNetPrep reads the shapes on the device: call shapes.to(device) first')
        self.shapes = shapes
        n_pts = shapes.device_points.shape[1]
        if n_pts > ops.MODELNET_MAX_PTS:
            raise ValueError(f'{n_pts} points per shape: at most {ops.MODELNET_MAX_PTS} are supported')
        self.partial = list(cfg.partial)
        self.p_keep = check_partial(self.partial, n_pts)
        self.k, self.gamma = percentile_position(n_pts, self.p_keep)
        self.rot_mag, self.trans_mag = float(cfg.rot_mag), float(cfg.trans_mag)
        self.seed, self.noise, self.clip = int(seed), float(noise), float(clip)
        self.step = 0
        self._pending: List = []

    def _check_pending(self, block: bool):
        keep = []
        for ev, word, step in self._pending:
            if block:
                ev.synchronize()
            elif not ev.query():
                keep.append((ev, word, step))
                continue
            w = int(word[0])
            if w & ops.STATUS_INPUT:
                raise ValueError(f'ModelNet batch of step {step}: a shape index is out of range or a coordinate is '
                                 'not finite')
            if w & ops.STATUS_CROP:
                raise ValueError(f'ModelNet batch of step {step}: a crop kept fewer than {RESAMPLE_POINTS} points')
        self._pending = keep

    def check(self):
        """Wait for every earlier call and raise ValueError if one met bad input."""
        self._check_pending(block=True)

    def draws(self, step: int, B: int, pair_base: int = 0) -> Dict[str, np.ndarray]:
        """The host draws of a call (pairs pair_base .. pair_base + B - 1): directions (B,2,3), euler (B,3) U[0,1),
        trans (B,3), transform and pose (B,3,4) float32."""
        u = np.stack([pair_draws(self.seed, step, pair_base + b) for b in range(B)]) if B else np.zeros((0, N_UNIFORM))
        dirs = np.stack([sphere_direction(2 * np.pi * u[:, 2 * s], -1.0 + 2.0 * u[:, 2 * s + 1]) for s in (0, 1)],
                        axis=1)
        trans = -self.trans_mag + (2 * self.trans_mag) * u[:, 7:10]
        mats = [euler_transform(u[b, 4:7], trans[b], self.rot_mag) for b in range(B)]
        return dict(uniforms=u, directions=dirs, euler=u[:, 4:7], trans=trans,
                    transform=np.stack([m for m, _ in mats]), pose=np.stack([p for _, p in mats]))

    def __call__(self, items, step: Optional[int] = None, pair_base: int = 0) -> LazyDict:
        self._check_pending(block=False)
        if isinstance(items, dict):
            items = items['idx']
        items = [int(i) for i in items]
        B = len(items)
        if B == 0:
            raise ValueError('expected at least one pair')
        if not all(0 <= i < len(self.shapes) for i in items):
            raise ValueError(f'shape indices {items} outside [0, {len(self.shapes)})')
        if step is None:
            step = self.step
        self.step = step + 1
        dev = self.shapes.device_points.device
        dr = self.draws(step, B, pair_base)

        # the per-pair scalars, the pose and the items in one pinned buffer, one asynchronous copy
        dbl = np.concatenate([dr['directions'].reshape(B, 6), dr['transform'].reshape(B, 12).astype(np.float64)],
                             axis=1)
        flt = dr['pose'].astype(np.float32).reshape(-1)
        ints = np.asarray(items, np.int32)
        raw = np.empty(dbl.nbytes + flt.nbytes + ints.nbytes, np.uint8)
        raw[:dbl.nbytes] = dbl.reshape(-1).view(np.uint8)
        raw[dbl.nbytes:dbl.nbytes + flt.nbytes] = flt.view(np.uint8)
        raw[dbl.nbytes + flt.nbytes:] = ints.view(np.uint8)
        params = torch.from_numpy(raw).pin_memory().to(dev, non_blocking=True)
        pdbl = params[:dbl.nbytes].view(torch.float64).view(B, ops.MODELNET_PARAMS)
        pose = params[dbl.nbytes:dbl.nbytes + flt.nbytes].view(torch.float32).view(B, 3, 4)
        items_d = params[dbl.nbytes + flt.nbytes:].view(torch.int32)

        status = ops.new_status(dev)
        out_xyz, out_mask, corr, corr_n = ops.modelnet_augment(
            self.shapes.device_points, pdbl, items_d, self.seed, step, self.k, self.gamma, self.noise, self.clip,
            RESAMPLE_POINTS, status, pair_base)
        word = torch.empty(1, dtype=torch.int32, pin_memory=True)
        word.copy_(status, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pending.append((ev, word, step))

        def correspondences():
            cn = corr_n.cpu().tolist()                    # the one D2H of this batch
            self._check_pending(block=True)
            return [corr[b, :, :cn[b]].long() for b in range(B)]

        pts = self.shapes.device_points
        out = LazyDict(lazy={'correspondences': correspondences},
                       src_xyz=list(out_xyz[:B]), tgt_xyz=list(out_xyz[B:]), src_overlap=list(out_mask[:B]),
                       tgt_overlap=list(out_mask[B:]), pose=pose, idx=items, tgt_raw=[pts[i] for i in items],
                       status=status)
        out['aug'] = dict(seed=self.seed, step=step, items=items, p_keep=float(self.p_keep), k=self.k,
                          gamma=self.gamma, noise=self.noise, clip=self.clip, **dr)
        return out
