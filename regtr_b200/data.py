"""Input side of the forward pass (SURVEY.md 8f N2): 3DMatch pair files -> list-layout batches in pinned
host memory -> the forward's `batch` dict.

Host-side mirror of the inference branch of
  * `ThreeDMatchDataset` (/root/reference/src/data_loaders/threedmatch.py:19-106): `<phase>_<benchmark>_info.pkl`
    (lists `rot` (3,3), `trans` (3,1), `src`, `tgt` relative paths, `overlap`) + one `torch.save`d float64
    ndarray per cloud;
  * `collate_pair` (/root/reference/src/data_loaders/collate_functions.py:4-22): variable-size fields stay
    python lists, `pose` is stacked (B,3,4), `overlap_p` becomes a tensor.
The overlap masks / correspondences the losses need are computed on the fly (`compute_overlap`, the branch the
reference takes when its precomputed h5 file is missing); with `float64=True` the clouds stay float64 for
`augment.TrainingPrep`, which computes the overlap and the training augmentations on the device.

At >1k pairs/s per GPU the loader is part of the path: `PairStream` reads ahead on worker threads, pins the
host clouds (so that `GraphedRegTR.submit` can issue asynchronous H2D copies straight into its static
buffers) and can bucket pairs by size so that consecutive forwards hit the same CUDA-graph capacity bucket.
"""
from __future__ import annotations

import os
import pickle
import queue
import threading
from typing import Dict, Iterable, Iterator, List, Optional, Sequence

import numpy as np
import torch

LIST_FIELDS = ['src_xyz', 'tgt_xyz', 'tgt_raw', 'src_overlap', 'tgt_overlap', 'correspondences',
               'src_path', 'tgt_path', 'idx']


def collate_pair(list_data: Sequence[Dict]) -> Dict:
    """collate_functions.py:4-22."""
    n = len(list_data)
    data = {k: [list_data[b][k] for b in range(n)] for k in LIST_FIELDS if k in list_data[0]}
    data['pose'] = torch.stack([list_data[b]['pose'] for b in range(n)], dim=0)
    if 'overlap_p' in list_data[0]:
        data['overlap_p'] = torch.tensor([list_data[b]['overlap_p'] for b in range(n)])
    return data


def compute_overlap(src: np.ndarray, tgt: np.ndarray, search_radius: float):
    """Overlap region and mutual correspondences of two ALIGNED clouds (utils/pointcloud.py:8-65): a point is
    in the overlap if the other cloud has a point within `search_radius`; its correspondence is the nearest such
    point; `src_tgt_corr` (2, M) keeps the mutual ones (with the reference's `src_corr > 0` quirk: a source
    point matched to target index 0 is never reported).  The reference searches with Open3D's KDTreeFlann
    (absent here: parity unpinned for ties and points exactly on the radius); this uses scipy's cKDTree."""
    from scipy.spatial import cKDTree
    def nearest_within(a, b):                       # for every point of a: nearest point of b within the radius, or -1
        d, i = cKDTree(b).query(a, k=1, distance_upper_bound=search_radius)
        return np.where(np.isfinite(d), i, -1).astype(np.int64)
    tgt_corr = nearest_within(tgt, src)
    src_corr = nearest_within(src, tgt)
    mutual = np.logical_and(tgt_corr[src_corr] == np.arange(len(src_corr)), src_corr > 0)
    return src_corr >= 0, tgt_corr >= 0, np.stack([np.nonzero(mutual)[0], src_corr[mutual]])


class ThreeDMatchPairs(torch.utils.data.Dataset):
    """Inference view of `ThreeDMatchDataset`: item -> {src_xyz, tgt_xyz (N,3) fp32, pose (3,4) fp32 (src -> tgt),
    idx, src_path, tgt_path, overlap_p}.  `root` holds the `test/<scene>/cloud_bin_<i>.pth` files,
    `info_file` is the benchmark's pickle."""

    def __init__(self, root: str, info_file: str, pin: bool = False, overlap_radius: Optional[float] = None,
                 float64: bool = False):
        """overlap_radius (cfg.overlap_radius, 0.0375 for 3DMatch): also produce the training / loss fields
        `src_overlap`, `tgt_overlap`, `correspondences` like the reference does when the precomputed h5 file is
        missing (threedmatch.py:79-86).
        float64=True: `src_xyz`, `tgt_xyz` and `pose` stay float64 as stored on disk -- the input of
        `augment.TrainingPrep`, which computes the overlap on the device (no CPU overlap then)."""
        if float64 and overlap_radius is not None:
            raise ValueError('float64=True leaves the overlap to augment.TrainingPrep: pass no overlap_radius')
        self.overlap_radius, self.float64 = overlap_radius, bool(float64)
        with open(info_file, 'rb') as fid:
            self.infos = pickle.load(fid)
        for k in ('rot', 'trans', 'src', 'tgt', 'overlap'):
            if k not in self.infos:
                raise KeyError(f'{info_file}: missing field {k!r}')
        self.root, self.pin = root, pin

    def __len__(self):
        return len(self.infos['rot'])

    def _cloud(self, rel):
        xyz = torch.load(os.path.join(self.root, rel), weights_only=False)
        t = torch.from_numpy(np.asarray(xyz))                          # float64 ndarray on disk (threedmatch.py:91)
        t = t.double() if self.float64 else t.float()
        return t.pin_memory() if self.pin else t

    def __getitem__(self, item):
        pose = np.concatenate([self.infos['rot'][item], self.infos['trans'][item]], axis=-1)   # se3_init
        pose_t = torch.from_numpy(np.asarray(pose, dtype=np.float64))
        out = {'src_xyz': self._cloud(self.infos['src'][item]), 'tgt_xyz': self._cloud(self.infos['tgt'][item]),
               'pose': pose_t if self.float64 else pose_t.float(), 'idx': item,
               'src_path': self.infos['src'][item], 'tgt_path': self.infos['tgt'][item],
               'overlap_p': self.infos['overlap'][item]}
        if self.overlap_radius is not None:
            s64 = np.asarray(torch.load(os.path.join(self.root, out['src_path']), weights_only=False))
            t64 = np.asarray(torch.load(os.path.join(self.root, out['tgt_path']), weights_only=False))
            sm, tm, corr = compute_overlap(s64 @ pose[:, :3].T + pose[:, 3], t64, self.overlap_radius)
            out.update(src_overlap=torch.from_numpy(sm), tgt_overlap=torch.from_numpy(tm),
                       correspondences=torch.from_numpy(corr))
        return out

    def sizes(self, items: Optional[Iterable[int]] = None) -> List[int]:
        """Total points per pair WITHOUT loading the clouds would need an index; this loads each once."""
        items = range(len(self)) if items is None else items
        out = []
        for i in items:
            d = self[i]
            out.append(int(d['src_xyz'].shape[0] + d['tgt_xyz'].shape[0]))
        return out


def bucket_order(sizes: Sequence[int], batch_size: int, bucket: int = 8192, window: int = 64) -> List[List[int]]:
    """Batches of `batch_size` item indices.  Inside windows of `window` consecutive items the pairs are
    grouped by capacity bucket (ceil(size / bucket)), so that successive forwards replay the same CUDA graph
    and batches are not padded by one outlier; the order of the windows -- and therefore of the stream as a
    whole -- stays that of the dataset.  Every index appears exactly once."""
    batches = []
    for w0 in range(0, len(sizes), window):
        idx = list(range(w0, min(w0 + window, len(sizes))))
        idx.sort(key=lambda i: (-(-sizes[i] // bucket), i))
        batches += [idx[a:a + batch_size] for a in range(0, len(idx), batch_size)]
    return batches


class PairStream:
    """Read-ahead iterator over collated batches: `workers` threads load and pin the clouds, the consumer gets
    `collate_pair` dicts in a deterministic order.  torch.load releases the GIL for the file I/O, and the
    float64 -> float32 conversion is a numpy/torch call, so threads (no process fork, no IPC copy) are enough."""

    def __init__(self, dataset, batches: Sequence[Sequence[int]], workers: int = 4, depth: int = 8):
        self.dataset, self.batches = dataset, [list(b) for b in batches]
        self.workers, self.depth = max(1, int(workers)), max(1, int(depth))

    def __len__(self):
        return len(self.batches)

    def __iter__(self) -> Iterator[Dict]:
        n = len(self.batches)
        slots: List[Optional[Dict]] = [None] * n
        ready = [threading.Event() for _ in range(n)]
        todo: "queue.Queue[int]" = queue.Queue()
        gate = threading.Semaphore(self.depth)             # at most `depth` batches loaded ahead of the consumer
        errors: List[BaseException] = []

        def work():
            while True:
                k = todo.get()
                if k < 0:
                    return
                try:
                    slots[k] = collate_pair([self.dataset[i] for i in self.batches[k]])
                except BaseException as exc:  # surfaced to the consumer
                    errors.append(exc)
                ready[k].set()

        threads = [threading.Thread(target=work, daemon=True) for _ in range(self.workers)]
        for t in threads:
            t.start()
        issued = 0
        try:
            for k in range(n):
                while issued < n and gate.acquire(blocking=issued <= k):
                    todo.put(issued)
                    issued += 1
                ready[k].wait()
                if errors:
                    raise errors[0]
                out, slots[k] = slots[k], None
                gate.release()
                yield out
        finally:
            for _ in threads:
                todo.put(-1)


def to_device_batch(batch: Dict, device) -> Dict:
    """The forward's inputs on `device` (non-blocking when the host tensors are pinned); other fields untouched."""
    out = dict(batch)
    for k in ('src_xyz', 'tgt_xyz'):
        out[k] = [t.to(device, non_blocking=True) for t in batch[k]]
    return out
