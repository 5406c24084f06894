"""Fixture of the reference's ModelNet crop chain: tests/golden/modelnet_transforms.npz.

    python tests/golden/make_modelnet_golden.py

Runs the UNMODIFIED data_loaders/modelnet_transforms.py of the reference (loaded by file path: the package __init__
imports h5py) on seeded synthetic 2048-point shapes (unions of ellipsoid and box surfaces with a few duplicated
points, so that crop distances tie), given as xyz + normals like the h5 files:
  * the deterministic test chain (SetDeterministic, SplitSourceRef, RandomCrop, RandomTransformSE3_euler,
    Resampler(1024), RandomJitter, ShufflePoints) for several idx at partial [0.7, 0.7] and [0.5, 0.5];
  * the train chain (the same without SetDeterministic) with every np.random draw recorded (uniform, choice, normal,
    permutation) next to the outputs.
numpy 2 shims: `np.bool = bool` (the transforms use the removed alias).  numpy 2 also promotes 1.0 - np.float32(p) to
float32 where numpy 1 gave float64: that moves the percentile's q in its last bits, but cannot move a threshold that
lies strictly between two order statistics, so the crop masks are those of numpy 1.
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_bridge  # noqa: E402
from regtr_b200.synthetic import make_modelnet_shapes  # noqa: E402

ROT_MAG, TRANS_MAG, NUM_POINTS = 45.0, 0.5, 1024        # conf/modelnet.yaml
TEST_CASES = [([0.7, 0.7], idx) for idx in (0, 1, 5)] + [([0.5, 0.5], idx) for idx in (0, 2, 7)]
TRAIN_CASES = [([0.7, 0.7], 3, 11), ([0.5, 0.5], 4, 12)]     # (partial, shape, np.random seed)


def load_transforms():
    if not hasattr(np, 'bool'):
        np.bool = bool
    sys.path.insert(0, ref_bridge.REF_SRC)
    spec = importlib.util.spec_from_file_location(
        'ref_modelnet_transforms', os.path.join(ref_bridge.REF_SRC, 'data_loaders', 'modelnet_transforms.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Recorder:
    """Wraps np.random's uniform / choice / normal / permutation; every draw is appended to `log`."""
    NAMES = ('uniform', 'choice', 'normal', 'permutation')

    def __init__(self):
        self.log, self.saved = [], []

    def __enter__(self):
        for f in self.NAMES:
            orig = getattr(np.random, f)
            self.saved.append((f, orig))

            def wrap(*a, _orig=orig, _name=f, **k):
                v = _orig(*a, **k)
                self.log.append((_name, np.array(v)))
                return v
            setattr(np.random, f, wrap)
        return self

    def __exit__(self, *exc):
        for f, orig in self.saved:
            setattr(np.random, f, orig)


def chain(T, partial, deterministic):
    ts = [T.SetDeterministic()] if deterministic else []
    return ts + [T.SplitSourceRef(), T.RandomCrop(partial), T.RandomTransformSE3_euler(rot_mag=ROT_MAG, trans_mag=TRANS_MAG),
                 T.Resampler(NUM_POINTS), T.RandomJitter(), T.ShufflePoints()]


def with_normals(xyz, rng):
    n = rng.normal(size=xyz.shape)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    return np.concatenate([xyz, n.astype(np.float32)], axis=1)


def run(T, points, idx, partial, deterministic):
    sample = {'points': points.copy(), 'label': np.int64(0), 'idx': np.array(idx, dtype=np.int32)}
    for t in chain(T, partial, deterministic):
        sample = t(sample)
    return sample


def record(out, p, sample):
    out[p + 'src_xyz'] = sample['points_src'][:, :3]
    out[p + 'tgt_xyz'] = sample['points_ref'][:, :3]
    out[p + 'src_overlap'] = sample['src_overlap']
    out[p + 'tgt_overlap'] = sample['ref_overlap']
    out[p + 'correspondences'] = sample['correspondences']
    out[p + 'pose'] = sample['transform_gt']


def main():
    T = load_transforms()
    shapes = make_modelnet_shapes(8, seed=2024)
    rng = np.random.default_rng(5)
    pts6 = np.stack([with_normals(s, rng) for s in shapes])
    out = {'shapes': shapes}
    for c, (partial, idx) in enumerate(TEST_CASES):
        p = f'test{c}/'
        out[p + 'partial'] = np.array(partial)
        out[p + 'idx'] = np.array(idx)
        record(out, p, run(T, pts6[idx], idx, partial, deterministic=True))
    for c, (partial, shape, seed) in enumerate(TRAIN_CASES):
        p = f'train{c}/'
        np.random.seed(seed)
        with Recorder() as rec:
            sample = run(T, pts6[shape], shape, partial, deterministic=False)
        out[p + 'partial'] = np.array(partial)
        out[p + 'idx'] = np.array(shape)
        for i, (name, v) in enumerate(rec.log):
            out[p + f'draw{i:02d}_{name}'] = v
        record(out, p, sample)
    np.savez_compressed(os.path.join(HERE, 'modelnet_transforms.npz'), **out)
    print(f'{len(TEST_CASES)} test and {len(TRAIN_CASES)} train cases -> modelnet_transforms.npz')


if __name__ == '__main__':
    main()
