"""Fixture of the reference's training augmentations: tests/golden/augment.npz.

    python tests/golden/make_augment_golden.py

Runs the UNMODIFIED data_loaders/transforms.py of the reference (loaded by file path: the package __init__ imports
h5py) in the order of its train loader (RigidPerturb -> Jitter -> ShufflePoints -> RandomSwap) on small seeded
pairs whose overlap and correspondences come from the float64 oracle, and records every random draw the transforms
take (np.random.uniform / randn / rand / permutation, random.random, torch.randn) next to their outputs.  Cases
cover the 'small' / 'large' / 'none' modes, truncation (max_pts below n) and both swap outcomes.
"""
import importlib.util
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import ref_bridge  # noqa: E402
import train_data_oracle as O  # noqa: E402

RADIUS = 0.0375
CASES = [('small', 30000), ('small', 70), ('large', 30000), ('large', 90), ('none', 30000), ('none', 60)]


def load_transforms():
    sys.path.insert(0, ref_bridge.REF_SRC)
    spec = importlib.util.spec_from_file_location('ref_transforms',
                                                  os.path.join(ref_bridge.REF_SRC, 'data_loaders', 'transforms.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class Recorder:
    """Wraps the random functions the transforms call; every draw is appended to `log` as (name, value)."""
    NAMES = (('np', 'uniform'), ('np', 'randn'), ('np', 'rand'), ('np', 'permutation'), ('random', 'random'),
             ('torch', 'randn'))

    def __init__(self):
        self.log = []
        self.saved = []

    def __enter__(self):
        mods = {'np': np.random, 'random': random, 'torch': torch}
        for m, f in self.NAMES:
            orig = getattr(mods[m], f)
            self.saved.append((mods[m], f, orig))

            def wrap(*a, _orig=orig, _name=f'{m}.{f}', **k):
                v = _orig(*a, **k)
                self.log.append((_name, np.array(v.numpy() if torch.is_tensor(v) else v)))
                return v
            setattr(mods[m], f, wrap)
        return self

    def __exit__(self, *exc):
        for mod, f, orig in self.saved:
            setattr(mod, f, orig)


def make_pair(rng):
    """Two seeded clouds with a clear overlap (80 % of the source lies within a few mm of the target)."""
    base = rng.uniform(-0.4, 0.4, size=(int(rng.integers(120, 200)), 3))
    tgt = base[:int(len(base) * 0.8)] + rng.normal(scale=0.004, size=(int(len(base) * 0.8), 3))
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    q *= np.sign(np.linalg.det(q))
    pose = np.concatenate([q, rng.normal(scale=0.5, size=(3, 1))], axis=1)
    src_world = np.concatenate([base[len(base) // 5:], rng.uniform(0.6, 0.9, size=(20, 3))])
    src = (src_world - pose[:, 3]) @ pose[:, :3]                    # pose maps src to tgt
    return src, tgt, pose


def main():
    T = load_transforms()
    out = {}
    rng = np.random.default_rng(7)
    seen = set()
    k = 0
    seed = 0
    while len(seen) < 2 * len(CASES):
        mode, max_pts = CASES[k % len(CASES)]
        src, tgt, pose = make_pair(rng)
        sm, tm, corr, _, _ = O.overlap(src, tgt, pose, RADIUS)
        data = {'src_xyz': torch.from_numpy(src).float(), 'tgt_xyz': torch.from_numpy(tgt).float(),
                'src_overlap': torch.from_numpy(sm), 'tgt_overlap': torch.from_numpy(tm),
                'correspondences': torch.from_numpy(corr), 'pose': torch.from_numpy(pose).float(),
                'src_path': 'a.pth', 'tgt_path': 'b.pth', 'idx': 0, 'overlap_p': 0.5}
        seed += 1
        np.random.seed(seed); random.seed(seed); torch.manual_seed(seed)
        with Recorder() as rec:
            for t in (T.RigidPerturb(mode), T.Jitter(0.005), T.ShufflePoints(max_pts=max_pts), T.RandomSwap()):
                data = t(data)
        swapped = data['src_path'] == 'b.pth'
        if (mode, max_pts, swapped) in seen:
            continue
        seen.add((mode, max_pts, swapped))
        p = f'case{len(seen) - 1}/'
        out.update({p + 'mode': np.array(mode), p + 'max_pts': np.array(max_pts), p + 'in_src': src,
                    p + 'in_tgt': tgt, p + 'in_pose': pose, p + 'in_src_overlap': sm, p + 'in_tgt_overlap': tm,
                    p + 'in_corr': corr, p + 'swapped': np.array(swapped)})
        for i, (name, v) in enumerate(rec.log):
            out[p + f'draw{i:02d}_{name}'] = v
        for key in ('src_xyz', 'tgt_xyz', 'pose', 'src_overlap', 'tgt_overlap', 'correspondences'):
            out[p + 'out_' + key] = data[key].numpy()
        k += 1
    np.savez_compressed(os.path.join(HERE, 'augment.npz'), **out)
    print(f'{len(seen)} cases -> augment.npz')


if __name__ == '__main__':
    main()
