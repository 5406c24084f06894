"""Generate tests/golden/eval_dgr.npz by running the UNMODIFIED reference `benchmark_dgr`
(src/benchmark/benchmark_3dmatch.py) on seeded est.log files.

Run in the build container only (needs /root/reference):
    python tests/golden/make_dgr_golden.py

Two cases, each stored with the exact bytes of every est.log (and of the synthetic gt.log files) so that the tests
read the npz alone:
  real   the two scenes of tests/golden/real/benchmarks/3DMatch, one pair each: one estimate near the ground truth,
         one far from it (a scene without a success: the reference prints nan), est keys that differ from gt's;
  synth  the seeded scenes of eval_inputs.make_scenes: est.log lists a subset of the gt pairs, so the reference's
         by-position pairing scores estimates against other pairs' ground truth.
The reference module uses `np.float`, removed in numpy 1.24: a shim restores it for the run.
"""
import importlib.util
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import eval_inputs as ei  # noqa: E402

REF = '/root/reference/src/benchmark/benchmark_3dmatch.py'
REAL_GT = os.path.join(HERE, 'real', 'benchmarks', '3DMatch')


def reference_module():
    if not hasattr(np, 'float'):
        np.float = float                      # the reference's read_trajectory uses np.float
    spec = importlib.util.spec_from_file_location('ref_benchmark_3dmatch', REF)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def est_text(entries):
    """est.log bytes (generic_reg_model.py:_save_3DMatch_log format)."""
    s = ''
    for tgt, src, T in entries:
        s += '{}\t{}\t{}\n'.format(tgt, src, -1)
        for i in range(4):
            s += '\t'.join(map('{0:.12f}'.format, T[i])) + '\n'
    return s.encode()


def gt_text(pairs, gt, n_frag):
    s = ''
    for (i, j), T in zip(pairs, gt):
        s += f'{i}\t{j}\t{n_frag}\n'
        for r in range(4):
            s += '\t'.join('{0:.12e}'.format(v) for v in T[r]) + '\n'
    return s.encode()


def real_case():
    rng = np.random.default_rng(2024)
    scenes = sorted(os.listdir(REAL_GT))
    est = {}
    for k, scene in enumerate(scenes):
        lines = open(os.path.join(REAL_GT, scene, 'gt.log')).readlines()
        T = np.array([[float(v) for v in ln.split()] for ln in lines[1:5]])
        noise = ei._pose(rng, 2.0, 0.03) if k == 0 else ei._pose(rng, 60.0, 1.0)
        est[scene] = est_text([(k + 100, k + 200, T @ noise)])       # keys unrelated to gt's
    return scenes, est, {}


def synth_case():
    scenes = ei.make_scenes(seed=321)
    est = {s: est_text(d['est']) for s, d in scenes.items()}
    gt = {s: gt_text(d['pairs'], d['gt'], d['n_frag']) for s, d in scenes.items()}
    return sorted(scenes), est, gt


def write(folder, texts, name):
    for scene, b in texts.items():
        os.makedirs(os.path.join(folder, scene), exist_ok=True)
        with open(os.path.join(folder, scene, name), 'wb') as f:
            f.write(b)


def main():
    ref = reference_module()
    fx = {}
    for case, (scenes, est, gt) in (('real', real_case()), ('synth', synth_case())):
        with tempfile.TemporaryDirectory() as tmp:
            est_dir = os.path.join(tmp, 'est')
            write(est_dir, est, 'est.log')
            gt_dir = REAL_GT if not gt else os.path.join(tmp, 'gt')
            if gt:
                write(gt_dir, gt, 'gt.log')
            fx[f'{case}_summary'] = np.frombuffer(ref.benchmark_dgr(est_dir, gt_dir).encode('utf-8'), np.uint8)
            # the per-pair errors, with the reference's own compute_rre / compute_rte on the inverted poses
            for scene in scenes:
                _, et = ref.read_trajectory(os.path.join(est_dir, scene, 'est.log'))
                _, gtr = ref.read_trajectory(os.path.join(gt_dir, scene, 'gt.log'))
                ei_, gi = [np.linalg.inv(t) for t in et], [np.linalg.inv(gtr[i]) for i in range(len(et))]
                fx[f'{case}_rre_{scene}'] = np.array([ref.compute_rre(a[:3, :3], b[:3, :3]) for a, b in zip(ei_, gi)])
                fx[f'{case}_rte_{scene}'] = np.array([ref.compute_rte(a[:3, 3], b[:3, 3]) for a, b in zip(ei_, gi)])
        fx[f'{case}_scenes'] = np.array(scenes)
        for scene in scenes:
            fx[f'{case}_est_{scene}'] = np.frombuffer(est[scene], np.uint8)
            if gt:
                fx[f'{case}_gt_{scene}'] = np.frombuffer(gt[scene], np.uint8)
    out = os.path.join(HERE, 'eval_dgr.npz')
    np.savez_compressed(out, **fx)
    print('wrote', out)
    for case in ('real', 'synth'):
        print(fx[f'{case}_summary'].tobytes().decode())


if __name__ == '__main__':
    main()
