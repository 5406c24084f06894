"""Generate tests/golden/attention.npz: the UNMODIFIED reference's `TransformerCrossEncoder.get_attentions()`.

Run where the reference is present:

    python tests/golden/make_attention_golden.py

For `fwd_modelnet_b1`, `fwd_3dmatch_small_b2` (two uneven pairs: padding in both the query and the key dimension)
and the post-norm variant `var_modelnet_postnorm_b1`, the reference model (seeded weights, seeded pairs, as in
make_golden.py) runs its forward through oracle/ref_bridge.py and the four stacked maps of `get_attentions()` are
stored the way the forward fixtures store large tensors:
  * `{case}|lens`: the coarse cloud lengths (src x B, tgt x B);
  * per map m in (src_satt, tgt_satt, src_xatt, tgt_xatt): `|shape`, `|step` and `|rows` (every step-th element of the
    flattened (L, B, rows, cols) stack), `|sum` (fp64 checksum) and `|rowsum` (sum over the keys of every row).
The reference leaves arbitrary values in padded QUERY rows (softmax over the valid keys of a padded token); they are
set to 0 here, the layout the library records.  Padded KEY columns are 0 in the reference itself (asserted).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import FORWARD_CASES  # noqa: E402
from oracle import ref_bridge  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

CASES = ('fwd_modelnet_b1', 'fwd_3dmatch_small_b2', 'var_modelnet_postnorm_b1')
MAPS = ('src_satt', 'tgt_satt', 'src_xatt', 'tgt_xatt')
SAMPLES = 4000          # about this many sampled entries per map


def sample_step(numel):
    return max(1, numel // SAMPLES) | 1       # odd: the sample walks across rows and columns


def map_lens(lens, B):
    """(query lengths, key lengths) per batch element of each of MAPS."""
    s, t = lens[:B], lens[B:]
    return dict(src_satt=(s, s), tgt_satt=(t, t), src_xatt=(s, t), tgt_xatt=(t, s))


def fixture(case, fx):
    cfg_name, wseed, makers, *rest = FORWARD_CASES[case]
    cfg = get_config(cfg_name, **(rest[0] if rest else {}))
    model = ref_bridge.build_reference_model(cfg, random_state_dict(cfg, wseed))
    pairs = [mk() for mk in makers]
    out = ref_bridge.reference_forward(model, [p['src_xyz'] for p in pairs], [p['tgt_xyz'] for p in pairs])
    lens = [int(v) for v in out['kpconv_meta']['stack_lengths'][-1]]
    B = len(pairs)
    (ss, ts), (sx, tx) = model.transformer_encoder.get_attentions()
    fx[f'{case}|lens'] = np.array(lens, np.int32)
    ml = map_lens(lens, B)
    for name, m in zip(MAPS, (ss, ts, sx, tx)):
        a = m.detach().double().numpy().copy()           # (L, B, rows, cols)
        ql, kl = ml[name]
        for b in range(B):
            assert np.all(a[:, b, :ql[b], kl[b]:] == 0), (case, name, 'padded keys not 0 in the reference')
            a[:, b, ql[b]:, :] = 0.0
        step = sample_step(a.size)
        fx[f'{case}|{name}|shape'] = np.array(a.shape, np.int64)
        fx[f'{case}|{name}|step'] = np.array(step)
        fx[f'{case}|{name}|rows'] = a.reshape(-1)[::step].astype(np.float32)
        fx[f'{case}|{name}|sum'] = np.array(a.sum())
        fx[f'{case}|{name}|rowsum'] = a.sum(-1).astype(np.float32)
    print(case, lens, {n: tuple(fx[f'{case}|{n}|shape']) for n in MAPS})


if __name__ == '__main__':
    torch.manual_seed(0)
    fx = {}
    for case in CASES:
        fixture(case, fx)
    path = os.path.join(HERE, 'attention.npz')
    np.savez_compressed(path, **fx)
    print(path, os.path.getsize(path) // 1024, 'KiB')
