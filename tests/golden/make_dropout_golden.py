"""Generate tests/golden/dropout.npz: the UNMODIFIED reference trained with dropout 0.1, with known masks.

Run where the reference is present:

    python tests/golden/make_dropout_golden.py

The reference RegTR (oracle/ref_bridge.py) is built with `dropout: 0.1` and the seeded weights and loss inputs of
tests/golden/eval_inputs.py (the weights of grad.npz); its cross-encoder runs in train mode, everything else in eval
mode.  While it runs, `torch.nn.functional.dropout` is replaced: `nn.Dropout` and the attention-weight dropout of
`F.multi_head_attention_forward` both call it, and the replacement serves, call by call, the masks of the keep rule
(tests/dropout_rule.py) at key (SEED, STEP, pair_base 0), mapped into the reference's padded layouts:
(B·H, L, S) for the attention weights (row b·H + h: pair b, head h), (L, B, D) for the other four sites.  It asserts
that the call order is the one of forward_pre (transformers.py:183-244) for every layer:
    self_attn(src) dropout1(src) self_attn(tgt) dropout1(tgt) multihead_attn(src) multihead_attn(tgt)
    dropout2(src) dropout2(tgt) dropout(src) dropout3(src) dropout(tgt) dropout3(tgt)
Stored per case: every loss value, per parameter the gradient's norm, sum and the entries of
`eval_inputs.grad_sample_index` (as grad.npz), and the log of the served masks (layer, site, side, pair, head,
rows, cols, number kept, CRC32 of the packed mask), which tests/test_dropout_host.py regenerates from the rule.
"""
from __future__ import annotations

import os
import sys
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import dropout_rule as R  # noqa: E402
import eval_inputs as ei  # noqa: E402
from make_golden import FORWARD_CASES, _np  # noqa: E402
from oracle import ref_bridge  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

P, SEED, STEP = 0.1, 20261017, 9
MODEL_CASES = ('fwd_modelnet_b1', 'fwd_3dmatch_small_b2')
# (site, side) of the 12 dropout calls of one layer, in forward_pre's order
LAYER_ORDER = [(1, 0), (2, 0), (1, 1), (2, 1), (3, 0), (3, 1), (4, 0), (4, 1), (5, 0), (6, 0), (5, 1), (6, 1)]


def mask_crc(m):
    return zlib.crc32(np.packbits(m.astype(bool)).tobytes())


class MaskServer:
    """Stand-in for F.dropout that serves the rule's masks in forward_pre's call order."""

    def __init__(self, s_lens, t_lens, n_layers, n_heads):
        self.s_lens, self.t_lens, self.H = s_lens, t_lens, n_heads
        self.B = len(s_lens)
        self.calls = [(layer, site, side) for layer in range(n_layers) for site, side in LAYER_ORDER]
        self.i, self.log = 0, []

    def __call__(self, input, p=0.5, training=True, inplace=False):
        if not training or p == 0.0:
            return input
        assert p == P, p
        layer, site, side = self.calls[self.i]
        self.i += 1
        B, H = self.B, self.H
        lens_q = self.s_lens if side == 0 else self.t_lens
        lens_o = self.t_lens if side == 0 else self.s_lens
        mask = torch.ones_like(input)
        if site in (1, 3):
            lens_k = lens_q if site == 1 else lens_o
            assert input.dim() == 3 and input.shape[0] == B * H, (layer, site, side, input.shape)
            assert input.shape[1] == max(lens_q) and input.shape[2] == max(lens_k), (layer, site, input.shape)
            for b in range(B):
                for h in range(H):
                    m = R.local_keep_mask(P, SEED, STEP, 0, B, b + side * B, layer, site, h, lens_q[b], lens_k[b])
                    mask[b * H + h, :lens_q[b], :lens_k[b]] = torch.from_numpy(m)
                    self.log.append([layer, site, side, b, h, lens_q[b], lens_k[b], int(m.sum()), mask_crc(m)])
        else:
            assert input.dim() == 3 and input.shape[1] == B and input.shape[0] == max(lens_q), (layer, site, input.shape)
            D = input.shape[2]
            for b in range(B):
                m = R.local_keep_mask(P, SEED, STEP, 0, B, b + side * B, layer, site, 0, lens_q[b], D)
                mask[:lens_q[b], b, :] = torch.from_numpy(m)
                self.log.append([layer, site, side, b, 0, lens_q[b], D, int(m.sum()), mask_crc(m)])
        return input * (mask * torch.tensor(R.scale(P), dtype=input.dtype))


def model_fixture(case, fx):
    cfg_name, wseed, makers = FORWARD_CASES[case][:3]
    cfg = get_config(cfg_name, dropout=P)
    sd = ei.loss_state_dict(random_state_dict(get_config(cfg_name), wseed))
    model = ref_bridge.build_reference_model(cfg, sd)              # strict=True
    model.eval()
    model.transformer_encoder.train()                               # the six dropouts on, nothing else in train mode
    for p_ in model.parameters():
        p_.requires_grad_(p_.is_floating_point())
    pairs = [mk() for mk in makers]
    batch = {'src_xyz': [torch.from_numpy(p['src_xyz']) for p in pairs],
             'tgt_xyz': [torch.from_numpy(p['tgt_xyz']) for p in pairs]}
    orig = torch.nn.functional.dropout
    server = {}

    def patched(input, p=0.5, training=True, inplace=False):
        return server['s'](input, p, training, inplace)
    # the coarse lengths are known only after the reference's preprocessing: wrap the encoder to read them
    enc = model.transformer_encoder
    enc_forward = enc.forward

    def enc_wrap(src, tgt, src_key_padding_mask=None, tgt_key_padding_mask=None, **kw):
        s_lens = (~src_key_padding_mask).sum(1).tolist()
        t_lens = (~tgt_key_padding_mask).sum(1).tolist()
        server['s'] = MaskServer(s_lens, t_lens, len(enc.layers), enc.layers[0].self_attn.num_heads)
        return enc_forward(src, tgt, src_key_padding_mask=src_key_padding_mask,
                           tgt_key_padding_mask=tgt_key_padding_mask, **kw)
    enc.forward = enc_wrap
    torch.nn.functional.dropout = patched
    try:
        pred = model(batch)
    finally:
        torch.nn.functional.dropout = orig
        del enc.forward
    s = server['s']
    assert s.i == len(s.calls), (s.i, len(s.calls))
    batch.update(ei.loss_inputs(pairs, [int(x.shape[0]) for x in batch['src_xyz']],
                                [int(x.shape[0]) for x in batch['tgt_xyz']]))
    losses = model.compute_loss(pred, batch)
    losses['total'].backward()
    for k, v in losses.items():
        fx[f'{case}|loss_{k}'] = _np(v)
    fx[f'{case}|mask_log'] = np.array(s.log, dtype=np.int64)
    fx[f'{case}|key'] = np.array([SEED, STEP, 0], dtype=np.int64)
    fx[f'{case}|p'] = np.array(P)
    n = 0
    for name, p_ in model.named_parameters():
        if p_.grad is None:
            continue
        g = p_.grad.detach().double().reshape(-1)
        idx = ei.grad_sample_index(name, g.numel())
        fx[f'{case}|g|{name}'] = np.concatenate([[float(g.norm()), float(g.sum())], g[torch.from_numpy(idx)].numpy()])
        n += 1
    print(case, {k: float(v) for k, v in losses.items()}, 'parameters with a gradient:', n, 'dropout calls:', s.i)


if __name__ == '__main__':
    torch.manual_seed(0)
    fx = {}
    for case in MODEL_CASES:
        model_fixture(case, fx)
    path = os.path.join(HERE, 'dropout.npz')
    np.savez_compressed(path, **fx)
    print(path, os.path.getsize(path) // 1024, 'KiB')
