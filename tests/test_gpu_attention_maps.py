"""GPU tests of the attention-map recording (`TransformerCrossEncoder.record_attentions`, `get_attentions()`) and of
its kernel `regtr_mha_probs_avg` (ops.mha_probs_avg).

Accuracy rows use the fp32 yardstick (tests/grad_yardstick.py): against float64, the GPU map's error must stay
within 10x the fp32 torch oracle's error on the same inputs (+1e-6)."""
import numpy as np
import pytest
import torch

from attention_map_oracle import attention_maps, cross_encoder_layer_maps, head_probs, pad_maps
from conftest import load_golden, make_case
from grad_yardstick import Yardstick
from stage_oracle import record
from test_attention_maps_host import check_maps_against_golden

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')
H, E = 8, 256


# ------------------------------------------------------------------------------------------------ kernel alone

def _ragged(peaked, seed=0):
    """Self problems of lengths {1, 17, 64, 65, 731}; cross problems 40 <-> 130 and 77 <-> 0 (an empty key range and
    an empty query range).  Each problem writes into its own block of a flat buffer at an odd pitch (k_len + 3) after
    a gap of 5, so that everything outside the blocks can be checked."""
    g = torch.Generator().manual_seed(seed)
    self_lens = [1, 17, 64, 65, 731]
    s_off = np.concatenate([[0], np.cumsum(self_lens)]).tolist()
    probs = [(s_off[i], n, s_off[i], n) for i, n in enumerate(self_lens)]
    c_lens = [40, 130, 77, 0]
    c_off = (s_off[-1] + np.concatenate([[0], np.cumsum(c_lens)])).tolist()
    probs += [(c_off[0], 40, c_off[1], 130), (c_off[1], 130, c_off[0], 40), (c_off[2], 77, c_off[3], 0),
              (c_off[3], 0, c_off[2], 77)]
    n = c_off[-1]
    qk = torch.randn(n, 2 * E, generator=g) * 1.5
    if peaked:          # scale q so that the largest score reaches ~40
        s_max = 0.0
        for q0, ql, k0, kl in probs:
            if ql and kl:
                s = (qk[q0:q0 + ql, :E].reshape(ql, H, 32).transpose(0, 1) @
                     qk[k0:k0 + kl, E:].reshape(kl, H, 32).permute(1, 2, 0)) / 32 ** 0.5
                s_max = max(s_max, float(s.abs().max()))
        qk[:, :E] *= 40.0 / s_max
    offs, pitch, at = [], [], 5
    for q0, ql, k0, kl in probs:
        offs.append(at); pitch.append(kl + 3); at += ql * (kl + 3) + 5
    return qk, probs, offs, pitch, at


def _launch(qk, probs, offs, pitch, numel, fill):
    qkd = qk.to(DEV)
    t = lambda i, dt=torch.int32: torch.tensor([p[i] for p in probs], dtype=dt, device=DEV)
    out = torch.full((numel,), fill, dtype=torch.float32, device=DEV)
    from regtr_b200 import ops
    ops.mha_probs_avg(qkd[:, :E], qkd[:, E:], out, torch.tensor(offs, dtype=torch.int64, device=DEV),
                      torch.tensor(pitch, dtype=torch.int32, device=DEV), t(0), t(1), t(2), t(3),
                      max(p[1] for p in probs), H)
    torch.cuda.synchronize()
    return out.cpu()


def _blocks(buf, probs, offs, pitch):
    return [buf[o:o + ql * pt].view(ql, pt)[:, :kl] if ql else buf[:0].view(0, kl)
            for (q0, ql, k0, kl), o, pt in zip(probs, offs, pitch)]


def _kernel_rows(case, got_blocks=None):
    qk, probs, offs, pitch, numel = case
    ys = Yardstick('regtr_mha_probs_avg vs float64')
    for j, ((q0, ql, k0, kl), got) in enumerate(zip(probs, got_blocks)):
        if not (ql and kl):
            continue
        q, k = qk[q0:q0 + ql, :E], qk[k0:k0 + kl, E:]
        ref = head_probs(q.double(), k.double(), H)
        ys.add(f'problem {j} ({ql} x {kl})', got, head_probs(q, k, H), ref)
    ys.report()
    return ys.failures()


@pytest.mark.parametrize('peaked', [False, True], ids=['plain', 'peaked'])
def test_probs_kernel_vs_float64(peaked):
    case = _ragged(peaked)
    qk, probs, offs, pitch, numel = case
    sentinel = -3.25
    buf = _launch(qk, probs, offs, pitch, numel, sentinel)
    blocks = _blocks(buf, probs, offs, pitch)
    assert not _kernel_rows(case, blocks)
    # rows sum to 1; nothing outside the blocks (padding columns, gaps, empty problems) is written
    written = torch.zeros(numel, dtype=torch.bool)
    for (q0, ql, k0, kl), o, pt, blk in zip(probs, offs, pitch, blocks):
        if ql and kl:
            assert (blk.double().sum(1) - 1).abs().max() <= 1e-5
            for r in range(ql):
                written[o + r * pt:o + r * pt + kl] = True
    assert torch.all(buf[~written] == sentinel)
    # zero-filled buffer: padding stays exactly 0 and the blocks are bit-identical to the first launch
    buf0 = _launch(qk, probs, offs, pitch, numel, 0.0)
    assert torch.all(buf0[~written] == 0)
    assert torch.equal(buf0[written], buf[written])


def test_probs_kernel_check_is_sharp():
    """A 1e-5 relative perturbation of the kernel's output fails the yardstick."""
    case = _ragged(False)
    qk, probs, offs, pitch, numel = case
    blocks = _blocks(_launch(qk, probs, offs, pitch, numel, 0.0), probs, offs, pitch)
    assert _kernel_rows(case, [b * (1 + 1e-5) for b in blocks])


# ------------------------------------------------------------------------------------------------ model level

def _model(case, **over):
    from regtr_b200.regtr import RegTR
    cfg, sd, src, tgt = make_case(case)
    for k, v in over.items():
        cfg[k] = v
    model = RegTR(cfg).to(DEV).eval()
    if over.get('pre_norm', cfg.pre_norm) != make_case(case)[0].pre_norm:
        sd = {k: v for k, v in sd.items() if k in model.state_dict()}     # no final norm without pre_norm
    model.load_state_dict(sd, strict=True)
    batch = lambda: {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src],
                     'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    return cfg, sd, src, tgt, model, batch


@pytest.mark.parametrize('case,pre_norm', [('fwd_modelnet_b1', True), ('fwd_3dmatch_small_b2', True),
                                           ('var_modelnet_postnorm_b1', False), ('fwd_3dmatch_small_b2', False)])
def test_layer_maps_vs_float64(case, pre_norm):
    """Every layer's four maps against float64 maps computed from that layer's recorded input (the model's own
    activations), pre-norm and post-norm."""
    cfg, sd, src, tgt, model, batch = _model(case, pre_norm=pre_norm)
    model.transformer_encoder.record_attentions = True
    with pytest.MonkeyPatch.context() as mp:
        rec = record(model, mp, inference=True)
        model(batch())
    torch.cuda.synchronize()
    ys = Yardstick(f'{case} pre_norm={pre_norm}: layer maps vs float64')
    for i, (box, layer) in enumerate(zip(rec['xenc'], model.transformer_encoder.layers)):
        x, (pos, plan) = box['x'].cpu(), box['rest']
        lens = plan.lens
        B = len(lens) // 2
        xs = torch.split(x[:sum(lens)], lens)
        ps = torch.split(pos[:sum(lens)].cpu(), lens) if pos is not None else [torch.zeros_like(v) for v in xs]
        want = {}
        for dt in (torch.float64, torch.float32):
            per = [[cross_encoder_layer_maps(sd, cfg, i, xs[b].to(dt), xs[B + b].to(dt), ps[b].to(dt),
                                             ps[B + b].to(dt))[2:] for b in range(B)]]
            want[dt] = pad_maps(per, max(lens[:B]), max(lens[B:]), dt)
        got = layer.satt_weights + layer.xatt_weights
        ref = want[torch.float64][0] + want[torch.float64][1]
        f32 = want[torch.float32][0] + want[torch.float32][1]
        for name, gm, fm, rm in zip(('src_satt', 'tgt_satt', 'src_xatt', 'tgt_xatt'), got, f32, ref):
            assert tuple(gm.shape) == tuple(rm.shape[1:])
            ys.add(f'layer {i} {name}', gm, fm[0], rm[0])
    ys.report()
    assert not ys.failures()


# The GPU forward meets the reference's features to FEAT_RTOL = 1e-4 of their maximum (tests/test_gpu_parity.py).
# Scores are bilinear in a layer's features: a relative error eps in q and k moves a score by at most 2 eps |s|, and
# a softmax row whose scores move by at most d moves each probability by at most 2 d (sum_k |dP_k| <= 2 d); the head
# average keeps that bound.  So a map entry may move by 4 FEAT_RTOL s_max, s_max the largest |score| of the case
# (from the float64 oracle).  Row sums are 1 to fp32 rounding.
FEAT_RTOL = 1e-4


@pytest.mark.parametrize('case', ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2', 'var_modelnet_postnorm_b1'])
def test_maps_match_reference_golden(case):
    cfg, sd, src, tgt, model, batch = _model(case)
    model.transformer_encoder.record_attentions = True
    b = batch()
    model(b)
    maps = model.transformer_encoder.get_attentions()
    lens = [int(v) for v in b['kpconv_meta']['_lens'][-1]]
    stats = {}
    attention_maps(sd, cfg, src, tgt, torch.float64, stats=stats)
    rtol = 4 * FEAT_RTOL * stats['s_max']
    print(f'{case}: s_max {stats["s_max"]:.2f}, map tolerance {rtol:.2e}')
    check_maps_against_golden(maps, lens, load_golden('attention'), case, rtol)


@pytest.mark.parametrize('extra', [0, 3])
def test_padded_adaptor_matches_packed(extra):
    """TransformerCrossEncoder.forward on padded (L, B, D) inputs with key-padding masks records the same maps as the
    packed path of RegTR.forward; padding beyond the longest cloud (extra) stays 0."""
    cfg, sd, src, tgt, model, batch = _model('fwd_3dmatch_small_b2')
    xenc = model.transformer_encoder
    xenc.record_attentions = True
    out = model(batch())
    packed = xenc.get_attentions()
    lens = [len(v) for v in out['src_feat_un']] + [len(v) for v in out['tgt_feat_un']]
    B = len(src)
    un = list(out['src_feat_un']) + list(out['tgt_feat_un'])
    with torch.no_grad():
        pe = torch.split(model.pos_embed(out.core['xyz_c'][:sum(lens)]), lens)
    Ls, Lt = max(lens[:B]) + extra, max(lens[B:]) + extra

    def pad(parts, L):
        t = torch.zeros((L, len(parts), E), device=DEV)
        for b, p in enumerate(parts):
            t[:len(p), b] = p
        return t

    def mask(ls, L):
        m = torch.ones((len(ls), L), dtype=torch.bool, device=DEV)
        for b, n in enumerate(ls):
            m[b, :n] = False
        return m
    with torch.no_grad():
        xenc(pad(un[:B], Ls), pad(un[B:], Lt), src_key_padding_mask=mask(lens[:B], Ls),
             tgt_key_padding_mask=mask(lens[B:], Lt), src_pos=pad(pe[:B], Ls), tgt_pos=pad(pe[B:], Lt))
    padded = xenc.get_attentions()
    for p_, q_ in zip(packed[0] + packed[1], padded[0] + padded[1]):
        r, c = p_.shape[2:]
        assert q_.shape[:2] == p_.shape[:2]
        assert torch.equal(q_[:, :, :r, :c], p_)
        assert torch.all(q_[:, :, r:] == 0) and torch.all(q_[:, :, :, c:] == 0)


def _core(out):
    return [out.core[k] for k in ('both_un', 'cond', 'corr', 'logit', 'pose')]


@pytest.mark.parametrize('impl', ['fp32', 'tf32_tc', 'bf16_tc'])
def test_recording_leaves_forward_unchanged(impl):
    from regtr_b200 import ops
    cfg, sd, src, tgt, model, batch = _model('fwd_3dmatch_small_b2', attention_impl=impl)
    fresh = _model('fwd_3dmatch_small_b2', attention_impl=impl)[4]
    xenc = model.transformer_encoder
    off = _core(model(batch()))
    xenc.record_attentions = True
    on1 = _core(model(batch()))
    maps1 = [m.clone() for pair in xenc.get_attentions() for m in pair]
    on2 = _core(model(batch()))
    maps2 = [m for pair in xenc.get_attentions() for m in pair]
    for a, b in zip(off, on1):
        assert torch.equal(a, b)
    for a, b in zip(on1, on2):
        assert torch.equal(a, b)
    for a, b in zip(maps1, maps2):
        assert torch.equal(a, b)
    for m in maps1:                 # valid rows of every map sum to 1
        rs = m.double().sum(-1)
        assert torch.all((rs == 0) | ((rs - 1).abs() <= 1e-5))
    # switched off: no maps, no map buffer, the launches of a model that never recorded
    xenc.record_attentions = False
    n0 = ops.LAUNCHES
    again = _core(model(batch()))
    n_off = ops.LAUNCHES - n0
    fresh(batch())                  # first call: one-time weight splits
    n0 = ops.LAUNCHES
    fresh(batch())
    n_fresh = ops.LAUNCHES - n0
    assert n_off == n_fresh
    for layer in xenc.layers:
        assert layer.satt_weights is None and layer.xatt_weights is None and not hasattr(layer, '_map_buf')
    for a, b in zip(off, again):
        assert torch.equal(a, b)
    with pytest.raises(RuntimeError, match='no attention maps recorded'):
        xenc.get_attentions()


def test_graphs_and_training_refuse_recording():
    from regtr_b200.regtr import GraphedRegTR
    cfg, sd, src, tgt, model, batch = _model('fwd_modelnet_b1')
    with pytest.raises(RuntimeError, match='no attention maps recorded'):
        model.transformer_encoder.get_attentions()
    model.transformer_encoder.record_attentions = True
    with pytest.raises(RuntimeError, match='record_attentions'):
        GraphedRegTR(model)(batch())
    with pytest.raises(RuntimeError, match='record_attentions'):
        model.forward_train(batch())
