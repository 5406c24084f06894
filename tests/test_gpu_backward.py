"""GPU tests of the attention-core backward and of RegTR.forward_train: the op against float64 torch autograd of the
same math, bit-for-bit determinism, and the model's parameter gradients against the unmodified reference's own
backward (tests/golden/grad.npz) and against the CPU oracle's autograd.  The LayerNorm and dense-layer backward are
in tests/test_gpu_train_ops.py."""
import math
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import FORWARD_CASES, load_golden, make_case
from grad_yardstick import Yardstick

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'


def _rel(got, want):
    """max |got - want| / max |want|"""
    want = want.double()
    return float((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-30))


# ----------------------------------------------------------------------------------------------- attention core

def _tables(problems):
    cols = list(zip(*problems))
    return [torch.tensor(c, dtype=torch.int32, device=DEV) for c in cols]


def _attention_case(seed=0):
    """Self problems of lengths {1, 17, 64, 65, 731}, then cross problems over four clouds (40, 130, 77, 0 tokens):
    q_len != k_len, and an empty partner both as key range and as query range.  Every key row is in exactly one
    problem's key range."""
    g = torch.Generator().manual_seed(seed)
    self_lens = [1, 17, 64, 65, 731]
    s_off = np.concatenate([[0], np.cumsum(self_lens)]).tolist()
    self_p = [(s_off[i], n, s_off[i], n) for i, n in enumerate(self_lens)]
    c_lens = [40, 130, 77, 0]
    c_off = (s_off[-1] + np.concatenate([[0], np.cumsum(c_lens)])).tolist()
    cross_p = [(c_off[0], 40, c_off[1], 130), (c_off[1], 130, c_off[0], 40), (c_off[2], 77, c_off[3], 0),
               (c_off[3], 0, c_off[2], 77)]
    n = c_off[-1]
    E, H = 256, 8
    qkv = (torch.randn(n, 3 * E, generator=g) * 1.5).to(DEV)
    d_o = torch.randn(n, E, generator=g).to(DEV)
    return qkv, d_o, self_p, cross_p, E, H


def _attention_ref(qkv, d_o, problems, E, H, dtype=torch.float64):
    """autograd in `dtype`: (O, lse base 2, dqkv) restricted to the rows the problems cover."""
    x = qkv.cpu().to(dtype).requires_grad_(True)
    g = d_o.cpu().to(dtype)
    o = torch.zeros(x.shape[0], E, dtype=dtype)
    lse = torch.full((x.shape[0], H), -math.inf, dtype=dtype)
    for qs, ql, ks, kl in problems:
        if ql == 0:
            continue
        q = x[qs:qs + ql, :E].view(ql, H, 32).transpose(0, 1)
        k = x[ks:ks + kl, E:2 * E].view(kl, H, 32).transpose(0, 1)
        v = x[ks:ks + kl, 2 * E:].view(kl, H, 32).transpose(0, 1)
        if kl == 0:
            continue
        s = q @ k.transpose(1, 2) / math.sqrt(32)
        o[qs:qs + ql] = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(ql, E)
        lse[qs:qs + ql] = (torch.logsumexp(s, -1) / math.log(2)).transpose(0, 1).detach()
    (o * g).sum().backward()
    return o.detach(), lse, x.grad


@pytest.mark.parametrize('kind', ['self', 'cross'])
def test_attention_backward_matches_float64(kind):
    """O and lse within 1e-4·max of float64; dQ, dK, dV under the fp32 yardstick (tests/grad_yardstick.py)."""
    from regtr_b200 import ops
    qkv, d_o, self_p, cross_p, E, H = _attention_case()
    problems = self_p if kind == 'self' else cross_p
    qs, ql, ks, kl = _tables(problems)
    max_q = max(p[1] for p in problems)
    max_k = max(p[3] for p in problems)
    q, k, v = qkv[:, :E], qkv[:, E:2 * E], qkv[:, 2 * E:]
    o, lse = ops.mha_varlen_lse(q, k, v, qs, ql, ks, kl, max_q, H)
    o_inf = ops.mha_varlen(q, k, v, qs, ql, ks, kl, max_q, H)
    d = torch.zeros_like(qkv)
    ops.mha_varlen_bwd(q, k, v, o, lse, d_o, d[:, :E], d[:, E:2 * E], d[:, 2 * E:], qs, ql, ks, kl, max_q, max_k, H)
    torch.cuda.synchronize()
    o_ref, lse_ref, d_ref = _attention_ref(qkv, d_o, problems, E, H)
    rows = torch.cat([torch.arange(p[0], p[0] + p[1]) for p in problems])
    krows = torch.cat([torch.arange(p[2], p[2] + p[3]) for p in problems])
    assert torch.equal(o[rows.to(DEV)], o_inf[rows.to(DEV)])            # the lse entry computes the same O
    assert _rel(o.cpu()[rows], o_ref[rows]) <= 1e-4
    lg, lr = lse.cpu()[rows].double(), lse_ref[rows]
    assert torch.equal(torch.isinf(lg), torch.isinf(lr))
    fin = torch.isfinite(lr)
    errs = {}
    errs['lse'] = float((lg[fin] - lr[fin]).abs().max() / lr[fin].abs().max())
    dc, dr = d.cpu(), d_ref
    print(kind, errs)
    assert max(errs.values()) <= 1e-4, errs
    d32 = _attention_ref(qkv, d_o, problems, E, H, torch.float32)[2]
    ys = Yardstick(f'attention backward, {kind} problems')
    ys.add('dq', dc[rows, :E], d32[rows, :E], dr[rows, :E])
    ys.add('dk', dc[krows, E:2 * E], d32[krows, E:2 * E], dr[krows, E:2 * E])
    ys.add('dv', dc[krows, 2 * E:], d32[krows, 2 * E:], dr[krows, 2 * E:])
    ys.report()
    assert not ys.failures(), ys.failures()
    if kind == 'cross':                                  # empty key range -> dQ = 0; no queries -> dK = dV = 0
        e = cross_p[2]
        assert float(dc[e[0]:e[0] + e[1], :E].abs().max()) == 0.0
        assert float(dc[e[0]:e[0] + e[1], E:].abs().max()) == 0.0
    # determinism: a second backward is bit-identical
    d2 = torch.zeros_like(qkv)
    ops.mha_varlen_bwd(q, k, v, o, lse, d_o, d2[:, :E], d2[:, E:2 * E], d2[:, 2 * E:], qs, ql, ks, kl, max_q, max_k, H)
    assert torch.equal(d, d2)


# ------------------------------------------------------------------------------------------------ whole model

def _model(case, sd=None):
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    sd = ei.loss_state_dict(sd0) if sd is None else sd
    model = RegTR(cfg).to(DEV)
    model.load_state_dict(sd, strict=True)
    model.kpf_encoder.requires_grad_(False)
    return cfg, sd, model, src, tgt


def _pairs(case):
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    return [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
            for kind, args in FORWARD_CASES[case][2]]


def _batch(case, src, tgt):
    b = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    li = ei.loss_inputs(_pairs(case), [len(s) for s in src], [len(t) for t in tgt])
    b['pose'] = li['pose'].to(DEV)
    b['src_overlap'] = [m.to(DEV) for m in li['src_overlap']]
    b['tgt_overlap'] = [m.to(DEV) for m in li['tgt_overlap']]
    return b


def _check_grads(got, want_norm_and_samples, worst):
    """test_oracle_grad.py's criteria: norm within 1e-3 relative, 32 sampled entries within 5e-3 of the rms."""
    for name, g in got.items():
        want = want_norm_and_samples[name]
        g = g.detach().double().reshape(-1).cpu()
        idx = ei.grad_sample_index(name, g.numel())
        scale = max(want[0] / np.sqrt(g.numel()), 1e-12)
        nrm = abs(float(g.norm()) - want[0]) / max(want[0], 1e-30)
        err = np.abs(g[torch.from_numpy(idx)].numpy() - want[2:]).max() / scale
        worst['norm'] = max(worst['norm'], nrm)
        worst['entry'] = max(worst['entry'], err)
        assert abs(float(g.norm()) - want[0]) <= 1e-3 * want[0] + 1e-9, (name, float(g.norm()), want[0])
        assert err <= 5e-3, (name, err)


def test_forward_train_gradients_match_reference_backward():
    """fwd_modelnet_b1, encoder frozen: forward_train -> compute_loss -> backward() against the unmodified
    reference's d(total)/d(parameter) for every parameter after the encoder (grad.npz)."""
    fx = load_golden('grad')
    cfg, sd, model, src, tgt = _model('fwd_modelnet_b1')
    batch = _batch('fwd_modelnet_b1', src, tgt)
    pred = model.forward_train(batch)
    losses = model.compute_loss(pred, batch)
    total = losses['total']
    assert total.requires_grad
    np.testing.assert_allclose(float(total.detach()), float(fx['loss_total']), rtol=2e-5)
    total.backward()
    names = [k[2:] for k in fx if k.startswith('g|') and not k.startswith('g|kpf_encoder.')]
    assert len(names) == 122
    params = dict(model.named_parameters())
    assert all(p.grad is None for n, p in params.items() if n.startswith('kpf_encoder.'))
    want = {n: fx['g|' + n] for n in names}
    worst = dict(norm=0.0, entry=0.0)
    _check_grads({n: params[n].grad for n in names}, want, worst)
    print('worst vs reference backward:', worst)


def test_forward_train_gradients_match_oracle_3dmatch_b2(monkeypatch):
    """fwd_3dmatch_small_b2 (two pairs of different sizes: four uneven attention problems): every post-encoder
    parameter gradient and the gradient reaching the encoder output feats_un against the CPU oracle's autograd."""
    from oracle import regtr_oracle as O
    from regtr_b200 import losses as LS
    case = 'fwd_3dmatch_small_b2'
    cfg, sd, model, src, tgt = _model(case)
    # oracle side: post-encoder parameters and the encoder output as leaves
    sdo = {k: (v.clone().requires_grad_(not k.startswith('kpf_encoder.')) if v.is_floating_point() else v)
           for k, v in sd.items()}
    leaf = {}
    enc = O.encoder

    def encoder_leaf(*a, **k):
        leaf['f'] = enc(*a, **k).detach().requires_grad_(True)
        return leaf['f']
    monkeypatch.setattr(O, 'encoder', encoder_leaf)
    pred_o = O.forward(sdo, cfg, src, tgt)
    meta_o = pred_o['kpconv_meta']
    bo = {'kpconv_meta': {k: [torch.as_tensor(np.asarray(v)) for v in meta_o[k]] for k in ('points', 'pools', 'stack_lengths')}}
    bo.update(ei.loss_inputs(_pairs(case), [len(s) for s in src], [len(t) for t in tgt]))
    mo = types.SimpleNamespace(cfg=cfg, feature_criterion=types.SimpleNamespace(W=sdo['feature_criterion.W']),
                               feature_criterion_un=types.SimpleNamespace(W=sdo['feature_criterion_un.W']))
    total_o = LS.compute_loss(mo, pred_o, bo)['total']
    total_o.backward()
    # GPU side: the stages of forward_train with feats_un made a leaf
    from regtr_b200.transformer import AttentionPlan
    batch = _batch(case, src, tgt)
    B = len(src)
    with torch.no_grad():
        meta = model.preprocessor(list(batch['src_xyz']) + list(batch['tgt_xyz']), lazy_upsamples=True)
        batch['kpconv_meta'] = meta
        pts = meta['_points']
        feats_un, _ = model.kpf_encoder(torch.ones_like(pts[0][:, 0:1]), meta)
    feats_un.requires_grad_(True)
    lens_c = meta['_lens'][-1]
    core = model._stage_attention_train(feats_un, pts[-1], meta['_offs'][-1], B, AttentionPlan(lens_c, DEV))
    pred = model._assemble(core, lens_c, B)
    total = model.compute_loss(pred, batch)['total']
    np.testing.assert_allclose(float(total.detach()), float(total_o.detach()), rtol=2e-5)
    total.backward()
    got, want = {}, {}
    for n, p in model.named_parameters():
        if n.startswith('kpf_encoder.'):
            assert p.grad is None
            continue
        got[n] = p.grad
        ref = sdo[n].grad.double().reshape(-1)
        idx = ei.grad_sample_index(n, ref.numel())
        want[n] = np.concatenate([[float(ref.norm()), float(ref.sum())], ref[torch.from_numpy(idx)].numpy()])
    ref = leaf['f'].grad.double().reshape(-1)
    got['feats_un'] = feats_un.grad
    want['feats_un'] = np.concatenate([[float(ref.norm()), float(ref.sum())],
                                       ref[torch.from_numpy(ei.grad_sample_index('feats_un', ref.numel()))].numpy()])
    assert got['feats_un'].shape == leaf['f'].shape
    worst = dict(norm=0.0, entry=0.0)
    _check_grads(got, want, worst)
    print('worst vs oracle autograd:', worst)


def test_training_step_is_deterministic():
    cfg, sd, model, src, tgt = _model('fwd_modelnet_b1')
    grads = []
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        batch = _batch('fwd_modelnet_b1', src, tgt)
        model.compute_loss(model.forward_train(batch), batch)['total'].backward()
        grads.append({n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None})
    assert grads[0].keys() == grads[1].keys() and len(grads[0]) == 122
    for n in grads[0]:
        assert torch.equal(grads[0][n], grads[1][n]), n


def test_sgd_steps_follow_in_place_updates_and_reduce_the_loss():
    """After every optimizer.step() the inference forward equals that of a fresh model loaded with the state_dict
    (the split-weight caches follow in-place updates), and the loss goes down."""
    from regtr_b200.regtr import RegTR
    cfg, sd, model, src, tgt = _model('fwd_modelnet_b1')
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=2e-3)
    losses = []
    for step in range(4):
        batch = _batch('fwd_modelnet_b1', src, tgt)
        opt.zero_grad(set_to_none=True)
        total = model.compute_loss(model.forward_train(batch), batch)['total']
        losses.append(float(total.detach()))
        total.backward()
        opt.step()
        fresh = RegTR(cfg).to(DEV)
        fresh.load_state_dict(model.state_dict(), strict=True)
        a = model(_batch('fwd_modelnet_b1', src, tgt))
        b = fresh(_batch('fwd_modelnet_b1', src, tgt))
        for k in ('src_feat', 'tgt_overlap', 'src_kp_warped'):
            assert torch.equal(a[k][0], b[k][0]), (step, k)
        assert torch.equal(a['pose'], b['pose']), step
    print('losses', losses)
    assert losses[-1] < losses[0]


def test_inference_path_unchanged_and_unsupported_branches_raise():
    from regtr_b200.regtr import RegTR
    cfg, sd, model, src, tgt = _model('fwd_modelnet_b1')
    batch = _batch('fwd_modelnet_b1', src, tgt)
    out = model(batch)
    assert not any(t.requires_grad for k in ('src_feat', 'tgt_feat', 'src_kp_warped', 'src_overlap')
                   for t in out[k])
    assert not out['src_feat_un'][0].requires_grad and not out['pose'].requires_grad
    losses = model.compute_loss(out, batch)
    assert not any(v.requires_grad for v in losses.values())
    enc_live = RegTR(cfg).to(DEV)
    with pytest.raises(ValueError, match='requires_grad_'):
        enc_live.forward_train(_batch('fwd_modelnet_b1', src, tgt))
    for over in (dict(pre_norm=False), dict(direct_regress_coor=False), dict(pos_emb_type='learned'),
                 dict(attention_impl='tf32_tc'), dict(attention_impl='bf16_tc')):
        from regtr_b200.config import get_config
        m = RegTR(get_config('modelnet', **over)).to(DEV)
        m.kpf_encoder.requires_grad_(False)
        with pytest.raises(NotImplementedError):
            m.forward_train(_batch('fwd_modelnet_b1', src, tgt))
