"""Tests of the device loss (regtr_b200/csrc/loss.cu, losses.compute_loss_device) against the torch restatement
`losses.compute_loss` evaluated in float64 on CPU copies of the same predictions, under the fp32 yardstick
(tests/grad_yardstick.py): the device route passes when its error is within 10x the error of the fp32 torch route on
the same inputs, plus 1e-6.  One CPU test pins the float64 restatement itself to the reference's loss.npz."""
import math
import os
import sys
import types
import warnings
from unittest import mock

import numpy as np
import pytest
import torch

from conftest import FORWARD_CASES, load_golden, make_case
from grad_yardstick import Yardstick

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

from regtr_b200 import losses as LS  # noqa: E402

DEV = 'cuda:0'
PACKED = ('both_un', 'cond', 'corr', 'logit')
CASES = ['fwd_modelnet_b1', 'fwd_3dmatch_small_b2']


# ------------------------------------------------------------------------------------------ the torch yardstick

def _torch_route(cfg, core, W, W_un, batch, lens_c, dtype, pyr=None, grad=False):
    """`losses.compute_loss` in `dtype` on CPU copies of the packed predictions (cut into per-cloud views exactly as
    the model does).  pyr: overlap pyramid to use instead of the route's own (so that both precisions weigh the tokens
    alike).  -> (losses, leaves): leaves are the packed tensors and the two W, with .grad after a backward."""
    from regtr_b200.regtr import RegTR
    cast = lambda t: t.detach().cpu().to(dtype)
    leaves = {k: cast(core[k]).requires_grad_(grad) for k in PACKED}
    leaves['W'], leaves['W_un'] = cast(W).requires_grad_(grad), cast(W_un).requires_grad_(grad)
    c = dict({k: leaves[k] for k in PACKED}, xyz_c=cast(core['xyz_c']), pose=None)
    pred = RegTR._assemble(c, list(lens_c), len(lens_c) // 2)
    meta = batch['kpconv_meta']
    b = dict(kpconv_meta={k: [torch.as_tensor(np.asarray(v.cpu() if torch.is_tensor(v) else v)) for v in meta[k]]
                          for k in ('points', 'pools', 'stack_lengths')},
             pose=cast(batch['pose']), src_overlap=[m.cpu() for m in batch['src_overlap']],
             tgt_overlap=[m.cpu() for m in batch['tgt_overlap']])
    mo = types.SimpleNamespace(cfg=cfg, feature_criterion=types.SimpleNamespace(W=leaves['W']),
                               feature_criterion_un=types.SimpleNamespace(W=leaves['W_un']))
    if pyr is None:
        out = LS.compute_loss(mo, pred, b)
    else:
        fixed = {k: cast(v) for k, v in pyr.items()}
        with mock.patch.object(LS, 'compute_overlaps', lambda _b: fixed):
            out = LS.compute_loss(mo, pred, b)
    return out, leaves, b


def _pyramid64(batch):
    """compute_overlaps in float64, slots summed in ascending order."""
    meta = batch['kpconv_meta']
    out = [torch.cat(list(batch['src_overlap']) + list(batch['tgt_overlap'])).cpu().double()]
    for p in range(1, len(meta['points'])):
        pool = meta['pools'][p - 1]
        pool = torch.as_tensor(np.asarray(pool.cpu() if torch.is_tensor(pool) else pool)).long()
        valid = pool < out[-1].shape[0]
        g = out[-1][pool.clamp_max(out[-1].shape[0] - 1)] * valid
        out.append((g.sum(1) / valid.sum(1)).clamp(0, 1))
    return out


def test_float64_restatement_matches_the_reference_losses():
    """The yardstick itself: `_torch_route` in float64 on the oracle's forward equals the unmodified reference's
    compute_loss (loss.npz)."""
    from oracle import regtr_oracle as O
    from regtr_b200.synthetic import make_modelnet_pair
    fx = load_golden('loss')
    cfg, sd, src, tgt = make_case('fwd_modelnet_b1')
    sd = ei.loss_state_dict(sd)
    pred = O.forward(sd, cfg, src, tgt)
    cat = lambda a, b, dim: torch.cat([torch.as_tensor(np.asarray(t)) for t in list(pred[a]) + list(pred[b])], dim=dim)
    core = dict(both_un=cat('src_feat_un', 'tgt_feat_un', 0), cond=cat('src_feat', 'tgt_feat', 1),
                corr=cat('src_kp_warped', 'tgt_kp_warped', 1), logit=cat('src_overlap', 'tgt_overlap', 1),
                xyz_c=cat('src_kp', 'tgt_kp', 0))
    batch = {'kpconv_meta': pred['kpconv_meta']}
    batch.update(ei.loss_inputs([make_modelnet_pair(1000)], [len(src[0])], [len(tgt[0])]))
    lens_c = [int(v) for v in np.asarray(pred['kpconv_meta']['stack_lengths'][-1])]
    out, _, b = _torch_route(cfg, core, sd['feature_criterion.W'], sd['feature_criterion_un.W'], batch, lens_c,
                             torch.float64)
    assert list(out) == ['overlap_5', 'feature_5', 'feature_un', 'corr_5', 'total']
    for k, v in out.items():
        np.testing.assert_allclose(float(v), float(fx[f'loss_{k}']), rtol=2e-4, err_msg=k)
    for lvl, want in enumerate(_pyramid64(batch)):
        np.testing.assert_allclose(want.numpy(), fx[f'overlap_pyr_{lvl}'], atol=1e-6)


# ------------------------------------------------------------------------------------------------ GPU fixtures

def _model(case, **over):
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    for k, v in over.items():
        cfg[k] = v
    model = RegTR(cfg).to(DEV)
    model.load_state_dict(ei.loss_state_dict(sd0), strict=True)
    model.kpf_encoder.requires_grad_(False)
    return cfg, model, src, tgt


def _batch(case, src, tgt):
    from regtr_b200.synthetic import make_3dmatch_pair, make_modelnet_pair
    pairs = [(make_modelnet_pair if kind == 'modelnet' else make_3dmatch_pair)(*args)
             for kind, args in FORWARD_CASES[case][2]]
    b = {'src_xyz': [torch.from_numpy(s).to(DEV) for s in src], 'tgt_xyz': [torch.from_numpy(t).to(DEV) for t in tgt]}
    li = ei.loss_inputs(pairs, [len(s) for s in src], [len(t) for t in tgt])
    b['pose'] = li['pose'].to(DEV)
    b['src_overlap'] = [m.to(DEV) for m in li['src_overlap']]
    b['tgt_overlap'] = [m.to(DEV) for m in li['tgt_overlap']]
    return b


def _leaf_pred(model, pred, batch):
    """The same predictions as detached packed leaves, cut into views again: the loss alone."""
    from regtr_b200.regtr import RegTR
    core = {k: (v.detach().clone().requires_grad_(True) if k in PACKED else v) for k, v in pred.core.items()}
    lens_c = batch['kpconv_meta']['_lens'][-1]
    return RegTR._assemble(core, lens_c, len(lens_c) // 2), core


def _device_loss_and_grads(model, pred, batch):
    model.zero_grad(set_to_none=True)
    leaf, core = _leaf_pred(model, pred, batch)
    out = model.compute_loss(leaf, batch)
    out['total'].backward()
    grads = {k: core[k].grad for k in PACKED}
    grads['W'], grads['W_un'] = model.feature_criterion.W.grad, model.feature_criterion_un.W.grad
    return out, grads


def _compare(cfg, model, pred, batch, title):
    """Values and gradients of the device route against the float64 torch route, under the yardstick."""
    assert LS.device_route(model, pred, batch)
    out, grads = _device_loss_and_grads(model, pred, batch)
    lens_c = batch['kpconv_meta']['_lens'][-1]
    W, W_un = model.feature_criterion.W, model.feature_criterion_un.W
    pyr = {k: v.cpu() for k, v in batch['overlap_pyr'].items()}
    ref = {}
    for dtype in (torch.float64, torch.float32):
        o, leaves, _ = _torch_route(cfg, pred.core, W, W_un, batch, lens_c, dtype, pyr=pyr, grad=True)
        o['total'].backward()
        ref[dtype] = (o, leaves)
    o64, o32 = ref[torch.float64][0], ref[torch.float32][0]
    assert list(out) == list(o64)
    ys = Yardstick(title)
    for k in out:
        assert out[k].dim() == 0 and out[k].dtype == torch.float32 and out[k].is_cuda
        ys.add(k, out[k], o32[k], o64[k])
    l64, l32 = ref[torch.float64][1], ref[torch.float32][1]
    for k, g in grads.items():
        assert g is not None and g.shape == l64[k].shape, k
        if float(l64[k].grad.abs().max()) == 0.0:
            assert int(torch.count_nonzero(g)) == 0, k
        else:
            ys.add('d ' + k, g, l32[k].grad, l64[k].grad)
    ys.report()
    assert not ys.failures(), ys.failures()
    for k in ('W', 'W_un'):                                  # the gradient of triu(W): nothing below the diagonal
        assert int(torch.count_nonzero(grads[k].tril(-1))) == 0
    off = [l for l in range(cfg.num_encoder_layers) if l not in cfg.feature_loss_on]
    assert int(torch.count_nonzero(grads['cond'][off])) == 0
    return out, grads


@pytest.fixture(scope='module', params=CASES)
def case(request):
    cfg, model, src, tgt = _model(request.param)
    batch = _batch(request.param, src, tgt)
    pred = model.forward_train(batch)
    return types.SimpleNamespace(name=request.param, cfg=cfg, model=model, src=src, tgt=tgt, batch=batch, pred=pred)


# ------------------------------------------------------------------------------------------------------- tests

@pytest.mark.gpu
def test_values_gradients_and_determinism(case):
    """(1), (3), (7): every loss value and d total / d (both_un, cond, corr, logit, W, W_un) against float64; the
    pyramid; a second run is bit-identical."""
    out, grads = _compare(case.cfg, case.model, case.pred, case.batch, f'device loss, {case.name}')
    assert int(torch.count_nonzero(grads['W_un'])) == 0      # wt_feature_un = 0.0: a zero tensor, not None
    # overlap pyramid: levels 0 and 1 bit-equal to the torch route's, deeper levels against float64
    dev_pyr = {k: v.cpu() for k, v in case.batch['overlap_pyr'].items()}
    _, _, b = _torch_route(case.cfg, case.pred.core, case.model.feature_criterion.W, case.model.feature_criterion_un.W,
                           case.batch, case.batch['kpconv_meta']['_lens'][-1], torch.float32)
    p64 = _pyramid64(case.batch)
    assert len(dev_pyr) == len(p64) == len(b['overlap_pyr'])
    for lvl, want in enumerate(p64):
        got = dev_pyr[f'pyr_{lvl}']
        assert got.dtype == torch.float32 and got.shape == want.shape
        if lvl <= 1:
            assert torch.equal(got, b['overlap_pyr'][f'pyr_{lvl}']), lvl
        assert float((got.double() - want).abs().max()) <= 1e-6, lvl
    out2, grads2 = _device_loss_and_grads(case.model, case.pred, case.batch)
    for k in out:
        assert torch.equal(out[k], out2[k]) or (torch.isnan(out[k]) and torch.isnan(out2[k])), k
    for k in grads:
        assert torch.equal(grads[k], grads2[k]), k


@pytest.mark.gpu
def test_geometry_matches_cdist_topk_away_from_thresholds(case, monkeypatch):
    """(2) The inputs hold no distance within 1e-6 relative of r_p or r_n and no tied nearest neighbour (checked in
    float64); then positives, anchors and per-pair anchor counts equal the cdist / topk ones."""
    from regtr_b200 import ops
    seen = {}
    real = ops.loss_forward

    def record(*a, **k):
        seen['st'] = real(*a, **k)
        return seen['st']
    monkeypatch.setattr(ops, 'loss_forward', record)
    with torch.no_grad():
        LS.compute_loss_device(case.model, case.pred, case.batch)
    st = seen['st']
    lens = case.batch['kpconv_meta']['_lens'][-1]
    B = len(lens) // 2
    xyz = torch.split(case.pred.core['xyz_c'].cpu(), lens)
    src_gt = LS.se3_transform_list(case.batch['pose'].cpu(), list(xyz[:B]))
    offs = np.concatenate([[0], np.cumsum(lens)])
    pos, anchor, n_anchor = st['pos'].cpu(), st['anchor'].cpu(), st['n_anchor'].cpu()
    for b in range(B):
        d64 = torch.cdist(src_gt[b].double(), xyz[B + b].double(), compute_mode='donot_use_mm_for_euclid_dist')
        for r in (case.cfg.r_p, case.cfg.r_n):
            assert float((d64 / r - 1).abs().min()) > 1e-6
        two = d64.topk(2, dim=-1, largest=False).values
        assert float((two[:, 1] - two[:, 0]).min()) > 0
        d1, i1 = torch.cdist(src_gt[b], xyz[B + b]).topk(k=1, dim=-1, largest=False)
        rows = slice(int(offs[b]), int(offs[b + 1]))
        assert torch.equal(pos[rows].long(), i1[:, 0] + int(offs[B + b]))
        mask = d1[:, 0] < case.cfg.r_p
        assert torch.equal(anchor[rows].bool(), mask)
        assert int(n_anchor[b]) == int(mask.sum()) > 0


def _synthetic(lens, seed=0, pose=None, xyz=None, w=None, r_p=0.5, r_n=1.0, nl=2, on=(1,)):
    """Seeded packed predictions for clouds of the given lengths -> arguments of ops.loss_forward."""
    from regtr_b200 import ops
    g = torch.Generator().manual_seed(seed)
    B, N = len(lens) // 2, sum(lens)
    rnd = lambda *s: torch.randn(*s, generator=g)
    xyz = rnd(N, 3) * 0.3 if xyz is None else xyz
    if pose is None:
        pose = torch.cat([torch.eye(3), torch.zeros(3, 1)], 1).repeat(B, 1, 1)
    w = torch.rand(N, generator=g) if w is None else w
    offs = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32)
    geo = ops.LossGeometry(xyz.to(DEV), offs.to(DEV), lens, pose.contiguous().to(DEV), w.to(DEV), on, on, on, r_p, r_n)
    args = [rnd(N, 256) * 0.2, rnd(nl, N, 256) * 0.2, rnd(nl, N, 3), rnd(nl, N, 1), rnd(256, 256) * 0.1, rnd(256, 256) * 0.1]
    return [t.to(DEV) for t in args] + [geo]


@pytest.mark.gpu
def test_geometry_rule_at_the_threshold_and_at_a_tie():
    """(2) The kernel's own rule: strictly below r_p, ties to the lowest target index."""
    from regtr_b200 import ops
    xyz = torch.tensor([[0., 0, 0], [10, 0, 0], [20, 0, 0],                           # sources
                        [-0.5, 0, 0], [0.5, 0, 0], [10.25, 0, 0], [9.75, 0, 0], [20.375, 0, 0]])
    st = ops.loss_forward(*_synthetic([3, 5], xyz=xyz, r_p=0.5, r_n=1.0))
    assert st['pos'][:3].tolist() == [3, 5, 7]          # equidistant targets: the lower index
    assert st['anchor'][:3].tolist() == [0, 1, 1]       # a nearest target at exactly r_p is no anchor
    assert int(st['n_anchor'][0]) == 2 and bool(torch.isfinite(st['vals']).all())


@pytest.mark.gpu
def test_more_layers_and_a_live_feature_un_term():
    """(3) wt_feature_un = 0.3, feature losses on layers 3 and 5, overlap and correspondence losses on 4 and 5: several
    terms and layers through the batched launches."""
    name = 'fwd_3dmatch_small_b2'
    cfg, model, src, tgt = _model(name, wt_feature_un=0.3, feature_loss_on=[3, 5], overlap_loss_on=[4, 5],
                                  corr_loss_on=[4, 5])
    batch = _batch(name, src, tgt)
    pred = model.forward_train(batch)
    out, grads = _compare(cfg, model, pred, batch, 'device loss, layers [3, 5] / [4, 5] and feature_un')
    assert list(out) == ['overlap_4', 'overlap_5', 'feature_3', 'feature_5', 'feature_un', 'corr_4', 'corr_5', 'total']
    assert int(torch.count_nonzero(grads['W_un'])) > 0 and int(torch.count_nonzero(grads['both_un'])) > 0


@pytest.mark.gpu
def test_end_to_end_parameter_gradients_match_the_torch_route(case):
    """(4) forward_train(train_encoder=True) -> compute_loss -> backward(): the device route and `losses.compute_loss`
    on the same pred reach the same parameters (all but the kernel points), and every gradient agrees to 1e-4 of its
    norm.  Both go through the same backward kernels; the loss gradients themselves are held against float64 above."""
    model = case.model
    for n, p in model.kpf_encoder.named_parameters():
        p.requires_grad_(not n.endswith('kernel_points'))
    try:
        got = {}
        for route in ('device', 'torch'):
            model.zero_grad(set_to_none=True)
            batch = _batch(case.name, case.src, case.tgt)
            pred = model.forward_train(batch, train_encoder=True)
            fn = model.compute_loss if route == 'device' else (lambda p, b: LS.compute_loss(model, p, b))
            fn(pred, batch)['total'].backward()
            got[route] = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    finally:
        model.kpf_encoder.requires_grad_(False)
        model.zero_grad(set_to_none=True)
    want = {n for n, _ in model.named_parameters() if not n.endswith('kernel_points')}
    assert set(got['device']) == set(got['torch']) == want
    worst = 0.0
    for n in want:
        a, b = got['device'][n].double(), got['torch'][n].double()
        if float(b.norm()) == 0.0:
            assert float(a.norm()) == 0.0, n
            continue
        worst = max(worst, float((a - b).norm() / b.norm()))
        assert float((a - b).norm()) <= 1e-4 * float(b.norm()), (n, float((a - b).norm() / b.norm()))
    print('worst relative difference of a parameter gradient:', worst)


def _count_loss(model, pred, batch, mode):
    """(library launches of the loss forward, of its backward, synchronisations warned about)."""
    from regtr_b200 import ops
    model.zero_grad(set_to_none=True)
    leaf, _ = _leaf_pred(model, pred, batch)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode(mode)
        try:
            n0 = ops.LAUNCHES
            total = model.compute_loss(leaf, batch)['total']
            n1 = ops.LAUNCHES
            total.backward()
            n2 = ops.LAUNCHES
        finally:
            torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    return n1 - n0, n2 - n1, sum('synchroniz' in str(x.message) for x in w)


@pytest.mark.gpu
def test_no_host_sync_and_launches_independent_of_the_batch_size():
    """(5) The loss and its backward raise nothing under sync debug mode 'error'; their launch counts at one and two
    pairs are equal once the split-K reduction launch of a GEMM (chosen from the token count) is set aside; the torch
    route on the same pred synchronises."""
    from regtr_b200 import lib, ops
    L = lib.load()
    counts = {}
    for name in ('fwd_3dmatch_small_b1', 'fwd_3dmatch_small_b2'):
        cfg, model, src, tgt = _model(name)
        batch = _batch(name, src, tgt)
        pred = model.forward_train(batch)
        _count_loss(model, pred, batch, 0)                                    # warm-up: scratch, weight vector
        fwd, bwd, _ = _count_loss(model, pred, batch, 'error')
        lens = batch['kpconv_meta']['_lens'][-1]
        n_src, terms = sum(lens[:len(lens) // 2]), len(cfg.feature_loss_on) + 1
        split_q = int(L.regtr_gemm_ws_bytes(n_src, 256, 256) > 256)
        split_w = int(L.regtr_gemm_ws_bytes(256, 260, (n_src + 3) // 4 * 4) > 256)
        counts[name] = (fwd - terms * split_q, bwd - terms * (split_q + split_w))
        print(name, 'loss forward / backward launches:', fwd, bwd, 'of which split-K:', terms * split_q,
              terms * (split_q + split_w))
    assert counts['fwd_3dmatch_small_b1'] == counts['fwd_3dmatch_small_b2'], counts
    with mock.patch.object(LS, 'device_route', lambda *a: False):
        _, _, syncs = _count_loss(model, pred, batch, 'warn')
    assert syncs >= 1


@pytest.mark.gpu
def test_degenerate_inputs():
    """(6) A pair without an anchor gives NaN feature losses and leaves the other pair's results untouched; overlap
    weights summing to less than 1e-6 are divided by 1e-6; empty clouds are skipped."""
    from regtr_b200 import ops
    lens = [40, 33, 50, 37]
    eye = torch.cat([torch.eye(3), torch.zeros(3, 1)], 1)
    far = eye.clone(); far[:, 3] = 100.0
    a = ops.loss_forward(*_synthetic(lens, seed=1))
    b = ops.loss_forward(*_synthetic(lens, seed=1, pose=torch.stack([eye, far])))
    keys = a['keys']
    feat = [keys.index('feature_1'), keys.index('feature_un')]
    assert bool(torch.isfinite(a['vals']).all()) and int(a['n_anchor'].min()) > 0
    assert bool(torch.isnan(b['vals'][feat]).all()) and b['n_anchor'].tolist() == [int(a['n_anchor'][0]), 0]
    assert torch.equal(a['pair_loss'][:, 0], b['pair_loss'][:, 0]) and bool(torch.isnan(b['pair_loss'][:, 1]).all())
    assert bool(torch.isfinite(b['vals'][keys.index('overlap_1')]))
    d = ops.loss_backward(b, torch.ones(len(keys), device=DEV))              # no fault with NaN values around
    assert bool(torch.isfinite(d[3]).all())
    N = sum(lens)
    z = ops.loss_forward(*_synthetic(lens, seed=1, w=torch.zeros(N)))
    assert float(z['vals'][keys.index('corr_1')]) == 0.0
    w = torch.zeros(N); w[3] = 1e-9
    args = _synthetic(lens, seed=1, w=w)
    t = ops.loss_forward(*args)
    corr, xyz = args[2][1, 3].double().cpu(), args[6].xyz[3].double().cpu()
    want = 1e-9 * float((corr - xyz).abs().sum()) / 1e-6
    assert math.isclose(float(t['vals'][keys.index('corr_1')]), want, rel_tol=1e-5)
    for lens_e in ([5, 0, 7, 4], [5, 3, 7, 0], [0, 3, 0, 4]):
        e = ops.loss_forward(*_synthetic(lens_e, seed=2))
        ops.loss_backward(e, torch.ones(len(keys), device=DEV))
        torch.cuda.synchronize()
        assert bool(torch.isfinite(e['vals'][keys.index('overlap_1')]))
        assert bool(torch.isnan(e['vals'][feat]).all())


@pytest.mark.gpu
def test_validation_path_without_grad(case):
    """(8) On outputs of `forward` under no_grad the device route is taken, nothing requires grad, and the values hold
    against float64 of the same predictions."""
    model = case.model
    batch = _batch(case.name, case.src, case.tgt)
    with torch.no_grad():
        pred = model(batch)
        assert LS.device_route(model, pred, batch)
        out = model.compute_loss(pred, batch)
    assert not any(v.requires_grad for v in out.values())
    lens_c = batch['kpconv_meta']['_lens'][-1]
    pyr = {k: v.cpu() for k, v in batch['overlap_pyr'].items()}
    W, W_un = model.feature_criterion.W, model.feature_criterion_un.W
    o64 = _torch_route(case.cfg, pred.core, W, W_un, batch, lens_c, torch.float64, pyr=pyr)[0]
    o32 = _torch_route(case.cfg, pred.core, W, W_un, batch, lens_c, torch.float32, pyr=pyr)[0]
    ys = Yardstick(f'device loss without grad, {case.name}')
    for k in out:
        ys.add(k, out[k], o32[k], o64[k])
    ys.report()
    assert not ys.failures(), ys.failures()
