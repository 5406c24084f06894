"""GPU tests of the circle feature loss on the library's kernels (regtr_circle_* in csrc/loss.cu, `feature_loss_type:
circle`): values and feature gradients against the float64 torch restatement `losses.circle_loss` under the fp32
yardstick (tests/grad_yardstick.py: within 10x the fp32 restatement's error, plus 1e-6), on the reference's loss-level
fixture sets (tests/golden/circle.npz) and on the model's own predictions; parameter gradients against the
unmodified reference's backward; determinism, launches and host syncs; the data-parallel normalisers; a trainer run."""
import os
import sys
import types
import warnings

import numpy as np
import pytest
import torch

from conftest import FORWARD_CASES, make_case
from grad_yardstick import Yardstick

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import eval_inputs as ei  # noqa: E402

from regtr_b200 import losses as LS  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'circle.npz')
PACKED = ('both_un', 'cond', 'corr', 'logit')


@pytest.fixture(scope='module')
def fx():
    return dict(np.load(GOLDEN))


# ------------------------------------------------------------------------------------------------------ op level

def _geometry(xyz, lens, r_p, r_n, norm=None):
    from regtr_b200 import ops
    B, N = len(lens) // 2, sum(lens)
    offs = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int32, device=DEV)
    pose = torch.cat([torch.eye(3), torch.zeros(3, 1)], 1).repeat(B, 1, 1).to(DEV)
    return ops.LossGeometry(xyz.to(DEV), offs, lens, pose, torch.zeros(N, device=DEV), [], [0], [], r_p, r_n,
                            norm=norm, feature_loss='circle')


def _op(feat, xyz, lens, r_p, r_n, norm=None):
    """One decoder layer whose features are `feat`, and feature_un on the same features: values (feature_0,
    feature_un) and d cond[0], d both_un for a unit upstream gradient."""
    from regtr_b200 import ops
    N = sum(lens)
    feat = feat.to(DEV)
    geo = _geometry(xyz, lens, r_p, r_n, norm)
    st = ops.loss_forward(feat, feat[None], torch.zeros(1, N, 3, device=DEV), torch.zeros(1, N, 1, device=DEV),
                          None, None, geo)
    d_un, d_cond, d_corr, d_logit, dW, dW_un = ops.loss_backward(st, torch.ones(2, device=DEV))
    assert dW is None and dW_un is None
    return st, d_cond[0], d_un


def _restated(feat, xyz, lens, r_p, r_n, dtype):
    B = len(lens) // 2
    f = feat.detach().cpu().to(dtype).requires_grad_(True)
    fs, xs = torch.split(f, lens), torch.split(xyz.cpu().to(dtype), lens)
    v = LS.circle_loss(list(fs[:B]), list(fs[B:]), list(xs[:B]), list(xs[B:]), r_p, r_n)
    v.backward()
    return v.detach(), f.grad


def _check_op(title, feat, xyz, lens, r_p, r_n):
    st, d_cond, d_un = _op(feat, xyz, lens, r_p, r_n)
    vals = st['vals']
    assert torch.equal(vals[0:1], vals[1:2]) or bool(torch.isnan(vals).all())
    assert torch.equal(d_cond, d_un)
    v64, g64 = _restated(feat, xyz, lens, r_p, r_n, torch.float64)
    v32, g32 = _restated(feat, xyz, lens, r_p, r_n, torch.float32)
    assert bool(torch.isnan(vals[0])) == bool(torch.isnan(v64)), (title, float(vals[0]), float(v64))
    ys = Yardstick(title)
    if not bool(torch.isnan(v64)):
        ys.add('value', vals[0], v32, v64)
    assert bool(torch.isfinite(d_cond).all())
    ys.add('d feat', d_cond, g32, g64)
    ys.report()
    assert not ys.failures(), ys.failures()
    return st, d_cond


@pytest.mark.parametrize('name', ['single', 'uneven', 'one_token', 'nan'])
def test_op_matches_float64_on_the_reference_sets(fx, name):
    """The reference's loss-level sets (both margins, both softplus branches, rows without a positive, a one-token
    cloud, uneven sizes, a pair with nothing selected): value and feature gradient under the yardstick; the value is
    NaN exactly where the reference's is, and the float64 restatement is the reference's value."""
    lens = [int(v) for v in fx[f'{name}|lens']]
    r_p, r_n = (float(v) for v in fx[f'{name}|radii'])
    feat, xyz = torch.from_numpy(fx[f'{name}|feat']), torch.from_numpy(fx[f'{name}|xyz'])
    st, d = _check_op(f'circle op, {name}', feat, xyz, lens, r_p, r_n)
    want = float(fx[f'{name}|value'])
    assert np.isnan(want) == bool(torch.isnan(st['vals'][0]))
    ref = torch.from_numpy(fx[f'{name}|grad']).double()
    assert float((d.cpu().double() - ref).abs().max() / ref.abs().max()) < 1e-3


def _synthetic(lens, seed=0):
    """Seeded features / key points like the fixture's: feature distances of geometric neighbours in ~[0.02, 2.5]."""
    rng = np.random.default_rng(seed)
    P = np.linalg.qr(rng.normal(size=(256, 3)))[0]
    xyz = rng.uniform(0.0, 1.5, (sum(lens), 3))
    lat = 0.3 * xyz + rng.choice([0.005, 0.3, 1.0], size=(sum(lens), 1)) * rng.normal(size=(sum(lens), 3))
    feat = lat @ P.T + 0.001 * rng.normal(size=(sum(lens), 256))
    return torch.from_numpy(feat.astype(np.float32)), torch.from_numpy(xyz.astype(np.float32))


def test_op_packed_batch_with_an_empty_target_cloud():
    """Three pairs packed, the second with no target token: its value is NaN (as the reference's empty mean), its
    source rows take no gradient, and the other pairs' rows hold against float64."""
    lens = [45, 18, 33, 40, 0, 27]
    feat, xyz = _synthetic(lens, seed=5)
    st, d = _check_op('circle op, packed batch with an empty target cloud', feat, xyz, lens, 0.35, 0.6)
    assert bool(torch.isnan(st['pair_loss'][:, 1]).all()) and bool(torch.isfinite(st['pair_loss'][:, [0, 2]]).all())
    assert int(torch.count_nonzero(d[45:63])) == 0
    assert st['n_sel'].tolist()[1] == 0 and st['n_sel'].tolist()[4] == 0


# ------------------------------------------------------------------------------------------------- model level

def _circle_model(case, **over):
    from regtr_b200.regtr import RegTR
    cfg, sd0, src, tgt = make_case(case)
    cfg['feature_loss_type'] = 'circle'
    for k, v in over.items():
        cfg[k] = v
    model = RegTR(cfg).to(DEV)
    model.load_state_dict({k: v for k, v in sd0.items() if not k.startswith('feature_criterion')}, strict=True)
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


def _leaf_pred(pred, batch):
    from regtr_b200.regtr import RegTR
    core = {k: (v.detach().clone().requires_grad_(True) if k in PACKED else v) for k, v in pred.core.items()}
    lens_c = batch['kpconv_meta']['_lens'][-1]
    return RegTR._assemble(core, lens_c, len(lens_c) // 2), core


def _torch_route(cfg, core, batch, dtype):
    """`losses.compute_loss` in `dtype` on CPU copies of the packed predictions, with the device route's overlap
    pyramid; -> (losses, leaves with .grad after backward)."""
    from unittest import mock
    from regtr_b200.regtr import RegTR
    cast = lambda t: t.detach().cpu().to(dtype)
    leaves = {k: cast(core[k]).requires_grad_(True) for k in PACKED}
    lens_c = batch['kpconv_meta']['_lens'][-1]
    pred = RegTR._assemble(dict(leaves, xyz_c=cast(core['xyz_c']), pose=None), list(lens_c), len(lens_c) // 2)
    meta = batch['kpconv_meta']
    b = dict(kpconv_meta={k: [torch.as_tensor(np.asarray(v.cpu() if torch.is_tensor(v) else v)) for v in meta[k]]
                          for k in ('points', 'pools', 'stack_lengths')},
             pose=cast(batch['pose']), src_overlap=[m.cpu() for m in batch['src_overlap']],
             tgt_overlap=[m.cpu() for m in batch['tgt_overlap']])
    fixed = {k: cast(v) for k, v in batch['overlap_pyr'].items()}
    with mock.patch.object(LS, 'compute_overlaps', lambda _b: fixed):
        out = LS.compute_loss(types.SimpleNamespace(cfg=cfg), pred, b)
    out['total'].backward()
    return out, leaves


@pytest.mark.parametrize('case,over', [('fwd_modelnet_b1', {}), ('fwd_3dmatch_small_b2', dict(wt_feature_un=0.3))])
def test_compute_loss_device_matches_float64(case, over):
    """compute_loss_device on the model's own predictions: every value and d total / d (both_un, cond, corr, logit)
    against the float64 torch route under the yardstick; a second run is bit-identical."""
    cfg, model, src, tgt = _circle_model(case, **over)
    batch = _batch(case, src, tgt)
    pred = model.forward_train(batch)
    assert LS.device_route(model, pred, batch)
    runs = []
    for _ in range(2):
        leaf, core = _leaf_pred(pred, batch)
        out = model.compute_loss(leaf, batch)
        out['total'].backward()
        runs.append((out, {k: core[k].grad for k in PACKED}))
    (out, grads), (out2, grads2) = runs
    for k in out:
        assert torch.equal(out[k], out2[k]), k
    for k in grads:
        assert torch.equal(grads[k], grads2[k]), k
    o64, l64 = _torch_route(cfg, pred.core, batch, torch.float64)
    o32, l32 = _torch_route(cfg, pred.core, batch, torch.float32)
    assert list(out) == list(o64) == ['overlap_5', 'feature_5', 'feature_un', 'corr_5', 'total']
    ys = Yardstick(f'circle device loss, {case} {over}')
    for k in out:
        assert bool(torch.isfinite(o64[k])), k
        ys.add(k, out[k], o32[k], o64[k])
    for k, g in grads.items():
        if float(l64[k].grad.abs().max()) == 0.0:
            assert int(torch.count_nonzero(g)) == 0, k
        else:
            ys.add('d ' + k, g, l32[k].grad, l64[k].grad)
    ys.report()
    assert not ys.failures(), ys.failures()
    assert (int(torch.count_nonzero(grads['both_un'])) > 0) == (cfg.wt_feature_un != 0)


def test_parameter_gradients_match_the_reference_backward(fx):
    """fwd_modelnet_b1 with the circle loss, encoder frozen: forward_train -> compute_loss -> backward() against the
    unmodified reference's d(total)/d(parameter) of every parameter after the encoder (norm within 1e-3, sampled
    entries within 5e-3 of the rms)."""
    case = 'fwd_modelnet_b1'
    cfg, model, src, tgt = _circle_model(case)
    batch = _batch(case, src, tgt)
    total = model.compute_loss(model.forward_train(batch), batch)['total']
    np.testing.assert_allclose(float(total.detach()), float(fx[f'{case}|loss_total']), rtol=2e-5)
    total.backward()
    names = [k.split('|g|')[1] for k in fx if k.startswith(f'{case}|g|') and '|g|kpf_encoder.' not in k]
    assert len(names) == 120                         # the 122 of the InfoNCE model less its two W
    params = dict(model.named_parameters())
    worst = dict(norm=0.0, entry=0.0)
    for name in names:
        want, g = fx[f'{case}|g|{name}'], params[name].grad.detach().double().reshape(-1).cpu()
        idx = ei.grad_sample_index(name, g.numel())
        scale = max(want[0] / np.sqrt(g.numel()), 1e-12)
        err = np.abs(g[torch.from_numpy(idx)].numpy() - want[2:]).max() / scale
        worst['norm'] = max(worst['norm'], abs(float(g.norm()) - want[0]) / max(want[0], 1e-30))
        worst['entry'] = max(worst['entry'], err)
        assert abs(float(g.norm()) - want[0]) <= 1e-3 * want[0] + 1e-9, (name, float(g.norm()), want[0])
        assert err <= 5e-3, (name, err)
    print('worst vs reference backward:', worst)


def _count_loss(model, pred, batch, mode):
    """(library launches of the loss forward, of its backward, synchronisations warned about)."""
    from regtr_b200 import ops
    model.zero_grad(set_to_none=True)
    leaf, _ = _leaf_pred(pred, batch)
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


def test_no_host_sync_and_launches_independent_of_the_batch_size():
    """The circle loss and its backward raise nothing under sync debug mode 'error', and launch as often at one
    pair as at two (no GEMM: nothing depends on the token count)."""
    counts = {}
    for name in ('fwd_3dmatch_small_b1', 'fwd_3dmatch_small_b2'):
        cfg, model, src, tgt = _circle_model(name)
        batch = _batch(name, src, tgt)
        pred = model.forward_train(batch)
        _count_loss(model, pred, batch, 0)                                    # warm-up: scratch, weight vector
        fwd, bwd, syncs = _count_loss(model, pred, batch, 'error')
        counts[name] = (fwd, bwd)
        print(name, 'circle loss forward / backward launches:', fwd, bwd)
    assert counts['fwd_3dmatch_small_b1'] == counts['fwd_3dmatch_small_b2'], counts


# ------------------------------------------------------------------------------------------------ data parallel

def test_norm_entries_and_slices_add_up():
    """With the call's own normalisers the _norm entries are bit-identical to the plain ones; two one-pair slices,
    each given the summed normalisers, add up to the two-pair batch's values and give its gradients."""
    from regtr_b200 import ops
    lens = [37, 29, 41, 33]
    feat, xyz = _synthetic(lens, seed=7)
    st, d, _ = _op(feat, xyz, lens, 0.35, 0.6)
    own = ops.loss_norms(_geometry(xyz, lens, 0.35, 0.6))
    st_n, d_n, _ = _op(feat, xyz, lens, 0.35, 0.6, norm=own)
    assert torch.equal(st['vals'], st_n['vals']) and torch.equal(d, d_n)
    offs = np.concatenate([[0], np.cumsum(lens)])
    rows = [np.r_[offs[0]:offs[1], offs[2]:offs[3]], np.r_[offs[1]:offs[2], offs[3]:offs[4]]]
    parts = [(feat[torch.from_numpy(r)], xyz[torch.from_numpy(r)], [lens[b], lens[2 + b]]) for b, r in enumerate(rows)]
    norms = [ops.loss_norms(_geometry(x, l, 0.35, 0.6)) for _, x, l in parts]
    total = norms[0] + norms[1]
    vals, grad = torch.zeros_like(st['vals']), torch.zeros_like(d)
    for (f, x, l), r in zip(parts, rows):
        s, g, _ = _op(f, x, l, 0.35, 0.6, norm=total.clone())
        vals += s['vals']
        grad[torch.from_numpy(r).to(DEV)] = g
    torch.testing.assert_close(vals, st['vals'], rtol=1e-6, atol=0)
    assert torch.equal(grad, d)


# ------------------------------------------------------------------------------------------------------- trainer

def test_trainer_runs_the_circle_loss_and_its_checkpoint_loads_strictly(tmp_path):
    """Three steps of Trainer.fit on synthetic ModelNet pairs with feature_loss_type='circle', then a validation:
    finite feature_5 and feature_un at every step and in validation, and the checkpoint the validation saves loads
    strictly into a fresh circle model."""
    from regtr_b200 import modelnet as MN
    from regtr_b200 import trainer as T
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.synthetic import make_modelnet_shapes
    from regtr_b200.weights import random_state_dict
    cfg = get_config('modelnet', train_batch_size=2, val_batch_size=2, feature_loss_type='circle', wt_feature_un=0.1)
    opt = types.SimpleNamespace(log_path=str(tmp_path / 'log'), resume=None, debug=False, summary_every=1000,
                                validate_every=3, nb_sanity_val_steps=0, num_workers=2)
    trainer = T.Trainer(opt, niter=3, grad_clip=cfg.grad_clip, seed=6)
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, 11), strict=True)
    seen = []
    real = model.compute_loss

    def record(pred, b):
        losses = real(pred, b)
        seen.append(torch.stack([losses['feature_5'].detach(), losses['feature_un'].detach()]))
        return losses
    model.compute_loss = record
    val_set = MN.ModelNetPairs(MN.ModelNetShapes.from_arrays(make_modelnet_shapes(2, seed=42)), cfg)
    trainer.fit(model, MN.ModelNetShapes.from_arrays(make_modelnet_shapes(5, seed=41)), val_set)  # 3 steps per epoch
    seen = torch.stack(seen).cpu()
    assert seen.shape[0] >= 3 and seen.shape[1] == 2 and bool(torch.isfinite(seen).all()), seen
    ck = torch.load(os.path.join(tmp_path, 'log', 'ckpt', 'model-3.pth'))
    fresh = RegTR(cfg)
    fresh.load_state_dict(ck['state_dict'], strict=True)
