"""Data-parallel training (Trainer(..., process_group=...)) against one process on the same global batch.

Two ranks run on one GPU over gloo, started with a spawn context and a FileStore under tmp_path (no network port); the
process group and the join have timeouts and the children are killed in `finally`.  ModelNet-sized synthetic batches
of 2 and 4 pairs (coarse clouds of uneven sizes) check the loss values, the all-reduced gradients, weights bit-identical
across ranks, exact resume, validation and a raising step.  The same gradient check runs over NCCL when two GPUs are
visible."""
import os
import traceback
from datetime import timedelta
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from regtr_b200 import modelnet as MN
from regtr_b200 import trainer as T
from regtr_b200.config import get_config
from regtr_b200.regtr import RegTR
from regtr_b200.synthetic import make_modelnet_shapes
from regtr_b200.weights import random_state_dict

pytestmark = pytest.mark.gpu
W = 2
TIMEOUT_S = 240
# The gradient bound: GRAD_FACTOR x the difference between two single-process runs with the pair order swapped, plus 1e-6
# of the gradient.  A rank's forward runs the GEMMs at its own token count, so their split-K partitions differ from the
# whole batch's, which the pair swap does not exercise: on one H100, B = 2 put 6 of 280 checks (the last cross-encoder
# layer's linear1 and norm3) between 4x and 5.7x the swap's spread, every other check below 4x; B = 4 stayed
# below 2.4x.
GRAD_FACTOR = 8.0
STEPS = {2: [[3, 0], [1, 4], [2, 5]], 4: [[3, 0, 6, 1], [1, 4, 7, 2], [2, 5, 0, 3]]}


def make_cfg(B):
    return get_config('modelnet', train_batch_size=B, val_batch_size=2, base_lr=1e-4)


def train_shapes():
    return MN.ModelNetShapes.from_arrays(make_modelnet_shapes(8, seed=30))


def val_pairs(cfg):
    return MN.ModelNetPairs(MN.ModelNetShapes.from_arrays(make_modelnet_shapes(3, seed=31)), cfg)


def make_opt(log_path, **kw):
    opt = SimpleNamespace(log_path=str(log_path), resume=None, debug=False, summary_every=1000,
                          validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=2)
    opt.__dict__.update(kw)
    return opt


def make_model(cfg, seed=12):
    model = RegTR(cfg)
    model.load_state_dict(random_state_dict(cfg, seed), strict=True)
    return model


def grads_of(model):
    return {n: p.grad.detach().cpu().clone() for n, p in model.named_parameters() if p.grad is not None}


def params_of(model):
    return {n: p.detach().cpu().clone() for n, p in model.named_parameters()}


class FlakyPrep:
    """A batch preparation that raises a Python exception at step index 1 when `fail`."""

    def __init__(self, real, fail):
        self.real, self.fail = real, fail

    step = property(lambda self: self.real.step, lambda self, v: setattr(self.real, 'step', v))

    def __call__(self, batch, **kw):
        if self.fail and self.real.step == 1:
            raise ValueError('injected failure in the batch preparation')
        return self.real(batch, **kw)


# ------------------------------------------------------------------------------------------------- the ranks

def _barrier(group, dev):
    torch.distributed.all_reduce(torch.zeros(1, device=dev), group=group)


def _scenarios(rank, out, group, dev, full):
    import regtr_b200.dist as D
    res = {}
    for B in (2, 4):                 # gradients, losses, 3 steps; rank 1 starts from other weights (broadcast)
        cfg = make_cfg(B)
        model = make_model(cfg, seed=12 if rank == 0 else 99)
        tr = T.Trainer(make_opt(os.path.join(out, f'g{B}')), niter=3, grad_clip=0.0, seed=5, process_group=group)
        tr.setup(model, train_shapes())
        steps = []
        for s, items in enumerate(STEPS[B], start=1):
            lo, hi = D.shard_range(B, rank, W)
            losses = tr.dp_training_step(model, {'idx': items[lo:hi]}, lo, s)
            steps.append(dict(losses={k: float(v) for k, v in losses.items()}, grads=grads_of(model) if s == 1 else None))
        res[f'grad{B}'] = dict(steps=steps, params=params_of(model))
    if not full:
        return res

    # a raising batch preparation on rank 1 at step 2: every rank skips that update, step 3 runs
    cfg = make_cfg(2)
    model = make_model(cfg)
    tr = T.Trainer(make_opt(os.path.join(out, 'err')), niter=3, grad_clip=0.0, seed=5, process_group=group)
    tr.setup(model, train_shapes())
    tr.prep = FlakyPrep(tr.prep, fail=rank == 1)
    snaps, rets = [], []
    for s, items in enumerate(STEPS[2], start=1):
        lo, hi = D.shard_range(2, rank, W)
        rets.append(tr.dp_training_step(model, {'idx': items[lo:hi]}, lo, s) is not None)
        snaps.append(params_of(model))
    res['err'] = dict(ran=rets, same_12=all(torch.equal(snaps[0][k], snaps[1][k]) for k in snaps[0]),
                      moved_3=any(not torch.equal(snaps[1][k], snaps[2][k]) for k in snaps[0]), params=snaps[-1])

    # resume: 2 steps + save + resume + 2 steps against 4 straight steps (5 shapes in batches of 2: the third step of
    # an epoch has one pair and rank 1 none); validation every 2 steps (val batches [0, 1], [2])
    vals = []
    real_finish = T.Trainer._finish_validation

    def spy(self, model, step, val_losses, metrics, save_ckpt):
        vals.append(dict(step=step, losses=dict(val_losses), metrics={k: v for k, v in metrics.items()
                                                                       if not k.endswith('hist')}))
        return real_finish(self, model, step, val_losses, metrics, save_ckpt)
    T.Trainer._finish_validation = spy
    try:
        five = MN.ModelNetShapes.from_arrays(make_modelnet_shapes(5, seed=30))
        for name, niter, resume in (('a', 4, None), ('b', 2, None),
                                    ('c', 2, os.path.join(out, 'b', 'ckpt', 'model-2.pth'))):
            tr = T.Trainer(make_opt(os.path.join(out, name), validate_every=2, resume=resume), niter=niter,
                           grad_clip=cfg.grad_clip, seed=5, process_group=group)
            tr.fit(make_model(cfg), five, val_pairs(cfg))
            _barrier(group, dev)
    finally:
        T.Trainer._finish_validation = real_finish
    res['vals'] = vals
    return res


def _rank_main(rank, backend, store_path, out, full):
    try:
        dev = torch.device('cuda', rank if backend == 'nccl' else 0)
        torch.cuda.set_device(dev)
        store = torch.distributed.FileStore(store_path, W)
        kw = dict(device_id=dev) if backend == 'nccl' else {}
        torch.distributed.init_process_group(backend, store=store, rank=rank, world_size=W,
                                             timeout=timedelta(seconds=TIMEOUT_S), **kw)
        try:
            res = _scenarios(rank, out, torch.distributed.group.WORLD, dev, full)
            torch.save(res, os.path.join(out, f'rank{rank}.pt'))
        finally:
            torch.distributed.destroy_process_group()
    except BaseException:
        with open(os.path.join(out, f'rank{rank}.err'), 'w') as f:
            f.write(traceback.format_exc())
        raise


def run_ranks(tmp_path, backend, full):
    out = str(tmp_path / backend)
    os.makedirs(out, exist_ok=True)
    ctx = mp.get_context('spawn')
    procs = [ctx.Process(target=_rank_main, args=(r, backend, str(tmp_path / f'store_{backend}'), out, full))
             for r in range(W)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=3 * TIMEOUT_S)
        errs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out)) if f.endswith('.err')]
        assert not errs, '\n'.join(errs)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        return [torch.load(os.path.join(out, f'rank{r}.pt')) for r in range(W)]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(10)


# -------------------------------------------------------------------------------------------- one process

def reversed_batch(b):
    """The prepared batch with its pairs in the opposite order: the same math, other summation orders."""
    return {'src_xyz': list(b['src_xyz'])[::-1], 'tgt_xyz': list(b['tgt_xyz'])[::-1],
            'src_overlap': list(b['src_overlap'])[::-1], 'tgt_overlap': list(b['tgt_overlap'])[::-1],
            'pose': torch.flip(b['pose'], dims=[0])}


def single_step(B, items, swap=False):
    cfg = make_cfg(B)
    model = make_model(cfg).cuda()
    prep = MN.ModelNetPrep(cfg, train_shapes().to(torch.device('cuda', 0)), seed=5)
    b = prep(items, step=0)
    if swap:
        b = reversed_batch(b)
    pred = model.forward_train(b, train_encoder=True)
    losses = model.compute_loss(pred, b)
    losses['total'].backward()
    return {k: float(v.detach()) for k, v in losses.items()}, grads_of(model)


def check_gradients(res, B):
    ref_losses, ref = single_step(B, STEPS[B][0])
    _, swp = single_step(B, STEPS[B][0], swap=True)
    for rank in range(W):
        step1 = res[rank][f'grad{B}']['steps'][0]
        assert step1['losses'].keys() == ref_losses.keys()
        for k, v in ref_losses.items():
            assert abs(step1['losses'][k] - v) <= 2e-5 * abs(v) + 1e-6, (B, rank, k, step1['losses'][k], v)
        g = step1['grads']
        assert g.keys() == ref.keys()
        over, worst = [], (0.0, None, None)
        for n in ref:
            base = ref[n].double()
            d_dp, d_sw = (g[n].double() - base), (swp[n].double() - base)
            for what, norm in (('max-abs', lambda t: t.abs().max()), ('frobenius', lambda t: t.norm())):
                ratio = float(norm(d_dp) / (norm(d_sw) + 1e-6 * norm(base) / GRAD_FACTOR))
                worst = max(worst, (ratio, n, what))
                if ratio > GRAD_FACTOR:
                    over.append((n, what, float(norm(d_dp)), float(norm(d_sw)), float(norm(base))))
        assert not over, (B, rank, worst, over)
    for k in res[0][f'grad{B}']['params']:                       # 3 steps: the ranks hold the same weights
        assert torch.equal(res[0][f'grad{B}']['params'][k].view(torch.int32),
                           res[1][f'grad{B}']['params'][k].view(torch.int32)), k


def test_two_ranks_on_one_gpu_equal_one_process(tmp_path):
    res = run_ranks(tmp_path, 'gloo', full=True)
    for B in (2, 4):
        check_gradients(res, B)

    # a raising step: skipped on both ranks, the next step runs, nothing hangs
    for r in range(W):
        e = res[r]['err']
        assert e['ran'] == [True, False, True] and e['same_12'] and e['moved_3'], (r, e['ran'])
    for k in res[0]['err']['params']:
        assert torch.equal(res[0]['err']['params'][k], res[1]['err']['params'][k]), k

    # resume: bit-identical to the straight run, checkpoints written by rank 0 only
    a = torch.load(str(tmp_path / 'gloo' / 'a' / 'ckpt' / 'model-4.pth'))
    c = torch.load(str(tmp_path / 'gloo' / 'c' / 'ckpt' / 'model-4.pth'))
    for key in ('state_dict', 'optimizer'):
        for k in a[key]['state'] if key == 'optimizer' else a[key]:
            x = a[key]['state'][k] if key == 'optimizer' else {'t': a[key][k]}
            y = c[key]['state'][k] if key == 'optimizer' else {'t': c[key][k]}
            for f in x:
                if torch.is_tensor(x[f]):
                    assert torch.equal(x[f].reshape(-1).view(torch.uint8), y[f].reshape(-1).view(torch.uint8)), (k, f)
    assert a['scheduler'] == c['scheduler'] and a['step'] == c['step'] == 4

    # validation: every rank reports the metrics of one process with the same weights
    vals = [v for v in res[0]['vals']]
    assert [v['step'] for v in vals] == [2, 4, 2, 4] and vals == res[1]['vals']
    cfg = make_cfg(2)
    model = make_model(cfg)
    model.load_state_dict(a['state_dict'])
    tr = T.Trainer(make_opt(tmp_path / 'single_val'), niter=1, seed=5)
    tr.setup(model, train_shapes())
    got = {}
    real = T.Trainer._finish_validation
    try:
        T.Trainer._finish_validation = lambda self, m, step, l, met, s: got.update(losses=l, metrics=met) or 0.0
        tr._run_validation(model, val_pairs(cfg), step=4, save_ckpt=False)
    finally:
        T.Trainer._finish_validation = real
    dp = vals[1]
    for k, v in got['metrics'].items():
        if k.endswith('hist'):
            continue
        if k.startswith('reg_success'):
            assert dp['metrics'][k] == v, k
        else:
            assert abs(dp['metrics'][k] - v) <= 1e-4 * abs(v) + 1e-6, (k, dp['metrics'][k], v)
    for k, v in got['losses'].items():
        assert abs(dp['losses'][k] - v) <= 2e-5 * abs(v) + 1e-6, (k, dp['losses'][k], v)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_two_ranks_over_nccl_equal_one_process(tmp_path):
    res = run_ranks(tmp_path, 'nccl', full=False)
    for B in (2, 4):
        check_gradients(res, B)


# --------------------------------------------------------------------------------------------- single process

def test_a_slice_with_its_pair_offset_draws_what_the_whole_batch_draws():
    from regtr_b200 import augment as A
    from regtr_b200.synthetic import make_3dmatch_pair
    dev = torch.device('cuda', 0)
    prep = MN.ModelNetPrep(make_cfg(4), train_shapes().to(dev), seed=5)
    whole, part = prep([3, 0, 6, 1], step=7), prep([6, 1], step=7, pair_base=2)
    for k in ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap'):
        assert all(torch.equal(x, y) for x, y in zip(whole[k][2:], part[k])), k
    assert torch.equal(whole['pose'][2:], part['pose'])
    assert all(torch.equal(x, y) for x, y in zip(whole['correspondences'][2:], part['correspondences']))

    pairs = [make_3dmatch_pair(40 + i, n_target=3000 + 500 * i) for i in range(3)]
    batch = {'src_xyz': [torch.from_numpy(p['src_xyz']).double() for p in pairs],
             'tgt_xyz': [torch.from_numpy(p['tgt_xyz']).double() for p in pairs],
             'pose': torch.from_numpy(np.stack([p['pose'] for p in pairs])).double()}
    prep = A.TrainingPrep(get_config('3dmatch'), seed=3)
    prep.step = 4
    whole = prep(batch)
    prep.step = 4
    part = prep({k: v[1:] for k, v in batch.items()}, pair_base=1)
    for k in ('src_xyz', 'tgt_xyz', 'src_overlap', 'tgt_overlap'):
        assert all(torch.equal(x, y) for x, y in zip(whole[k][1:], part[k])), k
    assert torch.equal(whole['pose'][1:], part['pose'])
    assert all(torch.equal(x, y) for x, y in zip(whole['correspondences'][1:], part['correspondences']))
    prep.check()


def test_one_rank_normalisers_are_bit_identical_to_the_plain_loss():
    from regtr_b200 import losses as LS
    cfg = make_cfg(4)
    model = make_model(cfg).cuda()
    b = MN.ModelNetPrep(cfg, train_shapes().to(torch.device('cuda', 0)), seed=5)(STEPS[4][0], step=0)
    out = []
    for reduce in (None, lambda norm: None):
        model.zero_grad(set_to_none=True)
        pred = model.forward_train(b, train_encoder=True)
        losses = LS.compute_loss_device(model, pred, b, reduce_norms=reduce)
        losses['total'].backward()
        out.append(({k: v.detach().cpu() for k, v in losses.items()}, grads_of(model)))
    (la, ga), (lb, gb) = out
    assert la.keys() == lb.keys() and ga.keys() == gb.keys()
    for k in la:
        assert torch.equal(la[k].view(torch.int32), lb[k].view(torch.int32)), k
    for k in ga:
        assert torch.equal(ga[k].view(torch.int32), gb[k].view(torch.int32)), k
