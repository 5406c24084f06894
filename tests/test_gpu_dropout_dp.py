"""Data-parallel training with transformer dropout: two ranks on one GPU over gloo (the harness of test_gpu_dp.py)
against one process.  Each rank's masks are those of its global pairs, bit for bit, and the all-reduced gradients of a
dropout 0.1 step match the one-process step within test_gpu_dp.py's criterion."""
import os
import traceback
from datetime import timedelta

import pytest
import torch
import torch.multiprocessing as mp

import test_gpu_dp as H
from regtr_b200 import modelnet as MN
from regtr_b200 import trainer as T

pytestmark = pytest.mark.gpu

P, SEED, B = 0.1, 5, 2
ITEMS = H.STEPS[2][0]
MASK_SITES = [(layer, site, head) for layer in (0, 5) for site in (1, 2, 3, 4, 5, 6)
              for head in ((0, 7) if site in (1, 3) else (0,))]


def make_cfg():
    cfg = H.make_cfg(B)
    cfg.dropout = P
    return cfg


def _rank_main(rank, store_path, out):
    try:
        import regtr_b200.dist as D
        from regtr_b200 import ops
        dev = torch.device('cuda', 0)
        torch.cuda.set_device(dev)
        store = torch.distributed.FileStore(store_path, H.W)
        torch.distributed.init_process_group('gloo', store=store, rank=rank, world_size=H.W,
                                             timeout=timedelta(seconds=H.TIMEOUT_S))
        try:
            model = H.make_model(make_cfg(), seed=12 if rank == 0 else 99)
            tr = T.Trainer(H.make_opt(os.path.join(out, 'g')), niter=1, grad_clip=0.0, seed=SEED,
                           process_group=torch.distributed.group.WORLD)
            tr.setup(model, H.train_shapes())
            keys, real = [], model.forward_train

            def forward_train(batch, train_encoder=False, **kw):
                keys.append(kw.get('dropout_key'))
                return real(batch, train_encoder=train_encoder, **kw)
            model.forward_train = forward_train
            lo, hi = D.shard_range(B, rank, H.W)
            losses = tr.dp_training_step(model, {'idx': ITEMS[lo:hi]}, lo, 1)
            (seed, step, pair_base), n_local = keys[0], hi - lo
            masks = {(layer, site, head, side): ops.dropout_keep_mask(P, seed, step, pair_base, n_local, side * n_local,
                                                                      layer, site, head, 64, 96).cpu()
                     for layer, site, head in MASK_SITES for side in (0, 1)}
            res = dict(keys=keys, lo=lo, losses={k: float(v) for k, v in losses.items()}, grads=H.grads_of(model),
                       masks=masks)
            torch.save(res, os.path.join(out, f'rank{rank}.pt'))
        finally:
            torch.distributed.destroy_process_group()
    except BaseException:
        with open(os.path.join(out, f'rank{rank}.err'), 'w') as f:
            f.write(traceback.format_exc())
        raise


def _one_process():
    cfg = make_cfg()
    model = H.make_model(cfg).cuda()
    prep = MN.ModelNetPrep(cfg, H.train_shapes().to(torch.device('cuda', 0)), seed=SEED)
    b = prep(ITEMS, step=0)
    losses = model.compute_loss(model.forward_train(b, train_encoder=True, dropout_key=(SEED, 1, 0)), b)
    losses['total'].backward()
    return {k: float(v.detach()) for k, v in losses.items()}, H.grads_of(model)


def test_two_ranks_draw_the_masks_of_their_global_pairs_and_match_one_process(tmp_path):
    from regtr_b200 import ops
    out = str(tmp_path / 'gloo')
    os.makedirs(out, exist_ok=True)
    ctx = mp.get_context('spawn')
    procs = [ctx.Process(target=_rank_main, args=(r, str(tmp_path / 'store'), out)) for r in range(H.W)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=3 * H.TIMEOUT_S)
        errs = [open(os.path.join(out, f)).read() for f in sorted(os.listdir(out)) if f.endswith('.err')]
        assert not errs, '\n'.join(errs)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        res = [torch.load(os.path.join(out, f'rank{r}.pt')) for r in range(H.W)]
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join(10)
    # masks: rank r's local clouds are global pair lo_r's src / tgt clouds of the one-process batch
    for r in range(H.W):
        assert res[r]['keys'] == [(SEED, 1, res[r]['lo'])]
        for (layer, site, head, side), m in res[r]['masks'].items():
            whole = ops.dropout_keep_mask(P, SEED, 1, 0, B, res[r]['lo'] + side * B, layer, site, head, 64, 96).cpu()
            assert torch.equal(m, whole), (r, layer, site, head, side)
    # gradients: within GRAD_FACTOR of the spread a pair-order swap gives at dropout 0 (the dropout masks follow the
    # pairs, so a swapped batch would draw other masks for the same position)
    ref_losses, ref = _one_process()
    _, base0 = H.single_step(B, ITEMS)
    _, swp0 = H.single_step(B, ITEMS, swap=True)
    for r in range(H.W):
        for k, v in ref_losses.items():
            assert abs(res[r]['losses'][k] - v) <= 2e-5 * abs(v) + 1e-6, (r, k, res[r]['losses'][k], v)
        g = res[r]['grads']
        assert g.keys() == ref.keys()
        over, worst = [], (0.0, None, None)
        for n in ref:
            base = ref[n].double()
            d_dp, d_sw = g[n].double() - base, swp0[n].double() - base0[n].double()
            for what, norm in (('max-abs', lambda t: t.abs().max()), ('frobenius', lambda t: t.norm())):
                ratio = float(norm(d_dp) / (norm(d_sw) + 1e-6 * norm(base) / H.GRAD_FACTOR))
                worst = max(worst, (ratio, n, what))
                if ratio > H.GRAD_FACTOR:
                    over.append((n, what, float(norm(d_dp)), float(norm(d_sw)), float(norm(base))))
        print('rank', r, 'worst ratio', worst)
        assert not over, (r, worst, over)
