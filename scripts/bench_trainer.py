"""Cost of the training loop over the bare training step.

    python scripts/bench_trainer.py [--pairs 2] [--dataset 8] [--steps 10] [--rounds 6] [--warmup 3] [--workers 4]

Writes a temporary 3DMatch-format dataset of synthetic ~20k-point pairs (synthetic.make_3dmatch_pair, float64 clouds
and info pickle, as the reference stores them) and deletes it afterwards.  In one process, alternating blocks of
--steps steps for --rounds rounds, it times:
  * loop:  Trainer.training_step on the batches of data.PairStream (read-ahead threads, pinned float64 clouds):
           TrainingPrep + forward_train(train_encoder=True) + compute_loss + backward + clip + AdamW + StepLR + the meter
           launch; validation and summaries off;
  * bare:  the step of `scripts/bench_train.py --train-encoder --optimizer library` (forward_train + compute_loss +
           backward + clip_grad_norm_ + AdamW.step + StepLR.step) on the same pairs, prepared beforehand and resident on
           the device.
Each block ends with a device synchronise and is timed with the host clock.  The difference is what the loop adds:
reading and preparing the batch, and its own bookkeeping.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import pickle
import statistics
import sys
import tempfile
import time
from types import SimpleNamespace

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_train import card  # noqa: E402
from regtr_b200 import data as D  # noqa: E402
from regtr_b200 import ops  # noqa: E402
from regtr_b200 import optim  # noqa: E402
from regtr_b200.augment import TrainingPrep  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.regtr import RegTR  # noqa: E402
from regtr_b200.synthetic import make_3dmatch_pair  # noqa: E402
from regtr_b200.trainer import Trainer, epoch_batches  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

WEIGHT_SEED = 2024


def write_dataset(root, n_pairs, n_pts=20000):
    infos = dict(rot=[], trans=[], src=[], tgt=[], overlap=[])
    os.makedirs(os.path.join(root, 'train', 'scene'))
    for i in range(n_pairs):
        p = make_3dmatch_pair(500 + i, n_target=n_pts)
        rels = [f'train/scene/cloud_bin_{2 * i}.pth', f'train/scene/cloud_bin_{2 * i + 1}.pth']
        for rel, x in zip(rels, (p['src_xyz'], p['tgt_xyz'])):
            torch.save(np.asarray(x, np.float64), os.path.join(root, rel))
        pose = np.asarray(p['pose'], np.float64)
        infos['rot'].append(pose[:, :3]); infos['trans'].append(pose[:, 3:])
        infos['src'].append(rels[0]); infos['tgt'].append(rels[1]); infos['overlap'].append(0.5)
    info = os.path.join(root, 'train_info.pkl')
    with open(info, 'wb') as f:
        pickle.dump(infos, f)
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=2, help='pairs per step (cfg.train_batch_size)')
    ap.add_argument('--dataset', type=int, default=8, help='pairs in the temporary dataset')
    ap.add_argument('--steps', type=int, default=10, help='steps per timed block')
    ap.add_argument('--rounds', type=int, default=6, help='alternations of a loop block and a bare block')
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--workers', type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_trainer.py needs a CUDA device (no CPU fallback)'
    cfg = get_config('3dmatch', train_batch_size=args.pairs)
    with tempfile.TemporaryDirectory(prefix='regtr_bench_trainer_') as tmp:
        info = write_dataset(tmp, args.dataset)
        ds = D.ThreeDMatchPairs(tmp, info, pin=True, float64=True)
        model = RegTR(cfg)
        model.load_state_dict(random_state_dict(cfg, WEIGHT_SEED), strict=True)
        opt = SimpleNamespace(log_path=os.path.join(tmp, 'log'), resume=None, debug=False, summary_every=10 ** 9,
                              validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=args.workers)
        trainer = Trainer(opt, niter=10 ** 9, grad_clip=cfg.grad_clip, seed=0)
        trainer.setup(model, ds)

        # the same pairs, prepared once and kept on the device, for the bare step
        n_batches = -(-len(ds) // args.pairs)
        prep = TrainingPrep(cfg, seed=1)
        order = epoch_batches(0, 0, len(ds), args.pairs)
        resident = [prep(D.collate_pair([ds[i] for i in b])) for b in order]
        prep.check()

        def bare(b):
            losses = model.compute_loss(model.forward_train(b, train_encoder=True), b)
            model.optimizer.zero_grad()
            losses['total'].backward()
            optim.clip_grad_norm_(model.parameters(), max_norm=cfg.grad_clip)
            model.optimizer.step()
            model.scheduler.step()

        total = args.warmup + args.rounds * args.steps
        stream_batches = [b for e in range(-(-total // n_batches)) for b in epoch_batches(0, e, len(ds), args.pairs)]
        stream = iter(D.PairStream(ds, stream_batches, workers=args.workers))
        gs = [0]

        def loop_steps(k):
            for _ in range(k):
                gs[0] += 1
                trainer.training_step(model, next(stream), gs[0])

        loop_steps(args.warmup)
        for i in range(args.warmup):
            bare(resident[i % len(resident)])
        torch.cuda.synchronize()
        loop_ms, bare_ms, k = [], [], 0
        launches = {}
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            n0 = ops.LAUNCHES
            loop_steps(args.steps)
            torch.cuda.synchronize()
            loop_ms.append((time.perf_counter() - t0) * 1e3 / args.steps)
            launches['loop'] = (ops.LAUNCHES - n0) / args.steps
            t0 = time.perf_counter()
            n0 = ops.LAUNCHES
            for _ in range(args.steps):
                bare(resident[k % len(resident)])
                k += 1
            torch.cuda.synchronize()
            bare_ms.append((time.perf_counter() - t0) * 1e3 / args.steps)
            launches['bare'] = (ops.LAUNCHES - n0) / args.steps
        stream.close()
        trainer.close()
        n_pts = int(np.mean([ds[i]['src_xyz'].shape[0] + ds[i]['tgt_xyz'].shape[0] for i in range(len(ds))]) / 2)
    name, power = card()
    lm, bm = statistics.median(loop_ms), statistics.median(bare_ms)
    print(json.dumps(dict(
        metric='ms per training step: Trainer loop (loader + prep + step + meters) vs bare step',
        workload=f'{args.pairs} synthetic 3DMatch-format pair(s)/step, ~{n_pts} pts/cloud, {args.dataset}-pair dataset, '
                 'KPConv encoder trained, clip + library AdamW + StepLR',
        steps_per_block=args.steps, rounds=args.rounds, warmup=args.warmup, workers=args.workers,
        loop_ms_per_step=lm, bare_ms_per_step=bm, loop_overhead_ms=lm - bm, loop_overhead_pct=100.0 * (lm - bm) / bm,
        loop_ms_blocks=[round(x, 3) for x in loop_ms], bare_ms_blocks=[round(x, 3) for x in bare_ms],
        library_launches_per_step=launches, gpu=name, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
