"""Cost of preparing ModelNet40 training batches, and of the training loop's step on them.

    python scripts/bench_modelnet_train.py [--pairs 4] [--shapes 64] [--iters 200] [--steps 10] [--rounds 6]
        [--warmup 3] [--host-batches 20]

Synthetic 2048-point shapes (synthetic.make_modelnet_shapes) stand in for the h5 data; conf/modelnet.yaml's chain
(partial [0.7, 0.7], rot_mag 45, trans_mag 0.5, 717 points per cloud).
  (a) prep:  modelnet.ModelNetPrep per batch of --pairs pairs (host draws, one pinned copy, one launch), timed with
             CUDA events over --iters calls after warm-up; against the host restatement's train chain
             (modelnet.crop_chain with numpy's RandomState) for the same number of pairs, host clock.
  (b) step:  Trainer.training_step on ModelNet batches (ModelNetPrep + forward_train(train_encoder=True) +
             compute_loss + backward + clip + AdamW + StepLR + the meter launch) against the bare step on batches
             prepared beforehand and resident on the device, in alternating blocks of --steps steps for --rounds
             rounds, each block ending with a device synchronise and timed with the host clock.
Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
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
from regtr_b200 import modelnet as MN  # noqa: E402
from regtr_b200 import ops  # noqa: E402
from regtr_b200 import optim  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.regtr import RegTR  # noqa: E402
from regtr_b200.synthetic import make_modelnet_shapes  # noqa: E402
from regtr_b200.trainer import Trainer, epoch_batches  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

WEIGHT_SEED = 2024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--pairs', type=int, default=4, help='pairs per batch (cfg.train_batch_size)')
    ap.add_argument('--shapes', type=int, default=64, help='synthetic training shapes')
    ap.add_argument('--iters', type=int, default=200, help='timed ModelNetPrep calls')
    ap.add_argument('--host-batches', type=int, default=20, help='batches through the host restatement')
    ap.add_argument('--steps', type=int, default=10, help='steps per timed block')
    ap.add_argument('--rounds', type=int, default=6, help='alternations of a loop block and a bare block')
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_modelnet_train.py needs a CUDA device (no CPU fallback)'
    dev = torch.device('cuda', 0)
    cfg = get_config('modelnet', train_batch_size=args.pairs)
    shapes = MN.ModelNetShapes.from_arrays(make_modelnet_shapes(args.shapes, seed=77)).to(dev)
    order = [b for e in range(64) for b in epoch_batches(0, e, len(shapes), args.pairs)]

    # (a) batch preparation
    prep = MN.ModelNetPrep(cfg, shapes, seed=1)
    for i in range(10):
        prep(order[i])
    prep.check()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    h0 = time.perf_counter()
    t0.record()
    for i in range(args.iters):
        prep(order[i % len(order)])
    t1.record()
    t1.synchronize()
    host_enqueue_ms = (time.perf_counter() - h0) * 1e3 / args.iters
    prep_ms = t0.elapsed_time(t1) / args.iters
    prep.check()
    rs = np.random.RandomState(0)
    h0 = time.perf_counter()
    for i in range(args.host_batches):
        for s in order[i % len(order)]:
            MN.crop_chain(shapes.points[s], cfg.partial, cfg.rot_mag, cfg.trans_mag, rs, idx=s)
    host_ms = (time.perf_counter() - h0) * 1e3 / args.host_batches

    # (b) the loop's step against the bare step
    with tempfile.TemporaryDirectory(prefix='regtr_bench_modelnet_') as tmp:
        model = RegTR(cfg)
        model.load_state_dict(random_state_dict(cfg, WEIGHT_SEED), strict=True)
        opt = SimpleNamespace(log_path=os.path.join(tmp, 'log'), resume=None, debug=False, summary_every=10 ** 9,
                              validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=0)
        trainer = Trainer(opt, niter=10 ** 9, grad_clip=cfg.grad_clip, seed=0)
        trainer.setup(model, shapes)
        rprep = MN.ModelNetPrep(cfg, shapes, seed=2)
        resident = [rprep(order[i]) for i in range(16)]
        rprep.check()

        def bare(b):
            losses = model.compute_loss(model.forward_train(b, train_encoder=True), b)
            model.optimizer.zero_grad()
            losses['total'].backward()
            optim.clip_grad_norm_(model.parameters(), max_norm=cfg.grad_clip)
            model.optimizer.step()
            model.scheduler.step()

        gs = [0]

        def loop_steps(k):
            for _ in range(k):
                gs[0] += 1
                trainer.training_step(model, {'idx': order[gs[0] % len(order)]}, gs[0])

        loop_steps(args.warmup)
        for i in range(args.warmup):
            bare(resident[i % len(resident)])
        torch.cuda.synchronize()
        loop_ms, bare_ms, k, launches = [], [], 0, {}
        for _ in range(args.rounds):
            t = time.perf_counter()
            n0 = ops.LAUNCHES
            loop_steps(args.steps)
            torch.cuda.synchronize()
            loop_ms.append((time.perf_counter() - t) * 1e3 / args.steps)
            launches['loop'] = (ops.LAUNCHES - n0) / args.steps
            t = time.perf_counter()
            n0 = ops.LAUNCHES
            for _ in range(args.steps):
                bare(resident[k % len(resident)])
                k += 1
            torch.cuda.synchronize()
            bare_ms.append((time.perf_counter() - t) * 1e3 / args.steps)
            launches['bare'] = (ops.LAUNCHES - n0) / args.steps
        trainer.prep.check()
        trainer.close()
    name, power = card()
    lm, bm = statistics.median(loop_ms), statistics.median(bare_ms)
    print(json.dumps(dict(
        metric='ModelNet training batches: ms per batch (prep) and per training step (loop vs bare)',
        workload=f'{args.pairs} pairs/batch of synthetic 2048-point shapes, partial [0.7, 0.7], 717 points per cloud',
        prep_ms_per_batch=prep_ms, prep_host_enqueue_ms_per_batch=host_enqueue_ms,
        host_restatement_ms_per_batch=host_ms, host_restatement_ms_per_pair=host_ms / args.pairs,
        steps_per_block=args.steps, rounds=args.rounds, warmup=args.warmup,
        loop_ms_per_step=lm, bare_ms_per_step=bm, loop_overhead_ms=lm - bm,
        loop_ms_blocks=[round(x, 3) for x in loop_ms], bare_ms_blocks=[round(x, 3) for x in bare_ms],
        library_launches_per_step=launches, gpu=name, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
