"""Data-parallel training throughput: steps/s and pairs/s of `Trainer.dp_training_step` at W = 1, 2, ... ranks, one
GPU per rank, on synthetic ModelNet40 shapes with the global batch fixed.

    python scripts/bench_train_dp.py [--batch 8] [--steps 20] [--warmup 5] [--max-world N]

W = 1 runs the single-GPU `Trainer.training_step`; W > 1 starts W processes (spawn, a FileStore in a temporary
directory, NCCL).  A world size larger than the visible GPU count is reported as "not measured".  Prints one JSON line
with the GPU name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from datetime import timedelta
from types import SimpleNamespace

import torch
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) if torch.cuda.is_available() else 'unknown'


def _run(rank, world, args, store_path, out_path):
    from regtr_b200 import dist as D
    from regtr_b200 import modelnet as MN
    from regtr_b200 import trainer as T
    from regtr_b200.config import get_config
    from regtr_b200.regtr import RegTR
    from regtr_b200.synthetic import make_modelnet_shapes
    from regtr_b200.weights import random_state_dict
    dev = torch.device('cuda', rank)
    torch.cuda.set_device(dev)
    group = None
    if world > 1:
        torch.distributed.init_process_group('nccl', store=torch.distributed.FileStore(store_path, world), rank=rank,
                                             world_size=world, timeout=timedelta(seconds=600), device_id=dev)
        group = torch.distributed.group.WORLD
    try:
        cfg = get_config('modelnet', train_batch_size=args.batch)
        shapes = MN.ModelNetShapes.from_arrays(make_modelnet_shapes(max(2 * args.batch, 16), seed=3))
        model = RegTR(cfg)
        model.load_state_dict(random_state_dict(cfg, 1), strict=True)
        with tempfile.TemporaryDirectory() as logdir:
            opt = SimpleNamespace(log_path=logdir, resume=None, debug=False, summary_every=10 ** 9,
                                  validate_every=10 ** 9, nb_sanity_val_steps=0, num_workers=1)
            tr = T.Trainer(opt, niter=args.steps, grad_clip=cfg.grad_clip, seed=0, process_group=group)
            tr.setup(model, shapes)
            order = T.epoch_batches(0, 0, len(shapes), args.batch)

            def step(s):
                bt = order[s % len(order)]
                if len(bt) < args.batch:
                    bt = order[0]
                if group is None:
                    tr.training_step(model, {'idx': bt}, s + 1)
                else:
                    lo, part = T.shard_slice(bt, rank, world)
                    tr.dp_training_step(model, {'idx': part}, lo, s + 1)
            for s in range(args.warmup):
                step(s)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for s in range(args.warmup, args.warmup + args.steps):
                step(s)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            tr.close()
        if rank == 0:
            with open(out_path, 'w') as f:
                json.dump(dict(seconds=dt), f)
    finally:
        if group is not None:
            torch.distributed.destroy_process_group()


def measure(world, args):
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, 'result.json')
        if world == 1:
            _run(0, 1, args, None, out)
        else:
            ctx = mp.get_context('spawn')
            procs = [ctx.Process(target=_run, args=(r, world, args, os.path.join(tmp, 'store'), out))
                     for r in range(world)]
            try:
                for p in procs:
                    p.start()
                for p in procs:
                    p.join(timeout=1800)
                if any(p.exitcode != 0 for p in procs):
                    raise RuntimeError(f'world {world}: exit codes {[p.exitcode for p in procs]}')
            finally:
                for p in procs:
                    if p.is_alive():
                        p.kill()
                        p.join(10)
        with open(out) as f:
            dt = json.load(f)['seconds']
    return dict(steps_per_s=args.steps / dt, pairs_per_s=args.steps * args.batch / dt, ms_per_step=1e3 * dt / args.steps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8, help='global batch (pairs per step)')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--max-world', type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_dp needs CUDA GPUs')
    n_gpu = torch.cuda.device_count()
    res = {}
    for w in (1, 2, 4, 8):
        if w > args.max_world or w > args.batch:
            continue
        res[str(w)] = measure(w, args) if w <= n_gpu else 'not measured'
    print(json.dumps(dict(gpu=gpu_info(), visible_gpus=n_gpu, batch=args.batch, steps=args.steps, warmup=args.warmup,
                          world=res)))


if __name__ == '__main__':
    main()
