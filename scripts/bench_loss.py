"""Time the training loss on its two routes in one process: the loss kernels (losses.compute_loss_device, what
RegTR.compute_loss takes for the model's own outputs) against the torch restatement (losses.compute_loss called
directly on the same pred).

    python scripts/bench_loss.py [--steps K] [--blocks N] [--warmup W]

Workloads and targets of scripts/bench_train.py: BASELINE config 2 at 1 pair per step and config 3 at 8, seeded
random weights, synthetic 3DMatch-shaped pairs, identity ground-truth pose and seeded level-0 overlap masks.  Per
workload, after a warm-up of both routes, blocks alternate device / torch / device / torch and report
  * loss_ms: CUDA-event time of loss forward + loss backward alone (the predictions as detached packed leaves),
  * step_ms: host-clock time of forward_train(train_encoder=True) + loss + backward() per step over a block of
    --steps steps ending in a synchronise; median and range over the blocks,
  * launches, syncs: library kernel launches (ops.LAUNCHES) and synchronisations counted by
    torch.cuda.set_sync_debug_mode('warn') in one untimed full step.
The 256 MB L2 flush between steps of the loss_ms measurement is not timed.  Prints one JSON line per workload with the
card's name and power limit.  Writes nothing to disk.
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench_train import POOL, WEIGHT_SEED, card  # noqa: E402
from regtr_b200 import losses, ops  # noqa: E402
from regtr_b200.config import get_config  # noqa: E402
from regtr_b200.regtr import RegTR  # noqa: E402
from regtr_b200.synthetic import make_batch  # noqa: E402
from regtr_b200.weights import random_state_dict  # noqa: E402

PACKED = ('both_un', 'cond', 'corr', 'logit')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=50, help='steps per block')
    ap.add_argument('--blocks', type=int, default=3, help='blocks per route')
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_loss.py needs a CUDA device (no CPU fallback)'
    dev = torch.device('cuda:0')
    cfg = get_config('3dmatch')
    model = RegTR(cfg).to(dev)
    model.load_state_dict(random_state_dict(cfg, WEIGHT_SEED), strict=True)
    b = make_batch(2, POOL)
    pool = [(torch.from_numpy(s).to(dev), torch.from_numpy(t).to(dev)) for s, t in zip(b['src_xyz'], b['tgt_xyz'])]
    gen = torch.Generator().manual_seed(WEIGHT_SEED)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    routes = {'device': lambda pred, batch: losses.compute_loss_device(model, pred, batch),
              'torch': lambda pred, batch: losses.compute_loss(model, pred, batch)}
    name, power = card()

    for config, B in ((2, 1), (3, 8)):
        def make(i):
            ids = [(i * B + j) % POOL for j in range(B)]
            batch = {'src_xyz': [pool[k][0] for k in ids], 'tgt_xyz': [pool[k][1] for k in ids],
                     'pose': torch.eye(3, 4, device=dev).expand(B, 3, 4).contiguous()}
            batch['src_overlap'] = [(torch.rand(len(s), generator=gen) < 0.5).to(dev) for s in batch['src_xyz']]
            batch['tgt_overlap'] = [(torch.rand(len(t), generator=gen) < 0.5).to(dev) for t in batch['tgt_xyz']]
            return batch

        def full_step(route, batch):
            model.zero_grad(set_to_none=True)
            routes[route](model.forward_train(batch, train_encoder=True), batch)['total'].backward()

        def loss_only(route, pred, batch, evs=None):
            core = {k: (v.detach().requires_grad_(True) if k in PACKED else v) for k, v in pred.core.items()}
            lens_c = batch['kpconv_meta']['_lens'][-1]
            leaf = RegTR._assemble(core, lens_c, B)
            model.zero_grad(set_to_none=True)
            if evs:
                flush.zero_()
                evs[0].record()
            routes[route](leaf, batch)['total'].backward()
            if evs:
                evs[1].record()

        batches = [make(i) for i in range(POOL)]
        for i in range(args.warmup):
            for route in routes:
                full_step(route, batches[i % POOL])
        pred = model.forward_train(batches[0], train_encoder=True)
        for route in routes:
            loss_only(route, pred, batches[0])
        torch.cuda.synchronize()

        counts = {}
        for route in routes:
            n0 = ops.LAUNCHES
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter('always')
                torch.cuda.set_sync_debug_mode('warn')
                try:
                    full_step(route, batches[0])
                finally:
                    torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
            counts[route] = (ops.LAUNCHES - n0, sum('synchroniz' in str(x.message) for x in w))

        loss_ms = {r: [] for r in routes}
        step_ms = {r: [] for r in routes}
        for _ in range(args.blocks):
            for route in routes:
                evs = [[torch.cuda.Event(enable_timing=True) for _ in range(2)] for _ in range(args.steps)]
                for e in evs:
                    loss_only(route, pred, batches[0], e)
                torch.cuda.synchronize()
                loss_ms[route].append(sum(e[0].elapsed_time(e[1]) for e in evs) / args.steps)
                t0 = time.perf_counter()
                for i in range(args.steps):
                    full_step(route, batches[i % POOL])
                torch.cuda.synchronize()
                step_ms[route].append((time.perf_counter() - t0) * 1e3 / args.steps)
        stat = lambda v: dict(median=statistics.median(v), min=min(v), max=max(v))
        print(json.dumps(dict(
            metric='training loss, forward + backward: loss kernels (device) against the torch restatement',
            workload=f'BASELINE config {config}: synthetic 3DMatch-like pairs, ~20k pts/cloud, {B} pair(s)/step',
            steps_per_block=args.steps, blocks=args.blocks,
            loss_ms={r: stat(loss_ms[r]) for r in routes}, step_ms={r: stat(step_ms[r]) for r in routes},
            launches_per_step={r: counts[r][0] for r in routes}, syncs_per_step={r: counts[r][1] for r in routes},
            gpu=name, power_limit=power)), flush=True)


if __name__ == '__main__':
    main()
