"""ModelNet / ModelLoNet benchmark of a checkpoint on the CUDA path (the reference's `test.py --benchmark ModelNet`):

    python scripts/eval_modelnet.py --root <data/modelnet40_ply_hdf5_2048> --ckpt <model.pth> \
        --benchmark ModelNet|ModelLoNet --out logs/ModelNet [--categories datasets/modelnet/modelnet40_half2.txt]

The test subset filtered by `test_categoryfile`, with the deterministic pairs of `modelnet.ModelNetPairs` at partial
[0.7, 0.7] (ModelNet) or [0.5, 0.5] (ModelLoNet), through `GraphedRegTR` (every cloud has 717 points, so one capacity
bucket serves them all).  Per batch `eval.compute_modelnet_metrics` on the final pose; then the summary in the format
of benchmark_modelnet.print_metrics, and <out>/pred_transforms.npy stacked (n_batches, B, 3, 4) as the reference
saves it.  Reading the h5 files needs h5py."""
import argparse
import logging
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from regtr_b200 import eval as E  # noqa: E402
from regtr_b200 import modelnet as MN  # noqa: E402

PARTIAL = {'ModelNet': [0.7, 0.7], 'ModelLoNet': [0.5, 0.5]}


def print_metrics(logger, summary, title='Metrics'):
    """benchmark_modelnet.print_metrics."""
    logger.info(title + ':')
    logger.info('=' * (len(title) + 1))
    logger.info('DeepCP metrics:{:.4f}(rot-rmse) | {:.4f}(rot-mae) | {:.4g}(trans-rmse) | {:.4g}(trans-mae)'.format(
        summary['r_rmse'], summary['r_mae'], summary['t_rmse'], summary['t_mae']))
    logger.info('Rotation error {:.4f}(deg, mean) | {:.4f}(deg, rmse)'.format(
        summary['err_r_deg_mean'], summary['err_r_deg_rmse']))
    logger.info('Translation error {:.4g}(mean) | {:.4g}(rmse)'.format(summary['err_t_mean'], summary['err_t_rmse']))
    logger.info('Chamfer error: {:.7f}(mean-sq)'.format(summary['chamfer_dist']))


def run_benchmark(forward_fn, pairs: MN.ModelNetPairs, batch_size: int, out_dir: str, device, logger=None):
    """Every pair through `forward_fn(batch) -> pred`: per-batch metrics, the summary, pred_transforms.npy.
    -> (summary dict, per-pair metrics dict, poses (n_batches, B, 3, 4))."""
    logger = logger or logging.getLogger('eval_modelnet')
    per_batch, poses = [], []
    for a in range(0, len(pairs), batch_size):
        batch = pairs.collate(range(a, min(a + batch_size, len(pairs))), device)
        pose = forward_fn(batch)['pose'][-1]
        data = {'points_src': torch.stack(batch['src_xyz']), 'points_ref': torch.stack(batch['tgt_xyz']),
                'points_raw': torch.stack(batch['tgt_raw']), 'transform_gt': batch['pose']}
        per_batch.append(E.compute_modelnet_metrics(data, pose))
        poses.append(pose.detach().cpu().numpy())
    metrics = {k: np.concatenate([m[k] for m in per_batch]) for k in per_batch[0]}
    summary = E.summarize_modelnet_metrics(metrics)
    print_metrics(logger, summary)
    poses = np.stack(poses, axis=0)
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, 'pred_transforms.npy'), poses)
    return summary, metrics, poses


def main(argv=None):
    from regtr_b200.config import get_config
    from regtr_b200.regtr import GraphedRegTR, RegTR
    ap = argparse.ArgumentParser()
    ap.add_argument('--root', required=True)
    ap.add_argument('--ckpt', required=True)
    ap.add_argument('--benchmark', required=True, choices=sorted(PARTIAL))
    ap.add_argument('--out', default='logs')
    ap.add_argument('--categories', default=None, help='test category file (default: the config\'s)')
    args = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO, format='%(asctime)s [%(levelname)s] %(name)s - %(message)s')
    dev = torch.device('cuda:0')
    cfg = get_config('modelnet')
    shapes = MN.ModelNetShapes(args.root, 'test', MN.read_categories(args.categories or cfg.test_categoryfile))
    pairs = MN.ModelNetPairs(shapes, cfg, partial=PARTIAL[args.benchmark])
    model = RegTR(cfg).to(dev).eval()
    state = torch.load(args.ckpt, map_location='cpu')
    model.load_state_dict(state.get('state_dict', state), strict=False)
    runner = GraphedRegTR(model)
    with torch.no_grad():
        run_benchmark(runner, pairs, int(cfg.test_batch_size), args.out, dev)


if __name__ == '__main__':
    main()
