"""Train RegTR on 3DMatch: the reference's `src/train.py` on the library path.

    python -m regtr_b200.train --config 3dmatch [--logdir ../logs] [--name NAME] [--summary_every 500]
        [--validate_every -1] [--debug] [--num_workers 4] [--resume CKPT] [--nb_sanity_val_steps 2]
        [--info-dir datasets/3dmatch] [--seed 0]

--config is a reference-format YAML file (conf/3dmatch.yaml) or a builtin config name.  The training and validation
pairs are listed in <info-dir>/train_info.pkl and <info-dir>/val_info.pkl (the reference reads the same files
relative to its working directory); the clouds are under cfg.root.  Logs, config.yaml, tensorboard summaries and
ckpt/ go to <logdir>/<dataset>/<yymmdd_HHMMSS>[_<name>].  With --resume and no --config, the config.yaml next to the
checkpoint directory is used.  The reference's --dev flag (which deletes a log directory) is not provided.
"""
from __future__ import annotations

import argparse
import logging
import os
import sys
from datetime import datetime

BUILTIN = ('3dmatch', 'modelnet')


def parser() -> argparse.ArgumentParser:
    ap = argparse.ArgumentParser(prog='python -m regtr_b200.train')
    ap.add_argument('--config', type=str, help='Path to the config file, or a builtin config name (3dmatch).')
    ap.add_argument('--logdir', type=str, default='../logs', help='Directory to store logs, summaries, checkpoints.')
    ap.add_argument('--name', type=str, help='Experiment name (used to name output directory')
    ap.add_argument('--summary_every', type=int, default=500, help='Interval to save tensorboard summaries')
    ap.add_argument('--validate_every', type=int, default=-1, help='Validation interval. Default: every epoch')
    ap.add_argument('--debug', action='store_true', help='If set, will enable autograd anomaly detection')
    ap.add_argument('--num_workers', type=int, default=4, help='Number of worker threads for data loading')
    ap.add_argument('--resume', type=str, help='Checkpoint to resume from')
    ap.add_argument('--nb_sanity_val_steps', type=int, default=2,
                    help='Number of validation sanity steps to run before training.')
    ap.add_argument('--info-dir', dest='info_dir', type=str, default=os.path.join('datasets', '3dmatch'),
                    help='Directory of train_info.pkl and val_info.pkl')
    ap.add_argument('--seed', type=int, default=0, help='Seed of the epoch order and the augmentations')
    return ap


def resolve_config(opt) -> str:
    """--config, or the config.yaml one level above the --resume checkpoint's directory (train.py:45-56)."""
    if opt.config is not None:
        return opt.config
    if opt.resume is None or not os.path.exists(opt.resume):
        raise SystemExit('--config needs to be supplied unless resuming from checkpoint')
    folder = opt.resume if os.path.isdir(opt.resume) else os.path.dirname(opt.resume)
    path = os.path.normpath(os.path.join(folder, '../config.yaml'))
    if not os.path.exists(path):
        raise SystemExit(f'Config not found in resume directory: {path}')
    print(f'Using config file from checkpoint directory: {path}')
    return path


def load_cfg(name_or_path: str):
    from .config import get_config, load_config
    if name_or_path in BUILTIN and not os.path.exists(name_or_path):
        return get_config(name_or_path)
    return load_config(name_or_path)


def prepare_logger(opt) -> str:
    """cvhelpers/misc.py prepare_logger: a timestamped log directory, INFO to the console and to log.txt."""
    stamp = datetime.now().strftime('%y%m%d_%H%M%S')
    log_path = os.path.join(opt.logdir, stamp + '_' + opt.name if opt.name is not None else stamp)
    os.makedirs(log_path, exist_ok=True)
    fmt, datefmt = '%(asctime)s [%(levelname)s] %(name)s - %(message)s', '%m/%d %H:%M:%S'
    root = logging.getLogger()
    root.handlers.clear()
    root.setLevel(logging.INFO)
    for h in (logging.StreamHandler(), logging.FileHandler(os.path.join(log_path, 'log.txt'))):
        h.setFormatter(logging.Formatter(fmt, datefmt=datefmt))
        h.setLevel(logging.INFO)
        root.addHandler(h)
    root.info(f'Output and logs will be saved to {log_path}')
    root.info('Command: {}'.format(' '.join(sys.argv)))
    root.info('Arguments: {}'.format(', '.join(f'{k}: {v}' for k, v in vars(opt).items())))
    return log_path


def write_config(cfg, source: str, out: str):
    """config.yaml of the log directory: the source file with a header line, or a builtin config as one section
    (load_config flattens it back)."""
    import yaml
    with open(out, 'w') as fid:
        fid.write(f'# Original file name: {source}\n')
        if os.path.exists(source):
            with open(source) as src:
                fid.write(src.read())
        else:
            yaml.safe_dump({'config': dict(cfg)}, fid, sort_keys=False)


def main(argv=None):
    opt = parser().parse_args(argv)
    opt.config = resolve_config(opt)
    cfg = load_cfg(opt.config)
    if cfg.dataset == 'modelnet':
        raise NotImplementedError('ModelNet training needs the ModelNet40 h5 loader and its transforms '
                                  '(data_loaders/modelnet.py), which this package does not provide')
    if cfg.dataset != '3dmatch':
        raise NotImplementedError(f'dataset {cfg.dataset!r}')
    opt.logdir = os.path.join(opt.logdir, cfg.dataset)
    if opt.name is None and len(cfg.get('expt_name', '')) > 0:
        opt.name = cfg.expt_name
    opt.log_path = prepare_logger(opt)
    write_config(cfg, opt.config, os.path.join(opt.log_path, 'config.yaml'))

    from .data import ThreeDMatchPairs
    from .regtr import RegTR
    from .trainer import Trainer
    if not os.path.isdir(cfg.root):
        raise AssertionError(f'Dataset not found in {cfg.root}')
    train_set = ThreeDMatchPairs(cfg.root, os.path.join(opt.info_dir, 'train_info.pkl'), pin=True, float64=True)
    val_set = ThreeDMatchPairs(cfg.root, os.path.join(opt.info_dir, 'val_info.pkl'), pin=True, float64=True)
    model = RegTR(cfg)
    trainer = Trainer(opt, niter=cfg.niter, grad_clip=cfg.grad_clip, seed=opt.seed)
    trainer.fit(model, train_set, val_set)
    return opt.log_path


if __name__ == '__main__':
    main()
