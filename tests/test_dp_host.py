"""Host side of data-parallel training: batch sharding, pair-keyed host draws of rank slices, the setup checks, the
torchrun environment, and that only rank 0 writes to the log directory."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from regtr_b200 import augment as A
from regtr_b200 import dist as D
from regtr_b200 import modelnet as MN
from regtr_b200 import trainer as T


class FakeGroup:
    def __init__(self, rank, size):
        self._rank, self._size = rank, size

    def rank(self):
        return self._rank

    def size(self):
        return self._size


@pytest.mark.parametrize('n', [1, 2, 3, 4, 7, 16, 33])
@pytest.mark.parametrize('world', [1, 2, 3, 8])
def test_shard_range_covers_the_batch_in_balanced_contiguous_slices(n, world):
    parts = [D.shard_range(n, r, world) for r in range(world)]
    assert parts[0][0] == 0 and parts[-1][1] == n
    assert all(parts[r][1] == parts[r + 1][0] for r in range(world - 1))
    sizes = [hi - lo for lo, hi in parts]
    assert max(sizes) - min(sizes) <= 1 and sizes == sorted(sizes, reverse=True)


@pytest.mark.parametrize('B,world', [(1, 1), (2, 2), (4, 2), (5, 2), (7, 3), (8, 8)])
def test_host_draws_of_rank_slices_concatenate_to_the_whole_batch(B, world):
    whole = A.sample_draws(11, 5, B)
    parts = [A.sample_draws(11, 5, hi - lo, lo) for lo, hi in (D.shard_range(B, r, world) for r in range(world))]
    for k, v in whole.items():
        assert np.array_equal(np.concatenate([p[k] for p in parts]), v), k

    fake = SimpleNamespace(seed=11, trans_mag=0.5, rot_mag=45.0)
    whole = MN.ModelNetPrep.draws(fake, 5, B)
    parts = [MN.ModelNetPrep.draws(fake, 5, hi - lo, lo) for lo, hi in (D.shard_range(B, r, world) for r in range(world))]
    for k, v in whole.items():
        assert np.array_equal(np.concatenate([p[k] for p in parts]), v), k


def test_a_batch_smaller_than_the_world_is_rejected():
    D.check_batch_size(2, 2)
    D.check_batch_size(5, 4)
    with pytest.raises(ValueError, match='smaller than the world size'):
        D.check_batch_size(1, 2)


def test_torchrun_environment():
    assert D.torchrun_env({}) is None
    assert D.torchrun_env({'WORLD_SIZE': '4', 'RANK': '2', 'LOCAL_RANK': '2'}) == (2, 4, 2)
    assert D.torchrun_env({'WORLD_SIZE': '1'}) == (0, 1, 0)
    for bad in ({'WORLD_SIZE': '2', 'RANK': '2'}, {'WORLD_SIZE': '0'}, {'WORLD_SIZE': 'x'},
                {'WORLD_SIZE': '2', 'RANK': '1', 'LOCAL_RANK': '-1'}):
        with pytest.raises(ValueError):
            D.torchrun_env(bad)
    from regtr_b200.train import init_distributed
    assert init_distributed({}) is None and init_distributed({'WORLD_SIZE': '1'}) is None


def _opt(path):
    return SimpleNamespace(log_path=str(path), resume=None, debug=False, summary_every=1000, validate_every=10,
                           nb_sanity_val_steps=0, num_workers=1)


def test_only_rank_zero_writes(tmp_path):
    t1 = T.Trainer(_opt(tmp_path / 'r1'), niter=1, process_group=FakeGroup(1, 2))
    assert (t1.rank, t1.world) == (1, 2) and t1.group is not None
    assert t1.train_writer is None and t1.val_writer is None
    model = torch.nn.Linear(2, 2)
    model.optimizer = model.scheduler = None
    t1._trainer_info = {}
    t1._finish_validation(model, 3, {}, {'reg_success_final': 1.0}, save_ckpt=True)
    assert not os.path.exists(tmp_path / 'r1')

    t0 = T.Trainer(_opt(tmp_path / 'r0'), niter=1, process_group=FakeGroup(0, 2))
    assert os.path.isfile(tmp_path / 'r0' / 'ckpt' / 'checkpoints.txt')
    t0._trainer_info = {}
    t0._finish_validation(model, 3, {}, {'reg_success_final': 1.0}, save_ckpt=True)
    assert os.path.isfile(tmp_path / 'r0' / 'ckpt' / 'model-3.pth')
    t0.close()

    single = T.Trainer(_opt(tmp_path / 's'), niter=1, process_group=FakeGroup(0, 1))
    assert single.group is None and single.world == 1
    single.close()
