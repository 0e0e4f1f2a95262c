"""DistributedSampler index math vs torch.utils.data.DistributedSampler as the oracle
(ref: ddp_example.py:70-72)."""
import itertools

import pytest
import torch
from torch.utils.data.distributed import DistributedSampler as TorchDS

from pytorch_distributed_train_b200.data import BatchSampler, DataLoader, DistributedSampler, SyntheticMNIST


class _DS:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


@pytest.mark.parametrize("n,replicas,shuffle,drop_last,seed,epoch", [
    (n, w, sh, dl, seed, ep)
    for n, w in [(10, 3), (7, 4), (60000, 8), (100, 1), (5, 8), (64, 2)]
    for sh, dl in itertools.product([True, False], [True, False])
    for seed, ep in [(0, 0), (3, 2)]
])
def test_matches_torch(n, replicas, shuffle, drop_last, seed, epoch):
    ds = _DS(n)
    for rank in range(replicas):
        ours = DistributedSampler(ds, replicas, rank, shuffle=shuffle, seed=seed, drop_last=drop_last)
        ref = TorchDS(ds, replicas, rank, shuffle=shuffle, seed=seed, drop_last=drop_last)
        ours.set_epoch(epoch)
        ref.set_epoch(epoch)
        assert list(ours) == list(ref)
        assert len(ours) == len(ref)


def test_shards_partition_dataset():
    ds = _DS(60000)
    seen = []
    for r in range(8):
        seen += list(DistributedSampler(ds, 8, r))
    assert sorted(seen) == list(range(60000))


def test_steps_per_epoch_match_reference():
    # 600/300/150/75 steps at 1/2/4/8 GPUs with batch 100
    ds = SyntheticMNIST(60000)
    for w, steps in [(1, 600), (2, 300), (4, 150), (8, 75)]:
        s = DistributedSampler(ds, w, 0)
        assert len(DataLoader(ds, batch_size=100, sampler=s)) == steps


def test_same_permutation_without_set_epoch():
    s = DistributedSampler(_DS(50), 2, 0)
    assert list(s) == list(s)
    a = list(s)
    s.set_epoch(1)
    assert list(s) != a


def test_invalid_rank():
    with pytest.raises(ValueError):
        DistributedSampler(_DS(4), 2, 2)


def test_batch_sampler():
    assert list(BatchSampler(range(7), 3, False)) == [[0, 1, 2], [3, 4, 5], [6]]
    assert list(BatchSampler(range(7), 3, True)) == [[0, 1, 2], [3, 4, 5]]


@pytest.mark.parametrize("n,world,shuffle,drop_last", [(103, 4, True, False), (103, 4, True, True), (10, 4, False, False), (3, 8, True, False)])
def test_indices_tensor_is_the_iterated_sequence(n, world, shuffle, drop_last):
    ds = list(range(n))
    for rank in range(world):
        s = DistributedSampler(ds, num_replicas=world, rank=rank, shuffle=shuffle, drop_last=drop_last, seed=3)
        for epoch in (0, 1):
            s.set_epoch(epoch)
            assert s.indices_tensor().tolist() == list(iter(s))
            assert s.indices_tensor() is s.indices_tensor()   # cached until the epoch changes
